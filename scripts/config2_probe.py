"""BASELINE config 2: Llama-3-8B, 256 concurrent Tasks, prompt lengths log-uniform on [128, 4096]
(seeded), continuous batching, max_tokens 64, 1 GPU.  Prints engine stats as JSON.
usage: python scripts/config2_probe.py [n_tasks] [max_tokens] [layers]
MAX_TOKENS_PER_STEP (default 8192) sets the engine's token rows per prefill step; bench.py runs 4096."""
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from agentcontrolplane_b200.engine import Engine  # noqa: E402

n = int(sys.argv[1]) if len(sys.argv) > 1 else 256
max_new = int(sys.argv[2]) if len(sys.argv) > 2 else 64
rng = np.random.default_rng(0xC0F162)
lens = np.exp(rng.uniform(np.log(128), np.log(4096), size=n)).astype(int)
pages = int(sum((l + max_new) // 32 + 2 for l in lens)) + 64
cfg = {"model": "llama-3-8b", "max_batch": n, "kv_pages": pages, "max_tokens_per_step": int(os.environ.get("MAX_TOKENS_PER_STEP", "8192")),
       "max_pages_per_seq": (4096 + max_new) // 32 + 2, "prefix_cache": False}
if len(sys.argv) > 3:
    cfg["layers"] = int(sys.argv[3])
print("mean prompt len", float(lens.mean()), "kv pages", pages, "=", round(pages * 4 * (cfg.get("layers", 32) / 32) / 1024, 1), "GiB", flush=True)
eng = Engine(cfg)
for rep in range(int(os.environ.get("REPS", "2"))):
    eng.stats_reset()
    t0 = time.time()
    tickets = []
    for i, l in enumerate(lens):
        prompt = [128000] + [int(t) for t in np.random.default_rng(1000 * rep + i).integers(0, 256, size=int(l) - 1)]
        tickets.append(eng.submit({"model": "llama-3-8b", "max_tokens": max_new, "acp": {"prompt_token_ids": prompt}}))
    ntok = 0
    for t in tickets:
        eng.wait(t, -1)
        st, body = eng.result(t)
        assert st == 200, body
        ntok += len(body["acp"]["token_ids"])
    wall = time.time() - t0
    s = eng.stats()
    dec_s = s["decode_ms"] / 1e3
    print(json.dumps({"rep": rep, "tasks": n, "wall_s": round(wall, 3), "reconciles_per_s": round(n / wall, 2),
                      "gen_tokens": ntok, "decode_tok_per_s": round(s["decode_tokens"] / dec_s, 1),
                      "decode_GBps": round(s["decode_bytes_algorithmic"] / dec_s / 1e9, 1),
                      "frac_of_3350": round(s["decode_bytes_algorithmic"] / dec_s / 1e9 / 3350, 3),   # H100 SXM data sheet
                      "decode_step_ms_p50": s.get("decode_step_ms_p50"), "decode_steps": s["decode_steps"],
                      "prefill_ms": round(s["prefill_ms"], 1), "prefill_tok_per_s": round(s["prefill_tokens"] / (s["prefill_ms"] / 1e3), 1),
                      "decode_ms": round(s["decode_ms"], 1)}), flush=True)
if os.environ.get("ACP_PROFILE"):
    prof = eng.stats().get("profile", {})
    for phase in ("decode", "prefill"):
        items = sorted(prof.get(phase, {}).items(), key=lambda kv: -kv[1]["ms"])
        tot = sum(v["ms"] for _, v in items) or 1.0
        print(f"--- {phase} profile (CUDA events per launch, warm cache, PDL overlap broken) total {tot:.2f} ms")
        for k, v in items:
            print(f"{k:24s} n={v['n']:6d} total={v['ms']:9.2f} ms  avg={1e3 * v['ms'] / v['n']:8.2f} us  {100 * v['ms'] / tot:5.1f}%")
eng.close()
