"""Dev probe: N concurrent requests of fixed prompt length through the C ABI; prints engine stats.
usage: python scripts/engine_probe.py [model] [n_requests] [prompt_len] [max_tokens] [layers]"""
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from agentcontrolplane_b200.engine import Engine  # noqa: E402

model = sys.argv[1] if len(sys.argv) > 1 else "llama-3-8b"
n_req = int(sys.argv[2]) if len(sys.argv) > 2 else 64
plen = int(sys.argv[3]) if len(sys.argv) > 3 else 512
max_new = int(sys.argv[4]) if len(sys.argv) > 4 else 64
cfg = {"model": model, "max_batch": max(64, n_req), "kv_pages": n_req * ((plen + max_new) // 32 + 2) + 8,
       "max_tokens_per_step": 8192, "max_pages_per_seq": max(32, (plen + max_new) // 32 + 2)}
if len(sys.argv) > 5:
    cfg["layers"] = int(sys.argv[5])
if os.environ.get("MTPS"):
    cfg["max_tokens_per_step"] = int(os.environ["MTPS"])
if os.environ.get("TP"):
    cfg["tp"] = int(os.environ["TP"])
t0 = time.time()
eng = Engine(cfg)
print("init s:", round(time.time() - t0, 2), flush=True)
for rep in range(int(os.environ.get('REPS', '3'))):
    eng.stats_reset()
    rng = np.random.default_rng(rep)
    t0 = time.time()
    tickets = []
    for i in range(n_req):
        prompt = [128000] + [int(t) for t in rng.integers(0, 256, size=plen - 1)]
        tickets.append(eng.submit({"model": model, "max_tokens": max_new, "acp": {"prompt_token_ids": prompt}}))
    for t in tickets:
        eng.wait(t, -1)
    wall = time.time() - t0
    ntok = 0
    for t in tickets:
        st, body = eng.result(t)
        assert st == 200, body
        ntok += len(body["acp"]["token_ids"])
    s = eng.stats()
    dec_tps = s["decode_tokens"] / (s["decode_ms"] / 1e3) if s["decode_ms"] else 0
    gbs = s.get("decode_bytes_algorithmic_per_gpu", s["decode_bytes_algorithmic"]) / (s["decode_ms"] / 1e3) / 1e9 if s["decode_ms"] else 0
    print(json.dumps({"rep": rep, "wall_s": round(wall, 3), "gen_tokens": ntok,
                      "reconciles_per_s": round(n_req / wall, 2),
                      "tp": s.get("tp", 1), "decode_tok_per_s": round(dec_tps, 1), "decode_GBps_per_gpu": round(gbs, 1),
                      "frac_of_3350": round(gbs / 3350, 3),   # H100 SXM data sheet
                      "decode_step_ms_p50": s.get("decode_step_ms_p50"),
                      "prefill_ms": round(s["prefill_ms"], 2), "prefill_tokens": s["prefill_tokens"],
                      "prefill_tok_per_s": round(s["prefill_tokens"] / (s["prefill_ms"] / 1e3), 1) if s["prefill_ms"] else 0,
                      "decode_ms": round(s["decode_ms"], 2), "decode_steps": s["decode_steps"]}), flush=True)
if os.environ.get("ACP_PROFILE"):
    prof = eng.stats().get("profile", {})
    for phase in ("decode", "prefill"):
        items = sorted(prof.get(phase, {}).items(), key=lambda kv: -kv[1]["ms"])
        tot = sum(v["ms"] for _, v in items) or 1.0
        print(f"--- {phase} profile (CUDA events per launch, warm cache, PDL overlap broken) total {tot:.2f} ms")
        for k, v in items:
            print(f"{k:24s} n={v['n']:6d} total={v['ms']:9.2f} ms  avg={1e3 * v['ms'] / v['n']:8.2f} us  {100 * v['ms'] / tot:5.1f}%")
eng.close()
