"""Long-context probe: one Llama-3.1-8B sequence at 8K, 32K, 64K and 128K tokens on one GPU.

For each context length it reports the prefill time and rate (algorithmic FLOPs, step_flops), the decode step time,
and, from a second process with ACP_PROFILE=1 (CUDA events around every launch; PDL overlap broken, so only the
shares are meaningful), the prefill attention rate and the decode attention / merge share of a decode step.  Then
the marginal decode K/V bandwidth (ctx_128K - ctx_8K) * kv_bytes_per_token / (t_128K - t_8K): what each extra
cached token costs a decode step.  The card name and power limit are read in the same run.

usage: python scripts/longctx_probe.py [model] [n_new]      (default llama-3.1-8b, 32 decode steps)
"""
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from agentcontrolplane_b200.engine import Engine  # noqa: E402

MODEL = sys.argv[1] if len(sys.argv) > 1 and not sys.argv[1].startswith("-") else "llama-3.1-8b"
N_NEW = int(sys.argv[2]) if len(sys.argv) > 2 and not sys.argv[2].startswith("-") else 32
CTX = [8192, 32768, 65536, 131072]   # prompt + generated tokens
PROFILE = "--profile" in sys.argv


def run_all():
    out = []
    eng = Engine({"model": MODEL, "max_batch": 8, "kv_pages": max(CTX) // 32 + 64, "max_tokens_per_step": 8192,
                  "max_pages_per_seq": max(CTX) // 32, "prefix_cache": False})
    # warm-up: every kernel and tile shape once
    warm = [128000] + [int(t) for t in np.random.default_rng(1).integers(0, 256, size=8191)]
    st, body = eng.complete({"model": MODEL, "max_tokens": 4, "acp": {"prompt_token_ids": warm}})
    assert st == 200, body
    for ctx in CTX:
        plen = ctx - N_NEW
        prompt = [128000] + [int(t) for t in np.random.default_rng(ctx).integers(0, 256, size=plen - 1)]
        eng.stats_reset()
        prof0 = eng.stats().get("profile", {})   # the profile accumulates over the engine's life: take differences
        t0 = time.time()
        st, body = eng.complete({"model": MODEL, "max_tokens": N_NEW,
                                 "acp": {"prompt_token_ids": prompt}})
        wall = time.time() - t0
        assert st == 200, body
        s = eng.stats()
        r = {"ctx": ctx, "prompt": plen, "gen": len(body["acp"]["token_ids"]), "wall_s": round(wall, 2),
             "prefill_ms": round(s["prefill_ms"], 1),
             "prefill_tflops": round(s["prefill_flops_algorithmic"] / (s["prefill_ms"] / 1e3) / 1e12, 1),
             "decode_steps": s["decode_steps"],
             "decode_step_ms": round(s["decode_ms"] / max(1, s["decode_steps"]), 3),
             "decode_step_ms_p50": s.get("decode_step_ms_p50"),
             "kv_bytes_per_token": s["kv_bytes_per_token"]}
        if PROFILE:
            prof = s.get("profile", {})
            pre, dec = ({k: {"ms": v["ms"] - prof0.get(ph, {}).get(k, {"ms": 0.0})["ms"]} for k, v in prof.get(ph, {}).items()}
                        for ph in ("prefill", "decode"))
            # attention FLOPs of the prompt: 4 * q_dim * (query, visible key) pairs * layers (q_dim 4096: the 8B shapes)
            layers = s["layers"]
            pairs = plen * (plen + 1) / 2
            ap = pre.get("attn_prefill", {"ms": 0.0})
            r["attn_prefill_ms"] = round(ap["ms"], 1)
            r["attn_prefill_tflops"] = round(4.0 * 4096 * pairs * layers / (ap["ms"] / 1e3) / 1e12, 1) if ap["ms"] else None
            tot = sum(v["ms"] for v in dec.values()) or 1.0
            for k in ("attn_decode", "attn_merge"):
                v = dec.get(k, {"ms": 0.0})
                r[k + "_us_per_step"] = round(1e3 * v["ms"] / max(1, s["decode_steps"]), 1)
                r[k + "_share"] = round(v["ms"] / tot, 4)
        out.append(r)
        print(json.dumps(r), flush=True)
    eng.close()
    return out


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


if __name__ == "__main__":
    if PROFILE:
        run_all()
        sys.exit(0)
    print(json.dumps({"gpu": gpu_info(), "model": MODEL, "n_new": N_NEW}), flush=True)
    res = run_all()
    a, b = res[0], res[-1]
    dt = (b["decode_step_ms"] - a["decode_step_ms"]) / 1e3
    # cached tokens read by a decode step grow by (ctx_b - ctx_a); both runs average over the same N_NEW steps
    bw = (b["ctx"] - a["ctx"]) * b["kv_bytes_per_token"] / dt if dt > 0 else float("nan")
    print(json.dumps({"marginal_kv_TBps": round(bw / 1e12, 3), "of_3.35_datasheet": round(bw / 3.35e12, 3)}), flush=True)
    print("--- ACP_PROFILE=1 run (separate process)", flush=True)
    env = dict(os.environ, ACP_PROFILE="1")
    subprocess.run([sys.executable, os.path.abspath(__file__), MODEL, str(N_NEW), "--profile"], env=env, check=True)
    print(json.dumps({"gpu": gpu_info()}), flush=True)
