"""Constrained decoding probe: what tool_choice "required" costs a decode step of Llama-3-8B (synthetic weights).

256 sequences decode together; 0, 1, 64 or 256 of them are constrained to the tool-call grammar (csrc/grammar.h),
the rest sample freely.  For each mix it reports the mean and median decode step time, the mean decoding batch,
and kernel launches per step.  A second process with ACP_PROFILE=1 (CUDA events around every launch; PDL overlap
broken, so only per-kernel times are meaningful) reports grammar_mask_kernel's time per launch and per constrained
row.  The card name and power limit are read in the same run.

usage: python scripts/grammar_probe.py [n_new]      (default 48 generated tokens per sequence)
"""
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from agentcontrolplane_b200.engine import Engine  # noqa: E402

MODEL = "llama-3-8b"
SEQS = 256
N_NEW = int(sys.argv[1]) if len(sys.argv) > 1 and not sys.argv[1].startswith("-") else 48
MIXES = [0, 1, 64, 256]
PROFILE = "--profile" in sys.argv
TOOLS = [{"type": "function", "function": {"name": n, "parameters": {"type": "object"}}}
         for n in ("get_weather", "get_time", "search_documents", "send_email")]


def requests(n_constrained, seed):
    rng = np.random.default_rng(seed)
    out = []
    for i in range(SEQS):
        prompt = [128000] + [int(t) for t in rng.integers(0, 256, size=63)]
        r = {"model": MODEL, "max_tokens": N_NEW, "tools": TOOLS, "acp": {"prompt_token_ids": prompt}}
        if i < n_constrained:
            r["tool_choice"] = "required"
        out.append(r)
    return out


def run_mix(eng, n_constrained):
    eng.stats_reset()
    s0 = eng.stats()
    ts = [eng.submit(r) for r in requests(n_constrained, n_constrained + 1)]
    statuses = []
    for t in ts:
        assert eng.wait(t, 600000)
        statuses.append(eng.result(t)[0])
    s = eng.stats()
    steps = s["decode_steps"] + s["prefill_steps"]
    r = {"constrained": n_constrained, "decode_steps": s["decode_steps"],
         "decode_step_ms_mean": round(s["decode_ms"] / max(1, s["decode_steps"]), 3),
         "decode_step_ms_p50": s.get("decode_step_ms_p50"),
         "mean_decode_batch": round(s["decode_tokens"] / max(1, s["decode_steps"]), 1),
         "launches_per_step": round((s["kernel_launches"] - s0["kernel_launches"]) / max(1, steps), 2),
         "status_counts": {str(k): statuses.count(k) for k in sorted(set(statuses))}}
    prof = s.get("profile", {}).get("decode", {}).get("grammar_mask")
    if prof:
        prof0 = s0.get("profile", {}).get("decode", {}).get("grammar_mask", {"n": 0, "ms": 0.0})
        n, ms = prof["n"] - prof0["n"], prof["ms"] - prof0["ms"]
        r["grammar_mask_us_per_launch"] = round(1e3 * ms / max(1, n), 2)
    return r


def run_all():
    eng = Engine({"model": MODEL, "max_batch": SEQS, "kv_pages": 2048, "max_tokens_per_step": 8192, "prefix_cache": False})
    run_mix(eng, 16)   # warm-up: every kernel and batch shape once
    out = []
    for n in MIXES:
        r = run_mix(eng, n)
        if "grammar_mask_us_per_launch" in r:
            # a launch masks the constrained rows of one step; the mean count per step is n while all are decoding
            r["grammar_mask_us_per_row"] = round(r["grammar_mask_us_per_launch"] / max(1, n), 3)
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
    print(json.dumps({"gpu": gpu_info(), "model": MODEL, "seqs": SEQS, "n_new": N_NEW}), flush=True)
    run_all()
    print("--- ACP_PROFILE=1 run (separate process)", flush=True)
    subprocess.run([sys.executable, os.path.abspath(__file__), str(N_NEW), "--profile"],
                   env=dict(os.environ, ACP_PROFILE="1"), check=True)
    print(json.dumps({"gpu": gpu_info()}), flush=True)
