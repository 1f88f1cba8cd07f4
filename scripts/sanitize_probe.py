"""Small end-to-end workload for compute-sanitizer (memcheck / racecheck / synccheck): every kernel of the
engine runs at least once on the tiny presets — chunked prefill (wgmma attention), decode (per-item and
chunked + merge attention, split-K GEMMs and their consumers, fused arg-max), sampling, logits, prefix
pages — plus one launch of each unit-test hook.
usage: compute-sanitizer --tool memcheck python scripts/sanitize_probe.py"""
import ctypes
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from agentcontrolplane_b200 import _lib  # noqa: E402
from agentcontrolplane_b200.engine import Engine  # noqa: E402

rng = np.random.default_rng(7)
for model, mode in (("tiny", "item"), ("tiny-g8", "chunked"), ("tiny-moe", "chunked")):   # tiny-moe: router / dispatch / gather / grouped GEMMs / combine
    with Engine({"model": model, "max_batch": 8, "kv_pages": 96, "max_tokens_per_step": 128, "attn_decode_mode": mode}) as eng:
        prompts = [[128000] + [int(t) for t in rng.integers(0, 256, size=n)] for n in (5, 40, 150, 150, 300)]
        prompts[3] = prompts[2][:130] + prompts[3][130:]          # shares four prefix pages with prompt 2
        ts = [eng.submit({"model": model, "max_tokens": 4, "acp": {"prompt_token_ids": p, "return_logits": 1}}) for p in prompts]
        ts.append(eng.submit({"model": model, "max_tokens": 3, "temperature": 0.8, "top_k": 20, "top_p": 0.9, "seed": 3,
                              "acp": {"prompt_token_ids": prompts[1]}}))
        for t in ts:
            assert eng.wait(t, 600000)
            st, body = eng.result(t)
            assert st == 200, body
        print(model, mode, "ok", eng.stats()["kernel_launches"], "launches", flush=True)
lib = _lib.load()
u16p = ctypes.POINTER(ctypes.c_uint16)
bits = lambda shape: ((rng.standard_normal(shape).astype(np.float32).view(np.uint32) + 0x8000) >> 16).astype(np.uint16)
for heads, kvh, q_len, ctx in ((4, 1, 70, 200), (8, 1, 33, 33)):
    q, k, v = bits((q_len, heads, 128)), bits((ctx, kvh, 128)), bits((ctx, kvh, 128))
    out = np.zeros((q_len, heads, 128), np.uint16)
    ms = ctypes.c_float(0)
    lib.acp_kernel_attn_prefill.argtypes = [u16p, u16p, u16p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, u16p,
                                            ctypes.c_int, ctypes.POINTER(ctypes.c_float)]
    for impl in (1, 0):
        rc = lib.acp_kernel_attn_prefill(q.ctypes.data_as(u16p), k.ctypes.data_as(u16p), v.ctypes.data_as(u16p), heads, kvh, q_len, ctx,
                                         impl, out.ctypes.data_as(u16p), 0, ctypes.byref(ms))
        assert rc == 0, rc
# persistent and tiled prefill GEMM (two N tiles, ragged), both epilogues
f32p, i32p = ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_int)
for epi in (0, 3):
    w, x = bits((256, 128)), bits((300, 128))
    outs = []
    for mode in (-1, 256):
        out = np.zeros((300, 128 if epi == 3 else 256), np.uint16)
        rc = lib.acp_kernel_gemm(w.ctypes.data_as(u16p), x.ctypes.data_as(u16p), 256, 300, 128, 1, epi, mode,
                                 out.ctypes.data_as(ctypes.c_void_p), None, None, 0, ctypes.byref(ms))
        assert rc == 0, rc
        outs.append(out)
    assert np.array_equal(outs[0], outs[1])
print("hooks ok", flush=True)
