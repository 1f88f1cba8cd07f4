"""Times the wgmma GEMM at the Llama-3-8B decode shapes (N = 64 live sequences) for a sweep
of split-K factors; prints one JSON line per (GEMM, N, split).  Needs a GPU.  Dev tool only.

  python scripts/gemm_probe.py [N ...]"""
import ctypes
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from agentcontrolplane_b200 import _lib  # noqa: E402


def main():
    lib = _lib.load()
    u16p = ctypes.POINTER(ctypes.c_uint16)
    rng = np.random.default_rng(0)
    shapes = {
        "qkv": (6144, 4096, [1, 2, 3, 4, 6]),
        "o": (4096, 4096, [1, 2, 4, 5, 9]),
        "gate_up": (28672, 4096, [1, 2, 4, 5]),
        "down": (4096, 14336, [1, 4, 9, 14]),
        "lm_head": (128256, 4096, [1]),
    }
    Ns = [int(a) for a in sys.argv[1:]] or [64]
    for name, (M, K, splits_list) in shapes.items():
        w = rng.integers(0x3000, 0x3C00, size=(M, K), dtype=np.uint16)  # small positive bf16
        for N in Ns:
            x = rng.integers(0x3000, 0x3F80, size=(N, K), dtype=np.uint16)
            for s in splits_list:
                epi = 2 if name == "lm_head" else 1
                out = np.zeros((s, N, M), np.float32) if epi == 1 else None
                av = np.zeros(N, np.float32)
                ai = np.zeros(N, np.int32)
                ms = ctypes.c_float(0)
                rc = lib.acp_kernel_gemm(
                    w.ctypes.data_as(u16p), x.ctypes.data_as(u16p), M, N, K, s, epi, 0,
                    out.ctypes.data_as(ctypes.c_void_p) if out is not None else None,
                    av.ctypes.data_as(ctypes.POINTER(ctypes.c_float)),
                    ai.ctypes.data_as(ctypes.POINTER(ctypes.c_int)), 20, ctypes.byref(ms))
                gbs = (M * K * 2) / (ms.value * 1e-3) / 1e9 if ms.value > 0 else 0
                r = dict(gemm=name, M=M, K=K, N=N, splits=s, rc=rc, ms=ms.value, weight_GBps=gbs)
                print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
