"""Times the wgmma GEMM through the C-ABI hook acp_kernel_gemm (CUDA events, L2 flushed before every launch).
Needs a GPU.  Dev tool only.

  python scripts/gemm_probe.py [N ...]      decode shapes (default N = 64 live sequences), a sweep of split-K
                                            factors; one JSON line per (GEMM, N, split)
  python scripts/gemm_probe.py prefill      the persistent prefill kernel at the Llama-3-8B layer shapes with
                                            N = 4096 tokens, then a K sweep at M = N = 4096 (see prefill())"""
import ctypes
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from agentcontrolplane_b200 import _lib  # noqa: E402

U16P = ctypes.POINTER(ctypes.c_uint16)
BF16_PEAK_TFLOPS = 989.0         # H100 SXM data sheet, dense bf16, at up to 700 W
FLOP_PER_CLK_SM = 4096           # dense bf16 wgmma rate of one H100 SM
SMS = 132


def _time_gemm(lib, w, x, epi, iters):
    M, K = w.shape
    N = x.shape[0]
    out = np.zeros((N, M // 2 if epi == 3 else M), np.uint16)
    av = np.zeros(N, np.float32)
    ai = np.zeros(N, np.int32)
    ms = ctypes.c_float(0)
    rc = lib.acp_kernel_gemm(w.ctypes.data_as(U16P), x.ctypes.data_as(U16P), M, N, K, 1, epi, 0,
                             out.ctypes.data_as(ctypes.c_void_p), av.ctypes.data_as(ctypes.POINTER(ctypes.c_float)),
                             ai.ctypes.data_as(ctypes.POINTER(ctypes.c_int)), iters, ctypes.byref(ms))
    assert rc == 0, f"acp_kernel_gemm rc={rc}"
    return ms.value


def prefill(lib):
    """Kernel time of the four layer GEMMs of one Llama-3-8B prefill chunk (N = 4096 tokens, bf16 out or fused
    SwiGLU), as TFLOP/s and as a fraction of the dense bf16 ceiling 132 SMs x 4096 FLOP/clk x clock.  The clock
    is SM_MHZ from the environment, else the card's maximum SM clock: the timed launches are milliseconds apart
    from each other (host-side set-up in between), too short for nvidia-smi's sampling to see their clock.
    Then one shape (M = N = 4096) over K: kernel time is linear in K, the slope is the mainloop rate (reported
    per SM per clock, against 4096) and the intercept the fixed cost of a tile (epilogue, ring fill, launch),
    reported per tile of the busiest CTA."""
    import subprocess
    rng = np.random.default_rng(0)
    iters = int(os.environ.get("ITERS", "10"))
    N = 4096
    shapes = [("qkv", 6144, 4096, 0), ("o", 4096, 4096, 0), ("gate_up", 28672, 4096, 3), ("down", 4096, 14336, 0)]
    x_full = rng.integers(0x3000, 0x3F80, size=(N, 14336), dtype=np.uint16)
    rows = []
    for name, M, K, epi in shapes:
        w = rng.integers(0x3000, 0x3C00, size=(M, K), dtype=np.uint16)   # small positive bf16
        ms = _time_gemm(lib, w, np.ascontiguousarray(x_full[:, :K]), epi, iters)
        rows.append(dict(gemm=name, M=M, N=N, K=K, epi=epi, ms=ms, tflops=2.0 * M * N * K / (ms * 1e-3) / 1e12))
    M = 4096
    w_full = rng.integers(0x3000, 0x3C00, size=(M, 14336), dtype=np.uint16)
    sweep = []
    for K in (1024, 2048, 4096, 8192, 14336):
        ms = _time_gemm(lib, np.ascontiguousarray(w_full[:, :K]), np.ascontiguousarray(x_full[:, :K]), 0, iters)
        sweep.append((K, ms))
    smi = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                         capture_output=True, text=True).stdout.strip().split(", ")
    mhz = float(os.environ.get("SM_MHZ") or smi[2])
    ceil_tflops = SMS * FLOP_PER_CLK_SM * mhz * 1e6 / 1e12
    for r in rows:
        r.update(frac_of_989=r["tflops"] / BF16_PEAK_TFLOPS, frac_of_clock_ceiling=r["tflops"] / ceil_tflops)
        print(json.dumps(r), flush=True)
    ks = np.array([k for k, _ in sweep], np.float64)
    ts = np.array([t for _, t in sweep], np.float64)
    slope, icpt = np.polyfit(ks, ts, 1)
    tiles = (M // 128) * (N // 256)
    waves = -(-tiles // SMS)                 # tiles the busiest CTA runs, one after the other
    per_clk = waves * 2.0 * 128 * 256 / (slope * 1e-3) / (mhz * 1e6)
    tile_k4096_ms = slope * 4096 / waves
    for K, t in sweep:
        print(json.dumps(dict(sweep="K", M=M, N=N, K=int(K), ms=t, tflops=2.0 * M * N * K / (t * 1e-3) / 1e12)), flush=True)
    print(json.dumps(dict(
        fit="ms = intercept + slope * K", M=M, N=N, tiles=tiles, tiles_per_cta=waves, slope_ms_per_k=slope,
        intercept_ms=icpt, mainloop_flop_per_clk_per_sm=per_clk, mainloop_frac_of_4096=per_clk / FLOP_PER_CLK_SM,
        fixed_us_per_tile=icpt * 1e3 / waves, fixed_frac_of_k4096_tile=(icpt / waves) / tile_k4096_ms,
        gpu=smi[0], power_limit_w=float(smi[1]), sm_mhz=mhz, ceiling_tflops=ceil_tflops)), flush=True)
    if hasattr(lib, "acp_kernel_gemm_persistent_clusters"):
        print(json.dumps(dict(persistent_clusters={f"{'fp8' if fp8 else 'bf16'}_epi{epi}": lib.acp_kernel_gemm_persistent_clusters(fp8, epi)
                                                   for fp8 in (0, 1) for epi in (0, 1, 3)})), flush=True)


def main():
    lib = _lib.load()
    if sys.argv[1:2] == ["prefill"]:
        prefill(lib)
        return
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
                    w.ctypes.data_as(U16P), x.ctypes.data_as(U16P), M, N, K, s, epi, 0,
                    out.ctypes.data_as(ctypes.c_void_p) if out is not None else None,
                    av.ctypes.data_as(ctypes.POINTER(ctypes.c_float)),
                    ai.ctypes.data_as(ctypes.POINTER(ctypes.c_int)), 20, ctypes.byref(ms))
                gbs = (M * K * 2) / (ms.value * 1e-3) / 1e9 if ms.value > 0 else 0
                r = dict(gemm=name, M=M, K=K, N=N, splits=s, rc=rc, ms=ms.value, weight_GBps=gbs)
                print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
