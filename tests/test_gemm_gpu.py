"""wgmma GEMM (agentcontrolplane_b200/csrc/gemm_wgmma.cuh) vs a numpy fp32 matmul of the same
bf16 inputs, through the C-ABI test hook acp_kernel_gemm (include/acp_infer_kernels.h)."""
import ctypes

import numpy as np
import pytest

from agentcontrolplane_b200 import _lib
from oracle.bf16 import bf16_round_to_bits, bits_to_f32

pytestmark = pytest.mark.gpu


def _gemm(w_bits, x_bits, splits=1, epi=0, bn=0, want_logits=True, iters=0):
    lib = _lib.load()
    M, K = w_bits.shape
    N = x_bits.shape[0]
    u16p = ctypes.POINTER(ctypes.c_uint16)
    ms = ctypes.c_float(0)
    amax_v = np.zeros(N, np.float32)
    amax_i = np.zeros(N, np.int32)
    if epi == 0:
        out = np.zeros((N, M), np.uint16)
    elif epi == 3:
        out = np.zeros((N, M // 2), np.uint16)
    elif epi == 1:
        out = np.zeros((splits, N, M), np.float32)
    else:
        out = np.zeros((N, M), np.float32) if want_logits else None
    rc = lib.acp_kernel_gemm(
        w_bits.ctypes.data_as(u16p), x_bits.ctypes.data_as(u16p), M, N, K, splits, epi, bn,
        out.ctypes.data_as(ctypes.c_void_p) if out is not None else None,
        amax_v.ctypes.data_as(ctypes.POINTER(ctypes.c_float)),
        amax_i.ctypes.data_as(ctypes.POINTER(ctypes.c_int)), iters, ctypes.byref(ms))
    assert rc == 0, f"acp_kernel_gemm rc={rc}"
    return out, amax_v, amax_i, ms.value


def _rand_bits(rng, shape, scale):
    return bf16_round_to_bits((rng.standard_normal(shape) * scale).astype(np.float32))


@pytest.mark.parametrize("M,N,K,bn", [
    (128, 16, 64, 0), (256, 16, 128, 0), (384, 32, 256, 0), (256, 64, 512, 0),
    (512, 128, 256, 0), (256, 256, 192, 0), (256, 300, 128, 0),   # two N tiles, ragged
    (200, 20, 96, 0),                                              # ragged M, N, K
    (768, 5, 512, 0), (1024, 64, 4096, 0), (256, 7, 64, 64),
    (2560, 2600, 192, 0),   # prefill-sized: persistent kernel, 220 tiles > 132 CTAs (several tiles per CTA)
    (384, 1000, 4096, 0),   # persistent kernel, long K (ring wraps many times per tile)
])
def test_gemm_bf16_out(M, N, K, bn):
    rng = np.random.default_rng(M * 131 + N * 7 + K)
    w = _rand_bits(rng, (M, K), 0.05)
    x = _rand_bits(rng, (N, K), 1.0)
    out, _, _, _ = _gemm(w, x, epi=0, bn=bn)
    ref = bits_to_f32(x) @ bits_to_f32(w).T
    got = bits_to_f32(out)
    # fp32 accumulation order differs from numpy's: allow one bf16 ulp of the result
    tol = np.maximum(np.abs(ref) * 2.0 ** -7, 1e-3)
    assert np.all(np.abs(got - ref) <= tol), float(np.max(np.abs(got - ref)))


@pytest.mark.parametrize("M,N,K,splits", [(256, 16, 512, 2), (384, 64, 4096, 5), (128, 33, 1024, 16),
                                          (4096, 64, 4096, 9)])
def test_gemm_splitk_partials(M, N, K, splits):
    rng = np.random.default_rng(splits * 1000 + M)
    w = _rand_bits(rng, (M, K), 0.05)
    x = _rand_bits(rng, (N, K), 1.0)
    out, _, _, _ = _gemm(w, x, splits=splits, epi=1)
    ref = bits_to_f32(x) @ bits_to_f32(w).T
    got = out.sum(axis=0)
    assert np.allclose(got, ref, rtol=2e-4, atol=2e-4), float(np.max(np.abs(got - ref)))
    # each split covers its own k-block range exactly
    nkb = (K + 63) // 64
    for s in range(splits):
        k0, k1 = (nkb * s // splits) * 64, min(K, (nkb * (s + 1) // splits) * 64)
        part = bits_to_f32(x)[:, k0:k1] @ bits_to_f32(w)[:, k0:k1].T
        assert np.allclose(out[s], part, rtol=2e-4, atol=2e-4)


def test_gemm_argmax_epilogue():
    rng = np.random.default_rng(7)
    M, N, K = 128256, 24, 512   # LM-head rows of Llama-3 (1002 m-tiles)
    w = _rand_bits(rng, (M, K), 0.02)
    x = _rand_bits(rng, (N, K), 1.0)
    logits, av, ai, _ = _gemm(w, x, epi=2)
    ref = bits_to_f32(x) @ bits_to_f32(w).T
    assert np.allclose(logits, ref, rtol=2e-4, atol=2e-4)
    # arg-max must agree with the kernel's own logits exactly (lowest index on ties)
    assert np.array_equal(ai, np.argmax(logits, axis=1).astype(np.int32))
    assert np.array_equal(av, logits[np.arange(N), ai])
    _, av2, ai2, _ = _gemm(w, x, epi=2, want_logits=False)
    assert np.array_equal(ai2, ai) and np.array_equal(av2, av)


def test_gemm_argmax_tie_break():
    # identical rows of W give exactly equal logits: the lowest row index must win
    M, N, K = 512, 16, 64
    w = np.tile(bf16_round_to_bits(np.linspace(-1, 1, K, dtype=np.float32)), (M, 1))
    x = bf16_round_to_bits(np.ones((N, K), np.float32))
    _, _, ai, _ = _gemm(w, x, epi=2)
    assert np.all(ai == 0)


def test_gemm_deterministic():
    rng = np.random.default_rng(3)
    w = _rand_bits(rng, (1024, 2048), 0.05)
    x = _rand_bits(rng, (64, 2048), 1.0)
    a, _, _, _ = _gemm(w, x, splits=4, epi=1)
    b, _, _, _ = _gemm(w, x, splits=4, epi=1)
    assert np.array_equal(a, b)


@pytest.mark.parametrize("M,N,K", [(256, 16, 128), (2048, 64, 512), (512, 300, 256), (2048, 3000, 320)])
def test_gemm_fused_swiglu_epilogue(M, N, K):
    """epi 3: interleaved (gate_j, up_j) rows -> bf16(bf16(silu(g)) * u), the oracle's expression."""
    from oracle.bf16 import bf16_round
    rng = np.random.default_rng(M + N)
    w = _rand_bits(rng, (M, K), 0.08)
    x = _rand_bits(rng, (N, K), 1.0)
    out, _, _, _ = _gemm(w, x, epi=3)
    gu = bf16_round(bits_to_f32(x) @ bits_to_f32(w).T)
    g, u = gu[:, 0::2], gu[:, 1::2]
    ref = bf16_round(bf16_round(g / (np.float32(1.0) + np.exp(-g))) * u)
    got = bits_to_f32(out)
    # three bf16 roundings are chained (g, u; silu(g); product): a 1e-6 difference in the fp32
    # accumulation can flip each of them by one ulp, so the bound is ~3 ulp (2^-7 each) ...
    err = np.abs(got - ref)
    tol = np.maximum(np.abs(ref) * 2.0 ** -5, 4e-3)
    assert np.all(err <= tol), float(np.max(err / np.maximum(np.abs(ref), 1e-3)))
    # ... but almost every element must agree to one ulp
    assert np.mean(err <= np.maximum(np.abs(ref) * 2.0 ** -7, 1e-3)) > 0.995


# ---- persistent prefill kernel (gemm_wgmma.cuh gemm_wx_persistent_kernel) vs the tiled kernel ----------------
# Same fp32 accumulation order (K in order, one accumulator per output element), so the two must agree BIT FOR
# BIT; the tiled kernel is the one test_gemm_bf16_out pins against numpy.
@pytest.mark.parametrize("M,N,K,epi", [
    (256, 300, 128, 0),       # two N tiles (ragged: the second has 44 valid rows)
    (256, 1000, 4096, 0),     # long K: the ring wraps many times per tile
    (2560, 2600, 192, 0),     # 20 m-tiles x 11 N tiles = 220 tiles > 132 CTAs: tile loop
    (4096, 8192, 4096, 0),    # Llama-3-8B wo at an 8192-token chunk
    (2048, 3000, 320, 3),     # fused SwiGLU epilogue
    (3584, 4096, 512, 3),
])
def test_gemm_persistent_matches_tiled(M, N, K, epi):
    rng = np.random.default_rng(M + 3 * N + K + epi)
    w = _rand_bits(rng, (M, K), 0.05)
    x = _rand_bits(rng, (N, K), 1.0)
    tiled, _, _, _ = _gemm(w, x, epi=epi, bn=256)
    pers, _, _, _ = _gemm(w, x, epi=epi, bn=-1)
    assert np.array_equal(tiled, pers), int(np.count_nonzero(tiled != pers))
    if epi == 0 and M * N <= 2560 * 2600:
        ref = bits_to_f32(x) @ bits_to_f32(w).T
        got = bits_to_f32(pers)
        assert np.all(np.abs(got - ref) <= np.maximum(np.abs(ref) * 2.0 ** -7, 1e-3))
    if epi == 3:
        # the SwiGLU epilogue both kernels share, against numpy (bounds of test_gemm_fused_swiglu_epilogue)
        from oracle.bf16 import bf16_round
        gu = bf16_round(bits_to_f32(x) @ bits_to_f32(w).T)
        g, u = gu[:, 0::2], gu[:, 1::2]
        ref = bf16_round(bf16_round(g / (np.float32(1.0) + np.exp(-g))) * u)
        err = np.abs(bits_to_f32(pers) - ref)
        assert np.all(err <= np.maximum(np.abs(ref) * 2.0 ** -5, 4e-3)), float(np.max(err))
        assert np.mean(err <= np.maximum(np.abs(ref) * 2.0 ** -7, 1e-3)) > 0.995


def test_gemm_persistent_repeatable():
    rng = np.random.default_rng(11)
    w = _rand_bits(rng, (1024, 1024), 0.05)
    x = _rand_bits(rng, (5000, 1024), 1.0)
    a, _, _, _ = _gemm(w, x, epi=0, bn=-1)
    for _ in range(3):
        b, _, _, _ = _gemm(w, x, epi=0, bn=-1)
        assert np.array_equal(a, b)


@pytest.mark.parametrize("M,N,K,mode", [(8192, 4096, 1024, 0), (8192, 4096, 1024, -1), (1024, 700, 3584, 0), (384, 1000, 256, 0)])
def test_gemm_persistent_fp32_plane_matches_tiled_kernel(M, N, K, mode):
    """epi 1 with ONE plane and more than 256 rows (the row-parallel O / down projections of a tensor-parallel
    prefill step) runs on the persistent kernels; the tiled kernel (bn = 256 forces it) is the reference: same
    accumulation order, so the fp32 planes must be bit-identical."""
    rng = np.random.default_rng(M + N + K)
    w = _rand_bits(rng, (M, K), 0.05)
    x = _rand_bits(rng, (N, K), 1.0)
    tiled, _, _, _ = _gemm(w, x, splits=1, epi=1, bn=256)
    pers, _, _, _ = _gemm(w, x, splits=1, epi=1, bn=mode)
    assert np.array_equal(tiled, pers), int(np.count_nonzero(tiled != pers))
    ref = bits_to_f32(x) @ bits_to_f32(w).T
    assert np.allclose(pers[0], ref, rtol=2e-4, atol=2e-4)
