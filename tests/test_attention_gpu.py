"""Prefill attention kernels (agentcontrolplane_b200/csrc/attention_prefill_tc.cu — wgmma — and round 1's
mma.sync kernel) vs a numpy fp32 causal softmax attention, through the C-ABI test hook
acp_kernel_attn_prefill (include/acp_infer_kernels.h): paged K/V with a shuffled page table, GQA group
sizes 1..16, ragged lengths, chunk offsets (the query block starts in the middle of the context)."""
import ctypes

import numpy as np
import pytest

from agentcontrolplane_b200 import _lib
from oracle.bf16 import bf16_round_to_bits, bits_to_f32

pytestmark = pytest.mark.gpu


def _attn(q_bits, k_bits, v_bits, impl=1, iters=0):
    lib = _lib.load()
    q_len, heads, _ = q_bits.shape
    ctx, kv_heads, _ = k_bits.shape
    u16p = ctypes.POINTER(ctypes.c_uint16)
    out = np.zeros((q_len, heads, 128), np.uint16)
    ms = ctypes.c_float(0)
    lib.acp_kernel_attn_prefill.argtypes = [u16p, u16p, u16p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                            ctypes.c_int, u16p, ctypes.c_int, ctypes.POINTER(ctypes.c_float)]
    rc = lib.acp_kernel_attn_prefill(q_bits.ctypes.data_as(u16p), k_bits.ctypes.data_as(u16p), v_bits.ctypes.data_as(u16p),
                                     heads, kv_heads, q_len, ctx, impl, out.ctypes.data_as(u16p), iters, ctypes.byref(ms))
    assert rc == 0, f"acp_kernel_attn_prefill rc={rc}"
    return out, ms.value


def _reference(q, k, v):
    """fp32 causal attention; q [q_len][H][128], k/v [ctx][KVH][128]; query i at position ctx - q_len + i"""
    q_len, H, d = q.shape
    ctx, KVH, _ = k.shape
    G = H // KVH
    pos = np.arange(ctx - q_len, ctx)
    mask = np.arange(ctx)[None, :] <= pos[:, None]
    out = np.empty((q_len, H, d), np.float32)
    scale = np.float32(1.0 / np.sqrt(d))
    for h in range(H):
        s = (q[:, h, :] @ k[:, h // G, :].T) * scale
        s = np.where(mask, s, -np.inf)
        p = np.exp(s - s.max(axis=-1, keepdims=True))
        out[:, h, :] = (p @ v[:, h // G, :]) / p.sum(axis=-1, keepdims=True)
    return out


def _case(rng, heads, kv_heads, q_len, ctx, qscale=1.0):
    q = bf16_round_to_bits((rng.standard_normal((q_len, heads, 128)) * qscale).astype(np.float32))
    k = bf16_round_to_bits(rng.standard_normal((ctx, kv_heads, 128)).astype(np.float32))
    v = bf16_round_to_bits(rng.standard_normal((ctx, kv_heads, 128)).astype(np.float32))
    return q, k, v


CASES = [
    (4, 1, 1, 1), (4, 1, 5, 5), (4, 1, 32, 32), (4, 1, 33, 33), (4, 1, 100, 100), (4, 2, 64, 64), (4, 2, 129, 300),
    (8, 1, 77, 300), (8, 1, 16, 16), (2, 2, 200, 200), (16, 1, 40, 90), (2, 1, 130, 130),
    (32, 8, 512, 512),          # Llama-3-8B heads, config 1's window
    (32, 8, 300, 1324),         # a later prefill chunk of a long window
    (8, 1, 600, 2500),          # Llama-3-70B TP=8 shard shape, long context
]


@pytest.mark.parametrize("impl", [1, 0])
@pytest.mark.parametrize("heads,kv_heads,q_len,ctx", CASES)
def test_prefill_attention_matches_fp32_reference(impl, heads, kv_heads, q_len, ctx):
    rng = np.random.default_rng(heads * 1000003 + q_len * 131 + ctx)
    q, k, v = _case(rng, heads, kv_heads, q_len, ctx)
    out, _ = _attn(q, k, v, impl=impl)
    ref = _reference(bits_to_f32(q), bits_to_f32(k), bits_to_f32(v))
    got = bits_to_f32(out)
    assert np.isfinite(got).all()
    # P is carried as bf16 hi + lo (~fp32): what is left is the final bf16 rounding of the output
    tol = np.maximum(np.abs(ref) * 2.0 ** -7, 2e-3)
    bad = np.abs(got - ref) > tol
    assert not bad.any(), (int(bad.sum()), float(np.max(np.abs(got - ref))), np.argwhere(bad)[:5].tolist())


def test_lazy_rescale_with_growing_scores():
    """Scores that keep growing along the context force the running max (and the lazy O rescale of
    the wgmma kernel) to move many times; large |q| makes the softmax peaky."""
    rng = np.random.default_rng(99)
    q, k, v = _case(rng, 4, 1, 96, 700, qscale=3.0)
    kf = bits_to_f32(k)
    kf *= np.linspace(0.2, 2.5, 700, dtype=np.float32)[:, None, None]
    k = bf16_round_to_bits(kf)
    out, _ = _attn(q, k, v, impl=1)
    ref = _reference(bits_to_f32(q), bits_to_f32(k), bits_to_f32(v))
    got = bits_to_f32(out)
    tol = np.maximum(np.abs(ref) * 2.0 ** -7, 2e-3)
    assert np.all(np.abs(got - ref) <= tol), float(np.max(np.abs(got - ref)))


def test_tc_kernel_is_deterministic_and_chunk_invariant():
    """The same query rows computed as one chunk or as the tail chunk of a longer prefill give the
    same bits (absolute key-tile boundaries), run to run."""
    rng = np.random.default_rng(7)
    q, k, v = _case(rng, 8, 2, 400, 400)
    full, _ = _attn(q, k, v, impl=1)
    again, _ = _attn(q, k, v, impl=1)
    assert np.array_equal(full, again)
    tail, _ = _attn(q[250:], k, v, impl=1)       # queries 250..399 as their own chunk over the same 400 keys
    assert np.array_equal(full[250:], tail)


def test_prefill_attention_speed_at_4096():
    """Not a bench value: prints the TFLOP/s of one 8-KV-head layer step at T = 4096 for the profile notes."""
    rng = np.random.default_rng(1)
    q, k, v = _case(rng, 32, 8, 4096, 4096)
    for impl in (1, 0):
        _, ms = _attn(q, k, v, impl=impl, iters=5)
        flops = 4.0 * 32 * 128 * (4096 * 4097 / 2)
        print(f"attn_prefill impl={impl}: T=4096 {ms * 1e3:.1f} us  {flops / ms / 1e9:.1f} TFLOP/s (causal FLOPs)")
