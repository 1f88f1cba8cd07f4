"""Prefill attention kernels (agentcontrolplane_b200/csrc/attention_prefill_tc.cu — wgmma — and round 1's
mma.sync kernel) vs the float64 causal attention and tolerance of oracle/attention_oracle.py, through the C-ABI
test hooks acp_kernel_attn_prefill / acp_kernel_attn_prefill_batch (include/acp_infer_kernels.h): paged K/V with a
shuffled page table, GQA group sizes 1..16, ragged lengths, chunk offsets (the query block starts in the middle of
the context), steps that pack several sequences, planted keys on and one past the diagonal, and stale bytes
(NaN, +Inf) in the cache slots no sequence owns."""
import ctypes

import numpy as np
import pytest

from agentcontrolplane_b200 import _lib
from oracle import attention_oracle as ao
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


def _attn_batch(qs, ks, vs, heads, kv_heads, impl=1, stale=0):
    """one prefill step of len(qs) sequences: qs[b] bf16 bits [q_len][heads][128], ks/vs[b] [ctx][kv_heads][128]"""
    lib = _lib.load()
    u16p, i32p = ctypes.POINTER(ctypes.c_uint16), ctypes.POINTER(ctypes.c_int)
    q_len = np.array([q.shape[0] for q in qs], np.int32)
    ctx = np.array([k.shape[0] for k in ks], np.int32)
    q, k, v = (np.ascontiguousarray(np.concatenate(x)) for x in (qs, ks, vs))
    out = np.zeros((int(q_len.sum()), heads, 128), np.uint16)
    lib.acp_kernel_attn_prefill_batch.argtypes = [u16p, u16p, u16p, ctypes.c_int, ctypes.c_int, ctypes.c_int, i32p,
                                                  i32p, ctypes.c_uint16, ctypes.c_int, u16p, ctypes.c_int,
                                                  ctypes.POINTER(ctypes.c_float)]
    rc = lib.acp_kernel_attn_prefill_batch(q.ctypes.data_as(u16p), k.ctypes.data_as(u16p), v.ctypes.data_as(u16p),
                                           heads, kv_heads, len(qs), q_len.ctypes.data_as(i32p),
                                           ctx.ctypes.data_as(i32p), stale, impl, out.ctypes.data_as(u16p), 0, None)
    assert rc == 0, f"acp_kernel_attn_prefill_batch rc={rc}"
    return np.split(out, np.cumsum(q_len)[:-1])


def _reference(q, k, v):
    """float64 causal attention; q [q_len][H][128], k/v [ctx][KVH][128]; query i at position ctx - q_len + i"""
    return ao.attention(q, k, v, np.arange(k.shape[0] - q.shape[0], k.shape[0]) + 1)


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
    ref, A = _reference(bits_to_f32(q), bits_to_f32(k), bits_to_f32(v))
    # P is carried as bf16 hi + lo (~fp32): what is left is the final bf16 rounding of the output
    worst = ao.assert_within(bits_to_f32(out), ref, A)
    print(f"prefill impl={impl} ({heads},{kv_heads}) q_len={q_len} ctx={ctx}: worst (|got-ref| - 2^-8|ref|)/A = {worst:.3g}")


def test_lazy_rescale_with_growing_scores():
    """Scores that keep growing along the context force the running max (and the lazy O rescale of
    the wgmma kernel) to move many times; large |q| makes the softmax peaky."""
    rng = np.random.default_rng(99)
    q, k, v = _case(rng, 4, 1, 96, 700, qscale=3.0)
    kf = bits_to_f32(k)
    kf *= np.linspace(0.2, 2.5, 700, dtype=np.float32)[:, None, None]
    k = bf16_round_to_bits(kf)
    out, _ = _attn(q, k, v, impl=1)
    ref, A = _reference(bits_to_f32(q), bits_to_f32(k), bits_to_f32(v))
    worst = ao.assert_within(bits_to_f32(out), ref, A)
    print(f"prefill lazy rescale: worst (|got-ref| - 2^-8|ref|)/A = {worst:.3g}")


# (q_len, ctx, planted keys) of the sequences of one step: q_len not a multiple of the block's tokens, page and
# 64-key tile boundaries, keys on a query's diagonal whose previous row sees them one position in its future
STEP = [(1, 1, []), (5, 300, [63, 64, 296, 299]), (200, 200, [1, 31, 32, 64, 150]), (129, 1500, [64, 1024, 1372, 1499]),
        (64, 64, [1, 63])]


def _step(rng, heads, kv_heads):
    qs, ks, vs, refs = [], [], [], []
    for q_len, ctx, keys in STEP:
        q, k, v = (bits_to_f32(x) for x in _case(rng, heads, kv_heads, q_len, ctx))
        pos = np.arange(ctx - q_len, ctx)
        if keys:
            q, k, v = ao.plant_prefill_keys(q, pos, k, v, keys)
        ref, A = ao.attention(q, k, v, pos + 1)
        ao.check_prefill_canaries(q, pos, k, v, keys, ref)
        qs.append(bf16_round_to_bits(q)); ks.append(bf16_round_to_bits(k)); vs.append(bf16_round_to_bits(v))
        refs.append((ref, A))
    return qs, ks, vs, refs


@pytest.mark.parametrize("impl", [1, 0])
@pytest.mark.parametrize("heads,kv_heads", [(32, 8), (8, 1), (4, 4)])
def test_batched_prefill_step_with_planted_keys_and_stale_pages(impl, heads, kv_heads):
    """Several sequences in one step (non-zero q_start and page offsets; a sequence's last Q box reads the next
    sequence's rows), planted keys on and one past the diagonal; the output must not change a bit when the slots
    no sequence owns hold NaN or +Inf instead of zeros (masked P is exactly 0, and 0 * NaN must never happen)."""
    rng = np.random.default_rng(heads * 7 + kv_heads + impl)
    qs, ks, vs, refs = _step(rng, heads, kv_heads)
    base = _attn_batch(qs, ks, vs, heads, kv_heads, impl=impl)
    worst = -np.inf
    for (q_len, ctx, _), out, (ref, A) in zip(STEP, base, refs):
        worst = max(worst, ao.assert_within(bits_to_f32(out), ref, A, (impl, heads, kv_heads, q_len, ctx)))
    print(f"prefill step impl={impl} ({heads},{kv_heads}): worst (|got-ref| - 2^-8|ref|)/A = {worst:.3g}")
    for stale in (0xFFFF, 0x7F80):
        got = _attn_batch(qs, ks, vs, heads, kv_heads, impl=impl, stale=stale)
        for (q_len, ctx, _), a, b in zip(STEP, base, got):
            assert np.array_equal(a, b), (hex(stale), q_len, ctx)


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
