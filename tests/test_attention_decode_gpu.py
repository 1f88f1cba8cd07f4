"""Decode attention kernels (agentcontrolplane_b200/csrc/attention.cu: attn_decode_item_kernel, attn_decode_kernel +
attn_merge_kernel, and the fused RoPE + K/V append of new_token_prologue) against the float64 reference of
oracle/attention_oracle.py, through the hook acp_kernel_attn_decode (include/acp_infer_kernels.h).

Contexts sit on page (32), tile (64) and chunk (1024) boundaries; 1025 leaves the last chunk only the new token,
9000 sends the merge through its tail loop and 131072 makes it combine 512 partials.  Every sequence carries one
planted key, so a dropped or misplaced key, page, tile or chunk moves the output by ~4, and the new token is planted
too.  Stale cache bytes (NaN, +Inf) in the slots no sequence owns must not change a bit."""
import ctypes

import numpy as np
import pytest

from agentcontrolplane_b200 import _lib
from oracle import attention_oracle as ao
from oracle.bf16 import bf16_round, bf16_round_to_bits, bits_to_f32
from oracle.llama_oracle import PRESETS, rope_tables
from llama31_presets import LLAMA31

pytestmark = pytest.mark.gpu

GQA = [(32, 8), (64, 8), (8, 1), (16, 1), (4, 4)]
CTXS = [1, 2, 31, 32, 33, 64, 65, 1023, 1024, 1025, 1026, 2049, 9000]
PLANTED = [0, 31, 32, 63, 64, 1023, 1024]
STALE = [0x0000, 0xFFFF, 0x7F80]
MAX_POS = 9000
_TABLES = {}


def _tables(max_pos, long_rope=False):
    key = (max_pos, long_rope)
    if key not in _TABLES:
        cfg = LLAMA31["tiny-3.1"] if long_rope else PRESETS["tiny"]
        _TABLES[key] = tuple(np.ascontiguousarray(t) for t in rope_tables(cfg, max_pos))
    return _TABLES[key]


def _hook(k, v, qkv_planes, splits, ctx, heads, kv_heads, mode, stale, cos, sin):
    """qkv_planes: [B][ld] bf16 values (splits 0) or [splits][B][ld] fp32"""
    lib = _lib.load()
    B = len(ctx)
    u16p, f32p, i32p = (ctypes.POINTER(t) for t in (ctypes.c_uint16, ctypes.c_float, ctypes.c_int))
    lib.acp_kernel_attn_decode.argtypes = [u16p, u16p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, f32p, f32p,
                                           ctypes.c_int, ctypes.c_int, i32p, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                           ctypes.c_uint16, u16p, u16p, u16p]
    qkv = bf16_round_to_bits(qkv_planes) if splits == 0 else np.ascontiguousarray(qkv_planes, np.float32)
    kb = np.ascontiguousarray(bf16_round_to_bits(k))
    vb = np.ascontiguousarray(bf16_round_to_bits(v))
    ctx_a = np.asarray(ctx, np.int32)
    out = np.zeros((B, heads, 128), np.uint16)
    k_new = np.zeros((B, kv_heads, 128), np.uint16)
    v_new = np.zeros_like(k_new)
    rc = lib.acp_kernel_attn_decode(kb.ctypes.data_as(u16p), vb.ctypes.data_as(u16p), qkv.ctypes.data, splits, B + 3,
                                    cos.ctypes.data_as(f32p), sin.ctypes.data_as(f32p), cos.shape[0], B,
                                    ctx_a.ctypes.data_as(i32p), heads, kv_heads, mode, stale,
                                    out.ctypes.data_as(u16p), k_new.ctypes.data_as(u16p), v_new.ctypes.data_as(u16p))
    assert rc == 0, f"acp_kernel_attn_decode rc={rc}"
    return out, k_new, v_new


class Step:
    """B decode sequences: cached K/V (post-RoPE, positions 0..ctx-2), the QKV row of each new token and the
    float64 reference; sequence b carries a planted key at planted[b] (ctx-1 = the new token)."""

    def __init__(self, heads, kv_heads, ctx, planted, seed, long_rope=False):
        rng = np.random.default_rng(seed)
        self.heads, self.kv_heads, self.ctx, self.planted = heads, kv_heads, list(ctx), list(planted)
        self.cos, self.sin = _tables(max(MAX_POS, max(ctx)), long_rope)
        qd, kvd = heads * 128, kv_heads * 128
        self.rows, self.k, self.v, self.ref, self.A = [], [], [], [], []
        for n, j in zip(self.ctx, self.planted):
            c, s = self.cos[n - 1], self.sin[n - 1]
            row = bf16_round(rng.standard_normal(qd + 2 * kvd).astype(np.float32))
            q = ao.rope(row[:qd].reshape(heads, 128), c, s)
            k = bf16_round(rng.standard_normal((n, kv_heads, 128)).astype(np.float32))
            v = bf16_round(rng.standard_normal((n, kv_heads, 128)).astype(np.float32))
            k[n - 1] = ao.rope(row[qd:qd + kvd].reshape(kv_heads, 128), c, s)
            v[n - 1] = row[qd + kvd:].reshape(kv_heads, 128)
            if n > 1:   # a lone new token holds all the mass: nothing to plant
                k, v = ao.plant_decode_key(q, k, v, j)
                if j == n - 1:   # the new token: its K/V come from the QKV row (K before RoPE)
                    row[qd:qd + kvd] = ao.unrope(k[n - 1], c, s).reshape(-1)
                    row[qd + kvd:] = v[n - 1].reshape(-1)
                    k[n - 1] = ao.rope(row[qd:qd + kvd].reshape(kv_heads, 128), c, s)
            ref, A = ao.attention(q[None], k, v, [n])
            if n > 1:
                ao.check_decode_canary(q, k, v, j, ref[0])
            self.rows.append(row)
            self.k.append(k)
            self.v.append(v)
            self.ref.append(ref[0])
            self.A.append(A[0])

    def run(self, splits=0, mode=0, stale=0, seed=0, only=None):
        idx = list(range(len(self.ctx))) if only is None else list(only)
        rows = np.stack([self.rows[i] for i in idx])
        planes = rows if splits == 0 else ao.split_exact(rows, splits, np.random.default_rng(seed))
        k = np.concatenate([self.k[i][:-1] for i in idx]).reshape(-1, self.kv_heads, 128)
        v = np.concatenate([self.v[i][:-1] for i in idx]).reshape(-1, self.kv_heads, 128)
        return _hook(k, v, planes, splits, [self.ctx[i] for i in idx], self.heads, self.kv_heads, mode, stale,
                     self.cos, self.sin)

    def check(self, res, what, only=None):
        out, k_new, v_new = res
        idx = list(range(len(self.ctx))) if only is None else list(only)
        worst = -np.inf
        for r, i in enumerate(idx):
            n = self.ctx[i]
            tag = (what, self.heads, self.kv_heads, n, self.planted[i])
            assert np.array_equal(bits_to_f32(k_new[r]), self.k[i][n - 1]), ("appended K", tag)
            assert np.array_equal(bits_to_f32(v_new[r]), self.v[i][n - 1]), ("appended V", tag)
            worst = max(worst, ao.assert_within(bits_to_f32(out[r]), self.ref[i], self.A[i], tag))
        return worst


def _planted(n):
    keys = PLANTED if n <= 4096 else [0, 1024]    # keeps the mixed batch's host arrays small
    return sorted({j for j in keys + [n - 2] if 0 <= j < n - 1} | {n - 1})


def _mixed_step(heads, kv_heads, seed=1):
    ctx = [n for n in CTXS for _ in _planted(n)]
    planted = [j for n in CTXS for j in _planted(n)]
    return Step(heads, kv_heads, ctx, planted, seed)


_STEPS = {}


def _step(heads, kv_heads):
    if (heads, kv_heads) not in _STEPS:
        _STEPS.clear()
        _STEPS[(heads, kv_heads)] = _mixed_step(heads, kv_heads)
    return _STEPS[(heads, kv_heads)]


@pytest.mark.parametrize("heads,kv_heads,splits", [(h, kvh, s) for h, kvh in GQA for s in (0, 1, 9)])
def test_decode_matches_float64_reference(heads, kv_heads, splits):
    """every context x every planted key in one mixed batch (chunked kernel + merge): output within the
    tolerance, appended K/V bit-exact"""
    st = _step(heads, kv_heads)
    worst = st.check(st.run(splits=splits, seed=splits), f"splits={splits}")
    print(f"decode G={heads // kv_heads} ({heads},{kv_heads}) splits={splits}: worst (|got-ref| - 2^-8|ref|)/A = "
          f"{worst:.3g} (bound {ao.ABS_A:.3g})")


@pytest.mark.parametrize("heads,kv_heads", GQA)
def test_item_and_chunked_kernels_are_bit_identical(heads, kv_heads):
    """contexts <= 1024 are one chunk: the per-item kernel and chunked + merge do the same arithmetic in the same
    order (model.cu picks either), so the bits agree"""
    st = _step(heads, kv_heads)
    short = [i for i, n in enumerate(st.ctx) if n <= 1024]
    item = st.run(mode=1, only=short)
    chunked = st.run(mode=2, only=short)
    st.check(item, "item", only=short)
    for a, b in zip(item, chunked):
        assert np.array_equal(a, b)


@pytest.mark.parametrize("heads,kv_heads", GQA)
def test_stale_cache_bytes_do_not_change_a_bit(heads, kv_heads):
    """NaN and +Inf patterns in every cache slot no sequence owns (page tails, spare pages, the new token's slot
    before the append) give the bits of a zeroed cache"""
    st = _step(heads, kv_heads)
    base = st.run(splits=1, stale=STALE[0])
    for stale in STALE[1:]:
        got = st.run(splits=1, stale=stale)
        for a, b in zip(base, got):
            assert np.array_equal(a, b), hex(stale)


@pytest.mark.parametrize("heads,kv_heads,splits", [(32, 8, 0), (8, 1, 9)])
def test_decode_is_batch_invariant(heads, kv_heads, splits):
    """each sequence gives the same bits alone as in the mixed batch of every length (chunk boundaries depend only
    on the sequence itself)"""
    st = _step(heads, kv_heads)
    batch = st.run(splits=splits, seed=3)
    for i in range(len(st.ctx)):
        if st.planted[i] != st.ctx[i] - 1:
            continue
        alone = st.run(splits=splits, seed=3, only=[i])
        # the split-K planes differ with the batch's rows, but they sum exactly to the same bf16 row
        for a, b in zip(batch, alone):
            assert np.array_equal(a[i], b[0]), st.ctx[i]


@pytest.mark.parametrize("heads,kv_heads", [(8, 1), (16, 1)])
def test_decode_at_131072_tokens(heads, kv_heads):
    """a 128K context: the merge combines 512 partials per head, RoPE at position 131071 on Llama-3.1's scaled
    tables; planted keys at the first key, a chunk boundary, the last cached key and the new token"""
    n = 131072
    planted = [0, 1024, n - 2, n - 1]
    st = Step(heads, kv_heads, [n] * len(planted), planted, seed=131072, long_rope=True)
    for splits in (0, 9):
        worst = st.check(st.run(splits=splits, seed=splits), f"131072 splits={splits}")
        print(f"decode 131072 G={heads // kv_heads} splits={splits}: worst (|got-ref| - 2^-8|ref|)/A = {worst:.3g}")


def test_per_item_mode_rejects_a_multi_chunk_context():
    st = Step(4, 4, [1025], [1024], seed=5)
    with pytest.raises(AssertionError, match="rc=-1"):
        st.run(mode=1)
