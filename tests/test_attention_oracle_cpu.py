"""The attention tolerance of oracle/attention_oracle.py discriminates (no GPU): the true float64 reference rounded
to bf16 passes it, and each mutant of the reference -- the kind of mistake a paged, tiled, chunked attention
kernel makes -- violates it somewhere on the same data."""
import numpy as np
import pytest

from oracle import attention_oracle as ao
from oracle.bf16 import bf16_round
from oracle.llama_oracle import PRESETS, rope_tables


def _rand(rng, *shape):
    return bf16_round(rng.standard_normal(shape).astype(np.float32))


@pytest.fixture(scope="module")
def prefill():
    """4 heads on 1 KV head, 200 query rows at positions 100..299, canaries at a page boundary (127 | 128, also a
    64-key tile boundary), inside a page (192 starts a tile) and near the end"""
    rng = np.random.default_rng(11)
    S, R = 300, 200
    pos = np.arange(S - R, S)
    keys = [127, 128, 192, 250]
    q, k, v = ao.plant_prefill_keys(_rand(rng, R, 4, 128), pos, _rand(rng, S, 1, 128), _rand(rng, S, 1, 128), keys)
    ref, A = ao.attention(q, k, v, pos + 1)
    ao.check_prefill_canaries(q, pos, k, v, keys, ref)
    return q, k, v, pos, ref, A


@pytest.fixture(scope="module")
def decode():
    """8 heads on 2 KV heads, a 3000-token context (three 1024-token chunks), the new token planted"""
    rng = np.random.default_rng(12)
    ctx = 3000
    cos, sin = rope_tables(PRESETS["tiny"], ctx)
    q = ao.rope(_rand(rng, 8, 128), cos[ctx - 1], sin[ctx - 1])
    k, v = ao.plant_decode_key(q, _rand(rng, ctx, 2, 128), _rand(rng, ctx, 2, 128), ctx - 1)
    ref, A = ao.attention(q[None], k, v, [ctx])
    ao.check_decode_canary(q, k, v, ctx - 1, ref[0])
    return q, k, v, ctx, ref, A


def _rejected(ref, A, mutant):
    return not ao.within(bf16_round(mutant.astype(np.float32)), ref, A).all()


def test_true_reference_rounded_to_bf16_passes(prefill, decode):
    for case in (prefill, decode):
        ref, A = case[-2], case[-1]
        assert ao.within(bf16_round(ref.astype(np.float32)), ref, A).all()


def test_prefill_mutants_are_rejected(prefill):
    q, k, v, pos, ref, A = prefill
    S = k.shape[0]
    page_from_neighbour_k, page_from_neighbour_v = k.copy(), v.copy()
    page_from_neighbour_k[96:128] = k[128:160]         # page 3 read from page 4
    page_from_neighbour_v[96:128] = v[128:160]
    tile_dropped = np.ones(S)
    tile_dropped[128:192] = 0.0
    mutants = {
        "diagonal key masked out": ao.attention(q, k, v, pos)[0],
        "diagonal + 1 let in": ao.attention(q, k, v, np.minimum(pos + 2, S))[0],
        "one 64-key tile dropped": ao.attention(q, k, v, pos + 1, key_weight=tile_dropped)[0],
        "one page read from its neighbour": ao.attention(q, page_from_neighbour_k, page_from_neighbour_v, pos + 1)[0],
    }
    kept = [name for name, m in mutants.items() if not _rejected(ref, A, m)]
    assert not kept, kept


def test_decode_mutants_are_rejected(decode):
    q, k, v, ctx, ref, A = decode

    def weighted(lo, hi, w):
        kw = np.ones(ctx)
        kw[lo:hi] = w
        return ao.attention(q[None], k, v, [ctx], key_weight=kw)[0]

    mutants = {
        "one decode chunk dropped": weighted(1024, 2048, 0.0),
        "one decode chunk merged twice": weighted(1024, 2048, 2.0),
        "new token dropped": weighted(ctx - 1, ctx, 0.0),
        "new token counted twice": weighted(ctx - 1, ctx, 2.0),
    }
    kept = [name for name, m in mutants.items() if not _rejected(ref, A, m)]
    assert not kept, kept


def test_bf16_p_is_rejected_in_the_cancellation_case():
    """Two keys with V = +1 and -1 and weights 1 : 0.984: the output (~0.008) is a difference of two nearly equal
    halves, so rounding P to bf16 (no lo part) moves it by far more than the bf16 rounding of the output."""
    q = np.zeros((1, 1, 128), np.float32)
    k = np.zeros((2, 1, 128), np.float32)
    v = np.zeros((2, 1, 128), np.float32)
    q[0, 0, 0] = 1.0
    k[1, 0, 0] = bf16_round(np.array([np.log(0.984) / ao.SCALE], np.float32))[0]
    v[0], v[1] = 1.0, -1.0
    ref, A = ao.attention(q, k, v, [2])
    assert 0.005 < ref[0, 0, 0] < 0.01
    assert ao.within(bf16_round(ref.astype(np.float32)), ref, A).all()
    assert _rejected(ref, A, ao.attention(q, k, v, [2], p_bf16=True)[0])


def test_split_exact_and_rope_inverse():
    rng = np.random.default_rng(5)
    x = _rand(rng, 3, 256)
    for splits in (1, 2, 9):
        assert np.array_equal(ao.reduce_planes(ao.split_exact(x, splits, rng)), x)
    cos, sin = rope_tables(PRESETS["tiny"], 100)
    y = _rand(rng, 4, 128)
    back = ao.rope(ao.unrope(y, cos[77], sin[77]), cos[77], sin[77])
    assert np.max(np.abs(back - y)) <= 2.0 ** -6 * np.max(np.abs(y))
