"""The mixture-of-experts oracle (oracle/moe_oracle.py) without a GPU: its dispatch against a naive per-token loop,
LlamaOracle._moe against the code it was factored out of, and its tolerances against mutants of the block.

The mutants are the ways a router / dispatch / grouped GEMM / combine kernel goes subtly wrong; each must fail the
check tests/test_moe_gpu.py applies to the kernels, while the unmutated block computed with fp32 GEMMs passes it."""
import numpy as np
import pytest

from oracle import moe_oracle as mo
from oracle.bf16 import bf16_round
from oracle.llama_oracle import PRESETS, LlamaOracle, router_logits

SEED = 0xACB200


# ---------------------------------------------------------------- dispatch


def _naive_dispatch(idx, e_first, e_local):
    counts = [0] * e_local
    for t in range(idx.shape[0]):
        for k in range(2):
            e = int(idx[t, k]) - e_first
            if 0 <= e < e_local:
                counts[e] += 1
    first = [sum(counts[:e]) for e in range(e_local)]
    seen = [0] * e_local
    row_of = np.full(idx.shape, -1, np.int32)
    for t in range(idx.shape[0]):
        for k in range(2):
            e = int(idx[t, k]) - e_first
            if 0 <= e < e_local:
                row_of[t, k] = first[e] + seen[e]
                seen[e] += 1
    return row_of, np.array([first, counts], np.int32).T


@pytest.mark.parametrize("T", [1, 2, 1023, 1024, 1025, 4097, 32767])
def test_dispatch_matches_per_token_loop(T):
    rng = np.random.default_rng(T)
    E = 8
    for bn in (16, 64, 256):
        for kind, idx in mo.forced_routings(T, E, bn, rng).items():
            for e_first, e_local in ((0, E), (0, 1), (3, 2), (4, 4), (7, 1)):
                row_of, ranges = mo.dispatch(idx, e_first, e_local)
                if T <= 4097 or bn == 16:   # the Python loop is slow: once per routing at T = 32767
                    n_row_of, n_ranges = _naive_dispatch(idx, e_first, e_local)
                    assert np.array_equal(row_of, n_row_of), (T, kind, e_first, e_local)
                    assert np.array_equal(ranges, n_ranges), (T, kind, e_first, e_local)
                tiles = mo.tile_list(ranges, bn)
                want = [(e, n0) for e in range(e_local) for n0 in range(0, int(ranges[e, 1]), bn)]
                assert tiles.tolist() == [list(t) for t in want]
                assert len(tiles) <= mo.tile_cap(T, bn, e_local), (T, kind, bn, e_local)
                # every local assignment has one row, rows are a permutation of 0..n-1
                local = row_of[row_of >= 0]
                assert np.array_equal(np.sort(local), np.arange(int(ranges[:, 1].sum())))
            if kind == "bn":
                counts = np.bincount(idx.reshape(-1), minlength=E)
                assert counts[0] == bn - 1 and counts[1] == bn and counts[2] == bn + 1
            if kind == "two":
                assert set(np.unique(idx)) == {1, E - 1}


def test_tile_cap_holds_with_a_partial_tile_per_expert():
    """every expert one row past a whole number of tiles: the most tiles 2T rows can make"""
    rng = np.random.default_rng(1)
    bn, E = 16, 8
    counts = [bn * q + 1 for q in (0, 1, 2, 3, 3, 2, 1, 0)]   # sum 2T = 200
    idx = mo.routing_from_counts(counts, rng)
    _, ranges = mo.dispatch(idx, 0, E)
    n = len(mo.tile_list(ranges, bn))
    assert n == 12 + E and n <= mo.tile_cap(idx.shape[0], bn, E)


# ---------------------------------------------------------------- _moe refactor


def _moe_pre_refactor(orc, xn2, l):
    """LlamaOracle._moe as it was before its stages moved to oracle/moe_oracle.py"""
    c = orc.cfg
    T = xn2.shape[0]
    r = router_logits(xn2, orc.w.router(l))
    e0 = np.argmax(r, axis=1)
    r_masked = r.copy()
    r_masked[np.arange(T), e0] = -np.inf
    e1 = np.argmax(r_masked, axis=1)
    ex = np.exp((r[np.arange(T), e1] - r[np.arange(T), e0]).astype(np.float32)).astype(np.float32)
    w0 = (np.float32(1.0) / (np.float32(1.0) + ex)).astype(np.float32)
    w1 = (ex / (np.float32(1.0) + ex)).astype(np.float32)
    out0 = np.zeros((T, c.hidden), np.float32)
    out1 = np.zeros((T, c.hidden), np.float32)
    for e in range(c.experts):
        for sel, dst in ((e0, out0), (e1, out1)):
            rows = np.nonzero(sel == e)[0]
            if rows.size == 0:
                continue
            gu = orc._r(xn2[rows] @ orc.w.expert_gu(l, e).T)
            g, u = gu[:, :c.ffn], gu[:, c.ffn:]
            act = orc._r(g / (np.float32(1.0) + np.exp(-g)))
            dst[rows] = orc._r(orc._r(act * u) @ orc.w.expert_down(l, e).T)
    return orc._r((w0[:, None] * out0).astype(np.float32) + (w1[:, None] * out1).astype(np.float32)), (e0, e1, w0, w1)


@pytest.mark.parametrize("mode", ["bf16", "fp32"])
def test_moe_refactor_is_bit_identical(mode):
    cfg = PRESETS["tiny-moe"]
    orc = LlamaOracle(cfg, SEED, mode=mode)
    rng = np.random.default_rng(5)
    for T in (1, 7, 64):
        xn2 = bf16_round(rng.standard_normal((T, cfg.hidden)).astype(np.float32))
        for l in range(cfg.layers):
            want, routing = _moe_pre_refactor(orc, xn2, l)
            got = orc._moe(xn2, l)
            assert got.dtype == want.dtype and np.array_equal(got.view(np.uint32), want.view(np.uint32)), (mode, T, l)
            for a, b in zip(orc.last_routing, routing):
                assert np.array_equal(a, b)


# ---------------------------------------------------------------- tolerances vs mutants


class Block:
    """A tiny-moe-sized block with forced routing, its float64 stage references, and the kernel-layout pipeline
    (fp32 GEMMs, the kernel's rounding points) that mutants are made from."""

    H, FFN, E, T, BN = 512, 768, 8, 200, 16

    def __init__(self, seed=3):
        rng = np.random.default_rng(seed)
        self.x = bf16_round(rng.standard_normal((self.T, self.H)).astype(np.float32))
        self.wgu = bf16_round((rng.standard_normal((self.E, 2 * self.FFN, self.H)) * 0.02).astype(np.float32))
        self.wd = bf16_round((rng.standard_normal((self.E, self.H, self.FFN)) * 0.02).astype(np.float32))
        # counts with partial last tiles, and an expert holding one row
        self.idx = mo.routing_from_counts([37, 1, 64, 65, 48, 80, 55, 50], rng)
        self.w = mo.random_weights(self.T, rng)
        self.row_of, self.ranges = mo.dispatch(self.idx, 0, self.E)
        self.ref_out = mo.moe_block(self.x, self.idx, self.w, lambda e: self.wgu[e], lambda e: self.wd[e], self.E,
                                    bf16_round)

    def run(self, mutation=None):
        """(he, ye, out) in the kernel's layout"""
        x, idx, w = self.x, self.idx.copy(), self.w.copy()
        if mutation == "second_is_third":
            third = (idx[:, 1] + 1) % self.E
            third = np.where(third == idx[:, 0], (third + 1) % self.E, third)
            idx[:, 1] = third
        row_of, ranges = mo.dispatch(idx, 0, self.E)
        n = int(ranges[:, 1].sum())
        xe = np.zeros((n + 1, self.H), np.float32)
        for k in range(2):
            xe[row_of[:, k]] = x
        he = np.zeros((n, self.FFN), np.float32)
        ye = np.zeros((n, self.H), np.float32)
        for e, (f, c) in enumerate(ranges):
            src = xe[f + 1:f + c + 1] if mutation == "shift_group" and e == 2 else xe[f:f + c]
            gu = bf16_round(src @ self.wgu[e].T)
            if mutation == "deinterleave":   # the kernel pairs rows 2j, 2j + 1 of an un-interleaved [gate; up]
                g, u = gu[:, 0::2], gu[:, 1::2]
            else:
                g, u = gu[:, :self.FFN], gu[:, self.FFN:]
            he[f:f + c] = mo.swiglu(g, u)
            ye[f:f + c] = bf16_round(he[f:f + c] @ self.wd[e].T)
            if mutation == "drop_last_partial_tile" and c % self.BN:
                ye[f + c - c % self.BN:f + c] = 0.0
        if mutation == "neighbour_row":   # one token's row from its neighbour in expert 3
            f = int(ranges[3, 0])
            ye[f + 10] = ye[f + 11]
        if mutation == "swap_w":
            w = w[:, ::-1].copy()
        ye_k = [np.where(row_of[:, k:k + 1] >= 0, ye[np.maximum(row_of[:, k], 0)], 0.0).astype(np.float32) for k in range(2)]
        return he, ye, mo.combine(ye_k[0], ye_k[1], w)

    def report(self, he, ye, out):
        """worst excess / one-ulp share of each stage, every stage checked on the previous stage's output"""
        r = {}
        he_w, he_s, ye_w = 0.0, 1.0, 0.0
        a_rows = np.zeros((ye.shape[0], self.H))
        for e, (f, c) in enumerate(self.ranges):
            if c == 0:
                continue
            rows = np.nonzero((self.idx == e).any(axis=1))[0]
            tok = np.zeros(c, np.int64)
            for k in range(2):
                sel = self.idx[:, k] == e
                tok[self.row_of[sel, k] - f] = np.nonzero(sel)[0]
            assert len(rows) == c
            g, u, ag, au = mo.gate_up_f64(self.x[tok], self.wgu[e])
            ref, slack = mo.swiglu_ref(g, u, ag, au)
            w_, s_ = mo.few_ulp_check(he[f:f + c], ref, slack)
            he_w, he_s = max(he_w, w_), min(he_s, s_)
            yref, a = mo.down_f64(he[f:f + c], self.wd[e])
            ye_w = max(ye_w, mo.gemm_excess(ye[f:f + c], yref, a))
            a_rows[f:f + c] = a
        a_k = [np.where(self.row_of[:, k:k + 1] >= 0, a_rows[np.maximum(self.row_of[:, k], 0)], 0.0) for k in range(2)]
        bw, bs = mo.block_check(out, self.ref_out, mo.block_abs(self.w, a_k[0], a_k[1]))
        r.update(he=he_w, he_share=he_s, ye=ye_w, block=bw, block_share=bs)
        return r


@pytest.fixture(scope="module")
def block():
    return Block()


def _passes(r, stage):
    if stage == "he":
        return r["he"] <= 1.0 and r["he_share"] >= mo.SWIGLU_ONE_ULP_SHARE
    if stage == "block":
        return r["block"] <= 1.0 and r["block_share"] >= mo.SWIGLU_ONE_ULP_SHARE
    return r[stage] <= 1.0


def test_unmutated_block_passes_every_stage(block):
    r = block.report(*block.run())
    assert all(_passes(r, s) for s in ("he", "ye", "block")), r
    # the fp32 GEMMs really do differ from float64 somewhere (the tolerance is exercised, not idle)
    assert r["he"] > 0 and r["ye"] > 0, r


def test_float64_block_passes_block_check(block):
    """moe_block with float64 GEMMs (exact accumulation, same rounding points) vs the fp32 one: the accumulation
    order the kernels are free to choose stays inside the block tolerance"""
    out64 = mo.moe_block(block.x.astype(np.float64), block.idx, block.w, lambda e: block.wgu[e].astype(np.float64),
                         lambda e: block.wd[e].astype(np.float64), block.E, bf16_round)
    he, ye, _ = block.run()
    r = block.report(he, ye, out64)
    assert _passes(r, "block"), r


# mutation -> the stage check that must catch it, besides the whole-block check
MUTANTS = {
    "swap_w": None,
    "second_is_third": None,
    "neighbour_row": "ye",
    "shift_group": "he",
    "drop_last_partial_tile": "ye",
    "deinterleave": "he",
}


@pytest.mark.parametrize("mutation", sorted(MUTANTS))
def test_mutant_fails_the_checks(block, mutation):
    r = block.report(*block.run(mutation))
    assert not _passes(r, "block"), (mutation, r)
    # by a wide margin: 8x the tolerance, or most elements off by more than one ulp
    assert r["block"] > 8 or r["block_share"] < 0.9, (mutation, r)
    if MUTANTS[mutation]:
        assert not _passes(r, MUTANTS[mutation]), (mutation, r)


def test_top2_weights_f64_agree_with_top2():
    rng = np.random.default_rng(9)
    x = bf16_round(rng.standard_normal((500, 512)).astype(np.float32))
    wr = bf16_round((rng.standard_normal((8, 512)) * 0.05).astype(np.float32))
    idx, w = mo.top2(router_logits(x, wr))
    w64 = mo.top2_weights_f64(router_logits(x, wr), idx)
    assert np.all(np.abs(w - w64) <= mo.WEIGHT_ULP * mo.f32_ulp(w64))
