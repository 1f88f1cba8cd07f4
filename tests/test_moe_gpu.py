"""The Mixtral mixture-of-experts block (agentcontrolplane_b200/csrc/moe.cu: router, dispatch, gather, combine; the
grouped mode of gemm_wgmma.cuh: gate/up GEMM with fused SwiGLU and down GEMM) stage by stage against
oracle/moe_oracle.py, through the hook acp_kernel_moe (include/acp_infer_kernels.h).

Every stage is checked on the kernel's own output of the stage before it, so a routing near-tie never excuses a
mismatch: topk_idx bit-equal to the oracle router, row_of / ranges / tile list equal to the oracle dispatch of the
kernel's topk_idx, he and ye within the float64 tolerances on the rows the kernel gathered, out bit-equal to the fp32
combine of the kernel's ye and weights.  The hook's guards (expert rows past the step, the dispatch array past its
tile list, the tile capacity, stores past an output) hold in every call."""
import ctypes

import numpy as np
import pytest

from agentcontrolplane_b200 import _lib
from oracle import moe_oracle as mo
from oracle.bf16 import bf16_round, bf16_round_to_bits, bits_to_f32
from oracle.llama_oracle import PRESETS, router_logits, shared_weights

pytestmark = pytest.mark.gpu

SEED = 0xACB200
WORST = {}   # stage -> worst tolerance excess seen (printed at the end of the module with -s)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nmoe worst tolerance excess per stage:", {k: round(v, 4) for k, v in sorted(WORST.items())})


def _note(stage, v):
    WORST[stage] = max(WORST.get(stage, 0.0), v)


def _hook(xn, wr, wgu, wdown, E, e_first=0, bn=0, t_cap=None, partial=False, topk=None, expect=0):
    """bf16 bit arrays in; dict of the hook's outputs (he / ye trimmed to the local assignments)"""
    lib = _lib.load()
    T, H = xn.shape
    e_local, ffn = wgu.shape[0], wgu.shape[1] // 2
    i32p, f32p, u16p = (ctypes.POINTER(t) for t in (ctypes.c_int32, ctypes.c_float, ctypes.c_uint16))
    lib.acp_kernel_moe.argtypes = [u16p, u16p, u16p, u16p] + [ctypes.c_int] * 9 + [i32p, f32p, i32p, f32p, i32p, i32p,
                                                                                   i32p, i32p, u16p, u16p, ctypes.c_void_p]
    c = lambda a, t: np.ascontiguousarray(a).ctypes.data_as(t) if a is not None else None   # noqa: E731
    xn, wgu, wdown = (np.ascontiguousarray(a, np.uint16) for a in (xn, wgu, wdown))
    wr = None if wr is None else np.ascontiguousarray(wr, np.uint16)
    tk_i, tk_w = (None, None) if topk is None else (np.ascontiguousarray(topk[0], np.int32), np.ascontiguousarray(topk[1], np.float32))
    r = dict(topk_idx=np.zeros((T, 2), np.int32), topk_w=np.zeros((T, 2), np.float32), row_of=np.zeros((T, 2), np.int32),
             ranges=np.zeros((e_local, 2), np.int32), tiles=np.zeros((2 * T + e_local, 2), np.int32),
             info=np.zeros(4, np.int32), he=np.zeros((2 * T, ffn), np.uint16), ye=np.zeros((2 * T, H), np.uint16),
             out=np.zeros((T, H), np.float32 if partial else np.uint16))
    rc = lib.acp_kernel_moe(c(xn, u16p), c(wr, u16p), c(wgu, u16p), c(wdown, u16p), T, H, ffn, E, e_first, e_local, bn,
                            t_cap or T, int(partial), c(tk_i, i32p), c(tk_w, f32p), c(r["topk_idx"], i32p),
                            c(r["topk_w"], f32p), c(r["row_of"], i32p), c(r["ranges"], i32p), c(r["tiles"], i32p),
                            c(r["info"], i32p), c(r["he"], u16p), c(r["ye"], u16p), r["out"].ctypes.data)
    assert rc == expect, f"acp_kernel_moe rc={rc}"
    if rc != 0:
        return None
    r["bn"], n_tiles, n_local, r["cap"] = (int(v) for v in r["info"])
    r["tiles"], r["he"], r["ye"] = r["tiles"][:n_tiles], r["he"][:n_local], r["ye"][:n_local]
    return r


class Weights:
    """bf16 bit patterns of one MoE layer: router [E][H], experts' [gate; up] [E][2 ffn][H] and down [E][H][ffn]"""

    def __init__(self, wr, wgu, wd):
        self.wr, self.wgu, self.wd = wr, wgu, wd
        self.E, self.H, self.ffn = wgu.shape[0], wgu.shape[2], wgu.shape[1] // 2

    @classmethod
    def random(cls, H, ffn, E, seed):
        """random bf16 weights of magnitude ~0.02: sign and mantissa random, exponent 2^-9 .. 2^-6 (cheap at
        Mixtral width, where a normal draw of 2.8 GB of weights would dominate the test)"""
        rng = np.random.default_rng(seed)

        def bits(shape):
            raw = rng.integers(0, 1 << 16, size=shape, dtype=np.uint16)
            return (raw & np.uint16(0x807F)) | ((np.uint16(118) + ((raw >> np.uint16(7)) & np.uint16(3))) << np.uint16(7))

        wr = bf16_round_to_bits((rng.standard_normal((E, H)) * 0.05).astype(np.float32))
        return cls(wr, bits((E, 2 * ffn, H)), bits((E, H, ffn)))

    @classmethod
    def preset(cls, name, layer=0):
        """the synthetic weights of a preset's layer (what the engine runs)"""
        cfg = PRESETS[name]
        w = shared_weights(cfg, SEED)
        return cls(bf16_round_to_bits(w.router(layer)),
                   np.stack([bf16_round_to_bits(w.expert_gu(layer, e)) for e in range(cfg.experts)]),
                   np.stack([bf16_round_to_bits(w.expert_down(layer, e)) for e in range(cfg.experts)]))


def _x(T, H, seed):
    return bf16_round_to_bits(np.random.default_rng(seed).standard_normal((T, H)).astype(np.float32))


def _per_assignment(rows, row_of, k):
    """rows[row_of[t][k]] for every token, zeros where the expert is remote (row -1 picks the appended zero row)"""
    return np.concatenate([rows, np.zeros((1,) + rows.shape[1:], rows.dtype)])[row_of[:, k]]


def check_stages(W, xn, r, e_first=0, e_local=None, partial=False, routed=True, gemms=True):
    """every stage of one hook call on its own inputs; returns A per (token, k) of the down GEMM (0 when remote)"""
    e_local = W.E if e_local is None else e_local
    T = xn.shape[0]
    x = bits_to_f32(xn)
    if routed:   # router: selection bit-exact, weights within a few fp32 ulp of float64
        logits = router_logits(x, bits_to_f32(W.wr))
        idx, _ = mo.top2(logits)
        assert np.array_equal(r["topk_idx"], idx), int(np.count_nonzero(r["topk_idx"] != idx))
        w64 = mo.top2_weights_f64(logits, r["topk_idx"])
        ex = float(np.max(np.abs(r["topk_w"] - w64) / (mo.WEIGHT_ULP * mo.f32_ulp(w64))))
        _note("router_w", ex)
        assert ex <= 1.0, ex
    # dispatch: exact integers
    row_of, ranges = mo.dispatch(r["topk_idx"], e_first, e_local)
    assert np.array_equal(r["row_of"], row_of)
    assert np.array_equal(r["ranges"], ranges)
    assert np.array_equal(r["tiles"], mo.tile_list(ranges, r["bn"]))
    assert r["cap"] == mo.tile_cap(T, r["bn"], e_local) and len(r["tiles"]) <= r["cap"]
    n = int(ranges[:, 1].sum())
    tok = np.zeros(n, np.int64)
    for k in range(2):
        sel = row_of[:, k] >= 0
        tok[row_of[sel, k]] = np.nonzero(sel)[0]
    he, ye = bits_to_f32(r["he"]), bits_to_f32(r["ye"])
    a_rows = np.zeros((n, W.H))
    if gemms:
        bad, total, worst_he, worst_ye = 0, 0, 0.0, 0.0
        for e in range(e_local):
            f, c = (int(v) for v in ranges[e])
            if c == 0:
                continue
            # gate / up + SwiGLU on the token rows the dispatch says were gathered: a wrong xe row fails here
            g, u, ag, au = mo.gate_up_f64(x[tok[f:f + c]], bits_to_f32(W.wgu[e_first + e]))
            ref, slack = mo.swiglu_ref(g, u, ag, au)
            w_, s_ = mo.few_ulp_check(he[f:f + c], ref, slack)
            worst_he = max(worst_he, w_)
            bad += round((1.0 - s_) * ref.size)
            total += ref.size
            # down on the kernel's own he rows
            yref, a = mo.down_f64(he[f:f + c], bits_to_f32(W.wd[e_first + e]))
            worst_ye = max(worst_ye, mo.gemm_excess(ye[f:f + c], yref, a))
            a_rows[f:f + c] = a
        _note("he", worst_he)
        _note("ye", worst_ye)
        assert worst_he <= 1.0, worst_he
        assert total == 0 or bad / total <= 1.0 - mo.SWIGLU_ONE_ULP_SHARE, bad / total
        assert worst_ye <= 1.0, worst_ye
    # combine: bit-exact on the kernel's ye and weights
    ye_k = [_per_assignment(ye, row_of, k) for k in range(2)]
    want = mo.combine(ye_k[0], ye_k[1], r["topk_w"], partial)
    got = r["out"] if partial else bits_to_f32(r["out"])
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), int(np.count_nonzero(got != want))
    return [_per_assignment(a_rows, row_of, k) for k in range(2)]


def check_block(W, xn, r, a_k):
    """the whole block against the bf16-mode oracle moe_block on the kernel's routing"""
    x = bits_to_f32(xn)
    ref = mo.moe_block(x, r["topk_idx"], r["topk_w"], lambda e: bits_to_f32(W.wgu[e]), lambda e: bits_to_f32(W.wd[e]),
                       W.E, bf16_round)
    worst, share = mo.block_check(bits_to_f32(r["out"]), ref, mo.block_abs(r["topk_w"], a_k[0], a_k[1]))
    _note("block", worst)
    assert worst <= 1.0 and share >= mo.SWIGLU_ONE_ULP_SHARE, (worst, share)


# ---------------------------------------------------------------- router


@pytest.mark.parametrize("E", [2, 8, 16])
def test_router_selection_is_bit_exact(E):
    W = Weights.random(512, 128, E, seed=E)
    xn = _x(300, 512, seed=E + 1)
    check_stages(W, xn, _hook(xn, W.wr, W.wgu, W.wd, E))


@pytest.mark.parametrize("tie", ["first_second", "second_third"])
def test_router_ties_pick_the_lowest_index(tie):
    """duplicate router rows give exactly equal logits: the lowest expert index must win the tie"""
    E, H = 8, 512
    W = Weights.random(H, 128, E, seed=21)
    x = bits_to_f32(_x(256, H, seed=22))
    wr = bits_to_f32(W.wr).copy()
    if tie == "first_second":
        wr[5] = wr[2] = 4 * wr[2]          # experts 2 and 5 lead together for about half the tokens
        a, b = 2, 5
    else:
        x[:, :32] = 1.0                    # expert 0 leads every token ...
        wr[0] = 0.0
        wr[0, :32] = 1.0
        wr[6] = wr[4] = 3 * wr[4]          # ... and 4 and 6 tie behind it for about half of them
        a, b = 4, 6
    W.wr = bf16_round_to_bits(wr)
    xn = bf16_round_to_bits(x)
    r = _hook(xn, W.wr, W.wgu, W.wd, E)
    check_stages(W, xn, r)
    logits = router_logits(bits_to_f32(xn), bits_to_f32(W.wr))
    assert np.array_equal(logits[:, a], logits[:, b])
    k = 0 if tie == "first_second" else 1
    tied = r["topk_idx"][:, k] == a
    assert tied.sum() >= 32, int(tied.sum())
    assert not np.any(r["topk_idx"][:, k] == b)


# ---------------------------------------------------------------- dispatch (forced routings)


@pytest.mark.parametrize("T", [1, 2, 1023, 1024, 1025, 4097, 32767])
def test_dispatch_forced_routings(T):
    """row_of / ranges / tile list equal the oracle dispatch for forced routings at a tiny width: uniform, two experts,
    empty experts, counts of exactly bn and bn +- 1, expert-parallel subsets; T > 1024 takes the several-tokens-per-
    thread path of moe_dispatch_kernel"""
    E = 8
    W = Weights.random(128, 64, E, seed=T)
    rng = np.random.default_rng(T)
    xn = _x(T, 128, seed=T + 7)
    bn = mo.pick_bn(T, E)
    for kind, idx in mo.forced_routings(T, E, bn, rng).items():
        w = mo.random_weights(T, rng)
        for e_first, e_local in ((0, E), (3, 2), (7, 1)):
            r = _hook(xn, None, W.wgu[e_first:e_first + e_local], W.wd[e_first:e_first + e_local], E, e_first=e_first,
                      partial=e_local < E, topk=(idx, w))
            assert np.array_equal(r["topk_idx"], idx) and np.array_equal(r["topk_w"], w)
            assert r["bn"] == bn
            check_stages(W, xn, r, e_first, e_local, partial=e_local < E, routed=False)


@pytest.mark.parametrize("t_cap", [1025, 32767])
def test_step_smaller_than_its_buffers(t_cap):
    """the buffers are sized for max_tokens_per_step; a short step must use only its own rows"""
    W = Weights.random(256, 128, 8, seed=5)
    xn = _x(37, 256, seed=6)
    check_stages(W, xn, _hook(xn, W.wr, W.wgu, W.wd, 8, t_cap=t_cap))


# ---------------------------------------------------------------- grouped GEMMs: tile-size invariance


def _bn_invariance(W, xn, bns):
    base = None
    for bn in bns:
        r = _hook(xn, W.wr, W.wgu, W.wd, W.E, bn=bn)
        assert r["bn"] == bn
        if base is None:
            base = r
            a_k = check_stages(W, xn, r)
            check_block(W, xn, r, a_k)
            continue
        check_stages(W, xn, r, gemms=False)
        # per-element accumulation does not depend on the N tile: any difference is a tile-list / row-offset bug
        assert np.array_equal(r["he"], base["he"]), (bn, int(np.count_nonzero(r["he"] != base["he"])))
        assert np.array_equal(r["ye"], base["ye"]), (bn, int(np.count_nonzero(r["ye"] != base["ye"])))
        assert np.array_equal(r["out"], base["out"]), bn


@pytest.mark.parametrize("T", [17, 300])
def test_grouped_gemm_bit_identical_for_every_bn(T):
    _bn_invariance(Weights.preset("tiny-moe"), _x(T, 512, seed=T), [64, 16, 32, 128, 256])


# ---------------------------------------------------------------- whole block


@pytest.mark.parametrize("T", [1, 7, 16, 17, 64, 65, 708, 1025])
def test_block_tiny_moe(T):
    W = Weights.preset("tiny-moe", layer=1)
    xn = _x(T, 512, seed=100 + T)
    r = _hook(xn, W.wr, W.wgu, W.wd, W.E)
    assert r["bn"] == mo.pick_bn(T, W.E)
    check_block(W, xn, r, check_stages(W, xn, r))
    # fp32 partial: the same routing and expert rows, the combine without its rounding
    p = _hook(xn, W.wr, W.wgu, W.wd, W.E, partial=True)
    assert np.array_equal(p["ye"], r["ye"])
    check_stages(W, xn, p, partial=True, gemms=False)
    assert np.array_equal(bf16_round_to_bits(p["out"]), r["out"])


@pytest.fixture(scope="module")
def mixtral():
    """Mixtral-8x7B's MoE width: hidden 4096, ffn 14336, 8 experts (2.8 GB of bf16 expert weights)"""
    return Weights.random(4096, 14336, 8, seed=8)


@pytest.mark.parametrize("T", [1, 100, 300])
def test_block_mixtral_width(mixtral, T):
    """BN 16 (T = 1), 32 (T = 100) and 128 (T = 300) expert tiles at K = 4096 (gate/up) and 14336 (down)"""
    xn = _x(T, 4096, seed=T)
    r = _hook(xn, mixtral.wr, mixtral.wgu, mixtral.wd, 8)
    assert r["bn"] == mo.pick_bn(T, 8)
    check_block(mixtral, xn, r, check_stages(mixtral, xn, r))


def test_mixtral_width_bit_identical_for_bn(mixtral):
    """the T = 300 step again with 256- and 16-row tiles"""
    xn = _x(300, 4096, seed=300)
    base = _hook(xn, mixtral.wr, mixtral.wgu, mixtral.wd, 8)
    for bn in (256, 16):
        r = _hook(xn, mixtral.wr, mixtral.wgu, mixtral.wd, 8, bn=bn)
        check_stages(mixtral, xn, r, gemms=False)
        assert np.array_equal(r["ye"], base["ye"]) and np.array_equal(r["out"], base["out"]), bn


# ---------------------------------------------------------------- expert parallel on one GPU


def _expert_parallel(W, xn, P, check=True):
    """run every rank of a P-way expert-parallel layer; the rank partials, summed in rank order in fp32, are exactly
    the single-rank fp32 partial (other ranks contribute exact zeros; a two-term fp32 sum commutes)"""
    E = W.E
    single = _hook(xn, W.wr, W.wgu, W.wd, E, partial=True)
    single_bf16 = _hook(xn, W.wr, W.wgu, W.wd, E)
    owners = np.zeros(single["row_of"].shape, np.int32)
    acc = None
    for rank in range(P):
        e0, el = rank * E // P, E // P
        r = _hook(xn, W.wr, W.wgu[e0:e0 + el], W.wd[e0:e0 + el], E, e_first=e0, partial=True)
        assert np.array_equal(r["topk_idx"], single["topk_idx"]) and np.array_equal(r["topk_w"], single["topk_w"])
        check_stages(W, xn, r, e0, el, partial=True, routed=rank == 0, gemms=check)
        owners += r["row_of"] >= 0
        acc = r["out"].copy() if acc is None else (acc + r["out"]).astype(np.float32)
    assert np.all(owners == 1)
    assert np.all(acc == single["out"]), int(np.count_nonzero(acc != single["out"]))   # as values: +0 == -0
    assert np.all(bits_to_f32(bf16_round_to_bits(acc)) == bits_to_f32(single_bf16["out"]))


@pytest.mark.parametrize("P", [2, 4, 8])
def test_expert_parallel_tiny_moe(P):
    W = Weights.preset("tiny-moe")
    _expert_parallel(W, _x(300, 512, seed=P), P)


def test_expert_parallel_mixtral_width(mixtral):
    """bench config 4's layout: 8 ranks of one expert each (e_local = 1) at Mixtral width"""
    _expert_parallel(mixtral, _x(300, 4096, seed=9), 8, check=False)


# ---------------------------------------------------------------- repeatability, rejected inputs


def test_repeatable():
    W = Weights.preset("tiny-moe")
    xn = _x(1025, 512, seed=3)
    a = _hook(xn, W.wr, W.wgu, W.wd, W.E)
    b = _hook(xn, W.wr, W.wgu, W.wd, W.E)
    for k in a:
        assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), k


@pytest.mark.parametrize("H,ffn,E,e_first,e_local,t_cap", [
    (192, 64, 8, 0, 8, 0),      # hidden % 128
    (128, 96, 8, 0, 8, 0),      # ffn % 64
    (128, 64, 1, 0, 1, 0),      # E < 2
    (128, 64, 17, 0, 17, 0),    # E > 16
    (128, 64, 8, 6, 3, 0),      # experts past E
    (128, 64, 8, 0, 8, 32768),  # 2 t_cap > 65535
])
def test_rejects_invalid_layouts(H, ffn, E, e_first, e_local, t_cap):
    xn = _x(4, H, seed=0)
    wgu = np.zeros((e_local, 2 * ffn, H), np.uint16)
    wd = np.zeros((e_local, H, ffn), np.uint16)
    wr = np.zeros((E, H), np.uint16)
    _hook(xn, wr, wgu, wd, E, e_first=e_first, t_cap=t_cap or None, expect=-1)
