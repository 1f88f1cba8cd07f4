"""Mixtral mixture-of-experts block (csrc/moe.cu and the grouped mode of csrc/gemm_wgmma.cuh), stage by stage.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

Every stage takes the previous stage's output as an argument, so a test can feed it what the kernel produced and
check one stage at a time:
    routing    router_logits (llama_oracle, bit-exact) -> top2 (the kernel's fp32 selection and weights);
               top2_weights_f64 = the weights in float64 from the kernel's fp32 logit difference
    dispatch   stable counting sort of the (token, k) assignments by expert, and the {expert, first row} tile list
               of the grouped GEMMs: exact integers
    experts    gate_up_f64, swiglu, down_f64: the GEMMs in float64 on the exact bf16 inputs, SwiGLU in the
               kernel's fp32 expression
    combine    fp32(fp32(w0 * a) + fp32(w1 * b)), bit-exact (numpy's fp32 multiply and add round like
               __fmul_rn / __fadd_rn), then one bf16 rounding or the fp32 partial
moe_block is LlamaOracle._moe's expert loop and combine (fp32 matmuls, bf16 at the engine's rounding points).

Tolerances, one statement each:
    GEMM stage (he's inputs, ye)   |got - ref| <= ulp(ref) + GEMM_ABS * A,   A = sum_k |x_k w_k|
        one bf16 ulp of the float64 result covers the output rounding (half an ulp) plus a rounding that fp32
        accumulation pushes across a midpoint; GEMM_ABS * A covers the fp32 accumulation error where the sum cancels.
    SwiGLU stage (he)              |got - ref| <= 4 ulp(ref) + slack everywhere, <= ulp(ref) for >= 99.5 %
        ref = swiglu(bf16(g), bf16(u)) of the float64 gate / up; slack = |u silu'(g)| dg + |silu(g)| du with dg, du
        the GEMM-stage bounds of g and u: three roundings are chained, and a one-ulp flip of g or u moves h.
    whole block (out)              the SwiGLU policy with A = w0 A0 + w1 A1 over the down GEMMs, BLOCK_ABS * A
"""
from __future__ import annotations

import numpy as np

from .bf16 import bf16_round
from .llama_oracle import router_logits  # noqa: F401  (re-exported: the routing stage starts here)

GEMM_ABS = 2.0 ** -14
BLOCK_ABS = 2.0 ** -10     # a one-ulp flip of h_j moves ye by up to 2^-7 |h_j wd_j|; 2^-12 was exceeded 2x on an H100
SWIGLU_FEW_ULP = 4
SWIGLU_ONE_ULP_SHARE = 0.995
WEIGHT_ULP = 4            # topk_w vs top2_weights_f64, in fp32 ulp (expf, one add, one divide)


# ---------------------------------------------------------------- routing


def top2(r: np.ndarray):
    """fp32 logits [T][E] -> (idx [T][2] int32, w [T][2] fp32): the two largest logits (lowest index wins ties),
    w0 = 1/(1+exp(r1-r0)), w1 = exp(r1-r0)/(1+exp(r1-r0)) in fp32, as moe_router_kernel computes them."""
    T = r.shape[0]
    t = np.arange(T)
    e0 = np.argmax(r, axis=1)
    r_masked = r.copy()
    r_masked[t, e0] = -np.inf
    e1 = np.argmax(r_masked, axis=1)
    ex = np.exp((r[t, e1] - r[t, e0]).astype(np.float32)).astype(np.float32)
    w0 = (np.float32(1.0) / (np.float32(1.0) + ex)).astype(np.float32)
    w1 = (ex / (np.float32(1.0) + ex)).astype(np.float32)
    return np.stack([e0, e1], axis=1).astype(np.int32), np.stack([w0, w1], axis=1)


def top2_weights_f64(r: np.ndarray, idx: np.ndarray) -> np.ndarray:
    """float64 weights [T][2] of the selected experts: 1/(1+e^d), e^d/(1+e^d) with d = fp32(r1 - r0), the
    kernel's own fp32 difference (its rounding is amplified by exp; everything after it is float64 here)."""
    t = np.arange(r.shape[0])
    d = (r[t, idx[:, 1]] - r[t, idx[:, 0]]).astype(np.float32).astype(np.float64)
    ex = np.exp(d)
    return np.stack([1.0 / (1.0 + ex), ex / (1.0 + ex)], axis=1)


def f32_ulp(x: np.ndarray) -> np.ndarray:
    return np.spacing(np.abs(np.asarray(x, np.float32))).astype(np.float64)


# ---------------------------------------------------------------- dispatch


def dispatch(topk_idx: np.ndarray, e_first: int, e_local: int):
    """(row_of [T][2] int32, ranges [e_local][2] int32): assignments of experts e_first .. e_first+e_local-1 sorted
    by expert, in (token, k) order inside an expert; -1 for an expert on another rank."""
    flat = np.asarray(topk_idx, np.int64).reshape(-1) - e_first
    local = (flat >= 0) & (flat < e_local)
    order = np.argsort(np.where(local, flat, e_local), kind="stable")
    n_local = int(local.sum())
    row_of = np.full(flat.shape, -1, np.int32)
    row_of[order[:n_local]] = np.arange(n_local, dtype=np.int32)
    counts = np.bincount(flat[local], minlength=e_local).astype(np.int32)
    first = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.int32)
    return row_of.reshape(-1, 2), np.stack([first, counts], axis=1)


def tile_list(ranges: np.ndarray, bn: int) -> np.ndarray:
    """[n][2] int32: one {expert, first row inside the expert} per bn-row tile, experts in order"""
    tiles = [(e, n0) for e, (_, rows) in enumerate(np.asarray(ranges)) for n0 in range(0, int(rows), bn)]
    return np.asarray(tiles, np.int32).reshape(-1, 2)


def tile_cap(T: int, bn: int, e_local: int) -> int:
    """csrc/moe.cu moe_tile_cap: the grid the grouped GEMMs launch (each expert wastes < one tile)"""
    return (2 * T + bn - 1) // bn + e_local


def pick_bn(T: int, experts: int) -> int:
    """Model::moe_mlp's N tile: gemm_pick_bn(ceil(2T / E))"""
    n = (2 * T + experts - 1) // experts
    return next(b for b in (16, 32, 64, 128) if n <= b) if n <= 128 else 256


def routing_from_counts(counts, rng) -> np.ndarray:
    """[T][2] expert ids where expert e takes exactly counts[e] assignments (sum = 2T, each <= T) and a token never
    picks one expert twice: the sorted 2T labels L give token t the pair (L[t], L[t + T]), tokens shuffled."""
    counts = np.asarray(counts, np.int64)
    T = int(counts.sum()) // 2
    assert counts.sum() == 2 * T and counts.max() <= T
    labels = np.repeat(np.arange(len(counts)), counts)
    idx = np.stack([labels[:T], labels[T:]], axis=1)[rng.permutation(T)]
    swap = rng.random(T) < 0.5
    idx[swap] = idx[swap][:, ::-1]
    assert np.all(idx[:, 0] != idx[:, 1])
    return idx.astype(np.int32)


def forced_routings(T, E, bn, rng):
    """forced routings of T tokens over E experts: uniform, all on two experts, half the experts empty, and expert
    row counts of exactly bn - 1, bn and bn + 1 (where 2T allows)"""
    out = {"random": np.stack([rng.permutation(E)[:2] for _ in range(T)]).astype(np.int32) if T <= 4097 else
           routing_from_counts(np.diff(np.linspace(0, 2 * T, E + 1).astype(np.int64)), rng)}
    out["two"] = routing_from_counts([T if e in (1, E - 1) else 0 for e in range(E)], rng)
    used = list(range(0, E, 2))
    c = np.diff(np.linspace(0, 2 * T, len(used) + 1).astype(np.int64))
    if T >= 2 and c.max() <= T:
        out["empty"] = routing_from_counts([c[used.index(e)] if e in used else 0 for e in range(E)], rng)
    if 2 * T >= 3 * bn + 2 * (E - 3) and E >= 5:
        rest = 2 * T - 3 * bn
        spread = np.diff(np.linspace(0, rest, E - 2).astype(np.int64))
        counts = np.asarray([bn - 1, bn, bn + 1] + list(spread))
        if counts.max() <= T:
            out["bn"] = routing_from_counts(counts, rng)
    return out


def random_weights(T: int, rng) -> np.ndarray:
    """[T][2] fp32 routing weights w0 >= w1, w0 + w1 ~ 1, as the router produces them"""
    w0 = rng.uniform(0.5, 1.0, T).astype(np.float32)
    return np.stack([w0, (np.float32(1.0) - w0).astype(np.float32)], axis=1)


# ---------------------------------------------------------------- expert stages (float64 on the bf16 inputs)


def _gemm_f64(x, w):
    x64, w64 = np.asarray(x, np.float64), np.asarray(w, np.float64)
    # A only scales the tolerance: its own rounding does not matter, so fp32 is enough
    return x64 @ w64.T, np.abs(np.asarray(x, np.float32)) @ np.abs(np.asarray(w, np.float32)).T


def gate_up_f64(x: np.ndarray, wgu: np.ndarray):
    """x [n][H] bf16 values, wgu [2 ffn][H] (gate rows, then up rows) -> (g, u, A_g, A_u) float64 [n][ffn]"""
    ffn = wgu.shape[0] // 2
    gu, a = _gemm_f64(x, wgu)
    return gu[:, :ffn], gu[:, ffn:], a[:, :ffn].astype(np.float64), a[:, ffn:].astype(np.float64)


def down_f64(h: np.ndarray, wdown: np.ndarray):
    """h [n][ffn] bf16 values, wdown [H][ffn] -> (ye, A) float64 [n][H]"""
    ye, a = _gemm_f64(h, wdown)
    return ye, a.astype(np.float64)


def swiglu(g: np.ndarray, u: np.ndarray) -> np.ndarray:
    """the fused epilogue on bf16 g, u: bf16(bf16(g / (1 + exp(-g))) * u), fp32 arithmetic"""
    g, u = np.asarray(g, np.float32), np.asarray(u, np.float32)
    return bf16_round(bf16_round(g / (np.float32(1.0) + np.exp(-g))) * u)


# ---------------------------------------------------------------- combine


def combine(ye0: np.ndarray, ye1: np.ndarray, w: np.ndarray, partial_f32: bool = False) -> np.ndarray:
    """out[t] = fp32(w0 * ye0[t]) + fp32(w1 * ye1[t]) in fp32 (rows of a remote expert are zeros), then one bf16
    rounding, or the fp32 partial"""
    w = np.asarray(w, np.float32)
    o = ((w[:, :1] * ye0).astype(np.float32) + (w[:, 1:] * ye1).astype(np.float32)).astype(np.float32)
    return o if partial_f32 else bf16_round(o)


def moe_block(x, topk_idx, topk_w, gu_of, down_of, experts: int, rnd):
    """LlamaOracle._moe after routing: x [T][H], topk_idx / topk_w [T][2], gu_of(e) = [gate; up] [2 ffn][H] and
    down_of(e) = [H][ffn] fp32 weights; rnd = bf16_round at the engine's rounding points (or fp32, no rounding)."""
    T, H = x.shape
    e0, e1 = topk_idx[:, 0], topk_idx[:, 1]
    w0, w1 = topk_w[:, 0], topk_w[:, 1]
    out0 = np.zeros((T, H), np.float32)
    out1 = np.zeros((T, H), np.float32)
    for e in range(experts):
        for sel, dst in ((e0, out0), (e1, out1)):
            rows = np.nonzero(sel == e)[0]
            if rows.size == 0:
                continue
            wgu = gu_of(e)
            ffn = wgu.shape[0] // 2
            gu = rnd(x[rows] @ wgu.T)
            g, u = gu[:, :ffn], gu[:, ffn:]
            act = rnd(g / (np.float32(1.0) + np.exp(-g)))
            dst[rows] = rnd(rnd(act * u) @ down_of(e).T)
    return rnd((w0[:, None] * out0).astype(np.float32) + (w1[:, None] * out1).astype(np.float32))


# ---------------------------------------------------------------- tolerances


def bf16_ulp(ref: np.ndarray) -> np.ndarray:
    """one bf16 ulp at |ref| (8 significant bits), 0 at 0"""
    ref = np.abs(np.asarray(ref, np.float64))
    _, e = np.frexp(ref)
    return np.where(ref > 0, np.ldexp(1.0, e - 8), 0.0)


def gemm_excess(got, ref, a) -> float:
    """max |got - ref| / (ulp(ref) + GEMM_ABS * A): <= 1 passes (NaN counts as a failure)"""
    err = np.abs(np.asarray(got, np.float64) - ref)
    r = err / (bf16_ulp(ref) + GEMM_ABS * a)
    return float(np.inf) if not np.all(np.isfinite(r)) else float(r.max(initial=0.0))


def swiglu_ref(g64, u64, a_g, a_u):
    """(ref, slack) of the SwiGLU stage from the float64 gate / up and their A"""
    ref = swiglu(bf16_round(g64.astype(np.float32)), bf16_round(u64.astype(np.float32))).astype(np.float64)
    s = 1.0 / (1.0 + np.exp(-g64))
    dsilu = s * (1.0 + g64 * (1.0 - s))
    dg = bf16_ulp(g64) + GEMM_ABS * a_g
    du = bf16_ulp(u64) + GEMM_ABS * a_u
    return ref, np.abs(u64 * dsilu) * dg + np.abs(g64 * s) * du


def few_ulp_check(got, ref, slack):
    """(worst |got - ref| / (4 ulp(ref) + slack), share of elements within one ulp(ref) + slack / 4): the first
    must be <= 1, the second >= SWIGLU_ONE_ULP_SHARE"""
    err = np.abs(np.asarray(got, np.float64) - ref)
    ulp = bf16_ulp(ref)
    r = err / (SWIGLU_FEW_ULP * ulp + slack + 1e-300)
    worst = float(np.inf) if not np.all(np.isfinite(r)) else float(r.max(initial=0.0))
    return worst, float(np.mean(err <= ulp + slack / SWIGLU_FEW_ULP))


def block_abs(topk_w, a0, a1):
    """A of the whole block: w0 A0 + w1 A1 (A_k = sum_j |h_j wd_j| of expert k's down GEMM, 0 for a remote one)"""
    w = np.asarray(topk_w, np.float64)
    return w[:, :1] * a0 + w[:, 1:] * a1


def block_check(got, ref, a):
    """few_ulp_check of a whole block against the bf16-mode moe_block, slack BLOCK_ABS * A"""
    return few_ulp_check(got, ref, BLOCK_ABS * a)
