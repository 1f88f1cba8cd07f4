"""float64 reference of the paged attention kernels (csrc/attention.cu, csrc/attention_prefill_tc.cu), the one
tolerance every attention test uses, and planted keys ("canaries") that make a wrong key visible.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

Inputs are bf16 values held in fp32 arrays.  What the kernels compute bit-exactly is mirrored bit-exactly: the
split-K reduction of the QKV projection (planes summed in index order from +0 in fp32, one bf16 rounding, like
csrc/gemm_out.cuh) and RoPE (fp32, separately rounded multiply / subtract as in LlamaOracle._rope, then bf16).
Softmax attention itself is computed in float64.

Tolerance: |got - ref| <= 2^-8 |ref| + 2^-14 A with A = sum_j p_j |v_j| / sum_j p_j (float64).  The first term is
the bf16 rounding of the output; the second covers fp32 accumulation, ex2.approx and the lazy rescale, and it
scales with the magnitudes that are summed instead of sitting at a fixed floor (random data at 65536 keys has
|out| ~ 1/256, where a fixed 2e-3 floor would let a dropped 64-key tile through).
"""
from __future__ import annotations

import numpy as np

from .bf16 import bf16_round

HEAD_DIM = 128
SCALE = float(np.float32(1.0) / np.sqrt(np.float32(HEAD_DIM)))   # the kernels' 1.0f / sqrtf(128.f)
REL = 2.0 ** -8
ABS_A = 2.0 ** -14


# ---------------------------------------------------------------- bit-exact parts


def reduce_planes(planes: np.ndarray) -> np.ndarray:
    """split-K planes [splits][...] fp32 -> bf16 values: 0 + p0 + p1 + ... in fp32, then one rounding"""
    acc = np.zeros(planes.shape[1:], np.float32)
    for p in planes:
        acc = (acc + p.astype(np.float32)).astype(np.float32)
    return bf16_round(acc)


def split_exact(x: np.ndarray, splits: int, rng) -> np.ndarray:
    """fp32 planes [splits][...] whose fp32 sum in index order is exactly the bf16 values x: planes 0..S-2 are
    bf16(x * w) with 2^-6 <= |w| <= 1, the last one the exact remainder (every partial sum spans < 24 bits)."""
    x = np.asarray(x, np.float32)
    if splits == 1:
        return x[None].copy()
    w = rng.uniform(2.0 ** -6, 1.0, (splits - 1,) + x.shape) * rng.choice([-1.0, 1.0], (splits - 1,) + x.shape)
    parts = bf16_round((x[None] * w).astype(np.float32))
    last = x.astype(np.float64) - parts.astype(np.float64).sum(0)
    planes = np.concatenate([parts, last[None].astype(np.float32)])
    assert np.array_equal(planes[-1].astype(np.float64), last)
    assert np.array_equal(reduce_planes(planes), bf16_round(x)), "split is not exact"
    return planes


def rope(x: np.ndarray, cos: np.ndarray, sin: np.ndarray) -> np.ndarray:
    """rotate-half RoPE of x [..., 128] with cos/sin [..., 64] broadcastable; bit-exact with rope_kv_kernel and
    the decode prologue (__fmul_rn / __fsub_rn / __fadd_rn, then bf16)"""
    x = np.asarray(x, np.float32)
    x1, x2 = x[..., :64], x[..., 64:]
    return bf16_round(np.concatenate([x1 * cos - x2 * sin, x2 * cos + x1 * sin], axis=-1).astype(np.float32))


def unrope(y: np.ndarray, cos: np.ndarray, sin: np.ndarray) -> np.ndarray:
    """bf16 values whose RoPE is close to y (the inverse rotation, float64): how a test plants a post-RoPE key"""
    y = np.asarray(y, np.float64)
    c, s = cos.astype(np.float64), sin.astype(np.float64)
    lo, hi = y[..., :64], y[..., 64:]
    return bf16_round(np.concatenate([lo * c + hi * s, hi * c - lo * s], axis=-1).astype(np.float32))


# ---------------------------------------------------------------- float64 attention


def _scores(q, k):
    """q [R][G][128] . k [S][128] * scale -> [R][G][S] (float64, through BLAS)"""
    R, G, d = q.shape
    return (q.reshape(R * G, d) @ k.T).reshape(R, G, -1) * SCALE


def _pv(p, v):
    """p [R][G][S] @ v [S][128] -> [R][G][128]"""
    R, G, S = p.shape
    return (p.reshape(R * G, S) @ v).reshape(R, G, -1)


def attention(q, k, v, limit, key_weight=None, p_bf16=False):
    """Softmax attention in float64.  q [R][H][128], k, v [S][KVH][128]; row r sees keys 0..limit[r]-1.
    Returns (out, A), both [R][H][128].  key_weight [S] multiplies each key's softmax weight (0 drops a key,
    2 counts it twice) and p_bf16 rounds the unnormalised weights to bf16 before P.V: both exist for the
    mutation tests of the tolerance."""
    q = np.asarray(q, np.float64)
    k = np.asarray(k, np.float64)
    v = np.asarray(v, np.float64)
    R, H, _ = q.shape
    S, KVH, _ = k.shape
    G = H // KVH
    vis = np.arange(S)[None, :] < np.asarray(limit)[:, None]                     # [R][S]
    out = np.empty((R, H, HEAD_DIM))
    A = np.empty((R, H, HEAD_DIM))
    for kh in range(KVH):
        hs = slice(kh * G, (kh + 1) * G)
        s = np.where(vis[:, None, :], _scores(q[:, hs], k[:, kh]), -np.inf)
        p = np.exp(s - s.max(-1, keepdims=True))
        if key_weight is not None:
            p = p * np.asarray(key_weight, np.float64)[None, None, :]
        l = p.sum(-1, keepdims=True)
        pv = bf16_round(p.astype(np.float32)).astype(np.float64) if p_bf16 else p
        out[:, hs] = _pv(pv, v[:, kh]) / l
        A[:, hs] = _pv(p, np.abs(v[:, kh])) / l
    return out, A


def key_mass(q, k, limit, j):
    """[R][H] softmax weight of key j (0 where the row does not see it), float64"""
    q = np.asarray(q, np.float64)
    k = np.asarray(k, np.float64)
    R, H, _ = q.shape
    S, KVH, _ = k.shape
    G = H // KVH
    vis = np.arange(S)[None, :] < np.asarray(limit)[:, None]
    m = np.zeros((R, H))
    for kh in range(KVH):
        hs = slice(kh * G, (kh + 1) * G)
        s = np.where(vis[:, None, :], _scores(q[:, hs], k[:, kh]), -np.inf)
        p = np.exp(s - s.max(-1, keepdims=True))
        m[:, hs] = p[:, :, j] / p.sum(-1)
    return m


# ---------------------------------------------------------------- the tolerance


def excess(got, ref, A):
    """(|got - ref| - 2^-8 |ref|) / A; the tolerance holds where this is <= 2^-14"""
    got = np.asarray(got, np.float64)
    ref = np.asarray(ref, np.float64)
    d = np.abs(got - ref) - REL * np.abs(ref)
    with np.errstate(divide="ignore", invalid="ignore"):
        e = np.where(A > 0, d / np.where(A > 0, A, 1.0), np.where(got == ref, -np.inf, np.inf))
    return np.where(np.isnan(got), np.inf, e)


def within(got, ref, A):
    return excess(got, ref, A) <= ABS_A


def assert_within(got, ref, A, what=""):
    """asserts the tolerance everywhere; returns the worst (|got-ref| - 2^-8|ref|) / A"""
    e = excess(got, ref, A)
    bad = ~(e <= ABS_A)
    assert not bad.any(), (what, int(bad.sum()), float(np.max(e)), np.argwhere(bad)[:5].tolist())
    return float(np.max(e))


# ---------------------------------------------------------------- planted keys


def _assert_canary(mass, seen, vj, ref):
    """a planted key holds 10 %..90 % of the softmax mass of every head that sees it and its V differs from
    those rows' outputs by >= 1 in every dimension"""
    m = mass[seen]
    assert m.size and m.min() >= 0.1 and m.max() <= 0.9, (m.min(), m.max())
    diff = np.abs(np.asarray(ref, np.float64) - np.asarray(vj, np.float64)[None, None, :])   # [R][G][128]
    assert diff[seen].min() >= 1.0, float(diff[seen].min())


def plant_decode_key(q_rot, k, v, j, amp=8.0):
    """Decode: one query row per head, q_rot [H][128] (post-RoPE); k, v [ctx][KVH][128] with the new token at
    ctx-1.  Key j of every KV head gets a K whose score equals log(sum of the other keys' weights) in every head
    of its group (least-norm solution of Q u = t), so it holds ~half the mass, and V = +-amp.  Returns new
    (k, v); the caller checks the result with check_decode_canary."""
    k = np.array(k, np.float32)
    v = np.array(v, np.float32)
    ctx, KVH, _ = k.shape
    H = q_rot.shape[0]
    G = H // KVH
    q = np.asarray(q_rot, np.float64)
    pattern = np.where((np.arange(HEAD_DIM) // 3) % 2 == 0, amp, -amp).astype(np.float32)
    others = np.arange(ctx) != j
    for kh in range(KVH):
        Q = q[kh * G:(kh + 1) * G]                                                  # [G][128]
        s = (Q @ k[others, kh].astype(np.float64).T) * SCALE                       # [G][ctx-1]
        mx = s.max(-1)
        t = (mx + np.log(np.exp(s - mx[:, None]).sum(-1))) / SCALE                  # target q.u per head
        u = Q.T @ np.linalg.solve(Q @ Q.T, t) if G > 1 else Q[0] * (t[0] / (Q[0] @ Q[0]))
        k[j, kh] = bf16_round(u.astype(np.float32))
        v[j, kh] = pattern
    return k, v


def check_decode_canary(q_rot, k, v, j, ref):
    """the planted-key conditions for key j of a decode row: q_rot, ref [H][128]"""
    mass = key_mass(np.asarray(q_rot)[None], k, [k.shape[0]], j)               # [1][H]
    G = q_rot.shape[0] // k.shape[1]
    for kh in range(k.shape[1]):
        hs = slice(kh * G, (kh + 1) * G)
        _assert_canary(mass[:, hs], np.ones((1, G), bool), v[j, kh], np.asarray(ref)[None, hs])


def plant_prefill_keys(q, pos, k, v, keys, beta=8.0, amp=8.0, future_lead=12.0):
    """Prefill: q [R][H][128] rows at absolute positions pos[R]; k, v [S][KVH][128].  Canary c at key keys[c]
    lives in dimension c alone: that dimension is zeroed in every other key, the canary's K is beta * e_c and its
    V = +-amp (a pattern per canary).  Every row that sees it gets q[c] so that its score equals log(sum of the
    non-canary weights) -- with m canaries visible each holds 1 / (m + 1) of the mass (diagonal canary: key ==
    the row's own position); the row one position before it gets a score future_lead above that (future
    canary: its reference weight is 0, a leak dominates the output).  At most 5 canaries.  Returns (q, k, v)."""
    assert len(keys) <= 5
    q = np.array(q, np.float32)
    k = np.array(k, np.float32)
    v = np.array(v, np.float32)
    pos = np.asarray(pos)
    n = len(keys)
    q[:, :, :n] = 0.0
    k[:, :, :n] = 0.0
    keys = list(keys)
    others = np.ones(k.shape[0], np.float64)
    others[keys] = 0.0
    for c, j in enumerate(keys):
        k[j] = 0.0
        k[j, :, c] = beta
        v[j] = np.where(((np.arange(HEAD_DIM) >> c) & 1) == 0, amp, -amp)[None, :]
    R, H, _ = q.shape
    G = H // k.shape[1]
    # log of the non-canary weight sum of every (row, head): canary dims of q are 0 here, so their scores are 0
    logz = np.empty((R, H))
    kk = k.astype(np.float64)
    for kh in range(k.shape[1]):
        hs = slice(kh * G, (kh + 1) * G)
        s = _scores(q[:, hs].astype(np.float64), kk[:, kh])
        s = np.where((np.arange(k.shape[0])[None, :] <= pos[:, None])[:, None, :] & (others > 0)[None, None, :],
                     s, -np.inf)
        mx = s.max(-1)
        logz[:, hs] = mx + np.log(np.exp(s - mx[..., None]).sum(-1))
    for c, j in enumerate(keys):
        t = np.where(pos[:, None] >= j, logz, np.where(pos[:, None] == j - 1, logz + future_lead, 0.0))
        assert np.isfinite(t).all(), "a row that sees a planted key must also see an unplanted one"
        q[:, :, c] = bf16_round((t / (beta * SCALE)).astype(np.float32))
    return q, k, v


def check_prefill_canaries(q, pos, k, v, keys, ref):
    """the planted-key conditions on the reference of plant_prefill_keys' data"""
    pos = np.asarray(pos)
    limit = pos + 1
    G = q.shape[1] // k.shape[1]
    for j in keys:
        mass = key_mass(q, k, limit, j)
        seen = np.broadcast_to((pos >= j)[:, None], mass.shape)
        if not seen.any():
            continue
        for kh in range(k.shape[1]):
            hs = slice(kh * G, (kh + 1) * G)
            _assert_canary(mass[:, hs], seen[:, hs], v[j, kh], np.asarray(ref)[:, hs])
