"""FP8 (e4m3) numerics of the engine's `-fp8` presets, numpy only: the e4m3 codec, the row quantiser,
the quantised synthetic weights and a forward pass whose four layer projections run per the FP8
contract of DESIGN.md §5.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

The contract, step for step (every function below restates one line of it):
    row quantiser (weights and activations), x = one row of fp32 values (bf16 values widened exactly):
        amax = max|x|
        s    = fp32(amax / 448)             (s = 1 when amax == 0)
        code = e4m3_rne(clamp(fp32(x / s), -448, 448))
    weights:      one scale per output row s_w[m] (quantised once at init)
    activations:  one scale per token s_x[n], from the bf16 xn / attn / h rows of the bf16 path
    GEMM:         acc[n][m] = sum_k code_w[m][k] * code_x[n][k]   (every product is exact)
                  y[n][m]   = fp32(fp32(acc * s_w[m]) * s_x[n])
                  then the bf16 path's own rounding point (bf16 mode) or none (fp32 mode)
Embeddings, norms, attention, the KV cache, the residual stream and the LM head stay bf16.
"""
from __future__ import annotations

import dataclasses

import numpy as np

from .llama_oracle import PRESETS, LlamaConfig, LlamaOracle, shared_weights

E4M3_MAX = np.float32(448.0)


def _decode_table() -> np.ndarray:
    """fp32 value of every e4m3fn code (0x7F / 0xFF are NaN; there is no infinity)."""
    c = np.arange(256, dtype=np.uint32)
    sign = np.where(c & 0x80, -1.0, 1.0)
    e = (c >> 3) & 0xF
    m = (c & 0x7).astype(np.float64)
    mag = np.where(e == 0, m * 2.0 ** -9, (1.0 + m / 8.0) * 2.0 ** (e.astype(np.float64) - 7.0))
    v = (sign * mag).astype(np.float32)
    v[(c & 0x7F) == 0x7F] = np.nan
    return v


DECODE = _decode_table()


def e4m3_decode(codes: np.ndarray) -> np.ndarray:
    return DECODE[np.asarray(codes, dtype=np.uint8)]


def e4m3_encode(x: np.ndarray) -> np.ndarray:
    """fp32 in [-448, 448] -> e4m3fn codes, round to nearest, ties to even (what cvt.rn.satfinite.e4m3x2.f32
    and torch's .to(float8_e4m3fn) do).  Out-of-range input is a caller error: the row quantiser clamps first.
      |x| <  2^-6 (subnormal codes 0..8):  code = rint(|x| * 2^9)           (exact scaling, ties to even)
      |x| >= 2^-6:  round the fp32 mantissa to 3 bits (ties to even; a carry bumps the exponent), then
                    code = (fp32 exponent - 127 + 7) << 3 | mantissa"""
    x = np.asarray(x, dtype=np.float32)
    if np.any(np.isnan(x)) or np.any(np.abs(x) > E4M3_MAX):
        raise ValueError("e4m3_encode: input outside [-448, 448]")
    a = np.abs(x)
    sub = np.rint(a * np.float32(512.0)).astype(np.uint32)
    bits = a.view(np.uint32)
    rounded = (bits + np.uint32(0x7FFFF) + ((bits >> 20) & np.uint32(1))) >> 20
    normal = rounded.astype(np.int64) - (120 << 3)
    code = np.where(a < np.float32(2.0 ** -6), sub, np.maximum(normal, 0)).astype(np.uint8)
    return code | np.where(np.signbit(x), 0x80, 0).astype(np.uint8)


def quantize_rows(x: np.ndarray):
    """The row quantiser over the last axis: (codes uint8, scales fp32 [rows])."""
    x = np.asarray(x, dtype=np.float32)
    amax = np.max(np.abs(x), axis=-1)
    s = (amax / E4M3_MAX).astype(np.float32)
    s = np.where(amax == 0, np.float32(1.0), s).astype(np.float32)
    q = np.clip((x / s[..., None]).astype(np.float32), -E4M3_MAX, E4M3_MAX)
    return e4m3_encode(q), s


def fp8_matmul(x_codes, s_x, w_codes, s_w, w_values=None) -> np.ndarray:
    """y[n][m] = fp32(fp32(acc * s_w[m]) * s_x[n]), acc = the EXACT sum of code products rounded once to fp32
    (products are multiples of 2^-18 below 2^18, so every float64 partial sum is exact).  w_values: the
    float64 values of w_codes when the caller has them."""
    wv = e4m3_decode(w_codes).astype(np.float64) if w_values is None else w_values
    acc = (e4m3_decode(x_codes).astype(np.float64) @ wv.T).astype(np.float32)
    return ((acc * s_w[None, :]).astype(np.float32) * s_x[:, None]).astype(np.float32)


@dataclasses.dataclass(frozen=True)
class Fp8LlamaConfig(LlamaConfig):
    """A preset whose four layer projections run in FP8; shapes and seeded weights are the base preset's."""
    base: str = ""


FP8_BASES = ("tiny", "tiny-g2", "tiny-g8", "llama-3-8b-l2", "llama-3-8b")
FP8_PRESETS = {
    f"{b}-fp8": Fp8LlamaConfig(**{**dataclasses.asdict(PRESETS[b]), "name": f"{b}-fp8"}, base=b) for b in FP8_BASES
}


class QuantWeights:
    """Row-quantised copies (codes, s_w) of a preset's synthetic bf16 projection weights, per the contract; the
    engine's synthetic `-fp8` presets quantise the same bf16 tensors on the GPU at init.  Logical row order
    ([q; k; v], [gate; up]); the engine's tiled layout only permutes rows, which carry their own scales."""

    def __init__(self, cfg: Fp8LlamaConfig, seed: int):
        self.bf16 = shared_weights(PRESETS[cfg.base], seed)
        self._cache = {}

    def _q(self, key, mat_fn):
        if key not in self._cache:
            self._cache[key] = quantize_rows(mat_fn())
        return self._cache[key]

    def decoded(self, qw):
        """float64 values of a quantised matrix's codes (cached: the forward pass reuses them every step)"""
        key = id(qw[0])
        if key not in self._cache:
            self._cache[key] = e4m3_decode(qw[0]).astype(np.float64)
        return self._cache[key]

    def wqkv(self, l):
        return self._q(("qkv", l), lambda: self.bf16.wqkv(l))

    def wo(self, l):
        return self._q(("o", l), lambda: self.bf16.wo(l))

    def wgu(self, l):
        return self._q(("gu", l), lambda: self.bf16.wgu(l))

    def wdown(self, l):
        return self._q(("down", l), lambda: self.bf16.wdown(l))


_QW_CACHE: dict = {}


def shared_quant_weights(cfg: Fp8LlamaConfig, seed: int) -> QuantWeights:
    key = (cfg, seed)
    if key not in _QW_CACHE:
        _QW_CACHE[key] = QuantWeights(cfg, seed)
    return _QW_CACHE[key]


class Fp8LlamaOracle(LlamaOracle):
    """LlamaOracle with the four layer projections per the FP8 contract (dense presets only).  mode 'bf16'
    keeps every bf16 rounding point of the bf16 oracle; 'fp32' has none."""

    def __init__(self, cfg: Fp8LlamaConfig, seed: int, mode: str = "bf16"):
        assert isinstance(cfg, Fp8LlamaConfig) and cfg.experts == 0
        super().__init__(cfg, seed, mode=mode, weights=shared_weights(PRESETS[cfg.base], seed))
        self.qw = shared_quant_weights(cfg, seed)

    def _proj(self, x, qw):
        codes, s_x = quantize_rows(x)
        w_codes, s_w = qw
        return self._r(fp8_matmul(codes, s_x, w_codes, s_w, self.qw.decoded(qw)))

    def forward(self, tokens, all_logits: bool = False):
        c = self.cfg
        toks = np.asarray(tokens, dtype=np.int64)
        T = len(toks)
        pos = np.arange(self.pos, self.pos + T)
        x = self.w.embed_rows(toks)
        scale = np.float32(1.0 / np.sqrt(c.head_dim))
        group = c.heads // c.kv_heads
        for l in range(c.layers):
            xn = self._rmsnorm(x, self.w.attn_norm(l))
            qkv = self._proj(xn, self.qw.wqkv(l))
            q = qkv[:, :c.q_dim].reshape(T, c.heads, c.head_dim)
            k = qkv[:, c.q_dim:c.q_dim + c.kv_dim].reshape(T, c.kv_heads, c.head_dim)
            v = qkv[:, c.q_dim + c.kv_dim:].reshape(T, c.kv_heads, c.head_dim)
            q = self._rope(q, pos)
            k = self._rope(k, pos)
            self.k[l] = np.concatenate([self.k[l], k], axis=0)
            self.v[l] = np.concatenate([self.v[l], v], axis=0)
            K, V = self.k[l], self.v[l]
            S = K.shape[0]
            attn = np.empty((T, c.heads, c.head_dim), np.float32)
            causal = (np.arange(S)[None, :] <= pos[:, None])
            for h in range(c.heads):
                kh = h // group
                s = (q[:, h, :] @ K[:, kh, :].T) * scale
                s = np.where(causal, s, -np.inf)
                m = s.max(axis=-1, keepdims=True)
                p = np.exp(s - m)
                attn[:, h, :] = (p @ V[:, kh, :]) / p.sum(axis=-1, keepdims=True)
            attn = self._r(attn.reshape(T, c.q_dim))
            o = self._proj(attn, self.qw.wo(l))
            x = self._r(x + o)
            xn2 = self._rmsnorm(x, self.w.ffn_norm(l))
            gu = self._proj(xn2, self.qw.wgu(l))
            g, u = gu[:, :c.ffn], gu[:, c.ffn:]
            act = self._r(g / (np.float32(1.0) + np.exp(-g)))
            h_ = self._r(act * u)
            d = self._proj(h_, self.qw.wdown(l))
            x = self._r(x + d)
        self.pos += T
        xf = self._rmsnorm(x if all_logits else x[-1:], self.w.final_norm())
        return (xf @ self.w.lm_head().T).astype(np.float32)
