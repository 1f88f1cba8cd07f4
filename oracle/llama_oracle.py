"""Numerical oracle for the local provider's transformer (Llama-3 architecture), numpy fp32.

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

The reference has NO numerics on this path: `LangchainClient.SendRequest`
(acp/internal/llmclient/langchaingo_client.go:83-115) hands the context window to
`llms.Model.GenerateContent` (:102, langchaingo v0.1.13, un-vendored) which POSTs it to a hosted
model.  What is restated here is therefore the PUBLISHED Llama-3 forward pass (RMSNorm eps 1e-5,
rotate-half RoPE theta 5e5, GQA attention, SwiGLU MLP, untied LM head) — pinned against HuggingFace
`transformers.LlamaForCausalLM` in fp32 by tests/golden/make_llama_golden.py (fixture
tests/golden/llama_tiny_golden.npz) — plus a `bf16` mode that rounds at exactly the points where
the CUDA engine (agentcontrolplane_b200/csrc/model.cu) stores bf16, so greedy token ids can be
compared bit-exactly.

bf16-mode rounding points (every arrow is a round-to-nearest-even to bf16):
    x  = E[tok]
    xn = g * bf16(x * rsqrt(mean(x^2)+eps))  -> bf16          (two roundings, like HF)
    qkv = xn @ Wqkv^T                        -> bf16
    q,k = rope(q,k) in fp32                  -> bf16
    a  = softmax(q k^T / sqrt(d)) v  (fp32)  -> bf16
    x  = x + bf16(a @ Wo^T)                  -> bf16
    gu = xn2 @ Wgu^T                         -> bf16
    h  = bf16(silu(g)) * u                   -> bf16
    x  = x + bf16(h @ Wd^T)                  -> bf16
    logits = rmsnorm(x) @ Wlm^T              (fp32, not rounded)
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from . import synth
from .bf16 import bf16_round, bits_to_f32


@dataclass(frozen=True)
class LlamaConfig:
    name: str
    hidden: int
    layers: int
    heads: int
    kv_heads: int
    ffn: int
    vocab: int = 128256
    head_dim: int = 128
    rope_theta: float = 500000.0
    eps: float = 1e-5
    w_std: float = 0.02
    max_pos: int = 8192
    # Llama-3.1 "llama3" RoPE frequency scaling: (factor, low_freq_factor, high_freq_factor,
    # original_max_position_embeddings) or None; same formula as csrc/model.cu rope_inv_freq()
    rope_scaling: tuple | None = None
    # Mixtral-style sparse mixture of experts: `experts` SwiGLU MLPs of width `ffn` per layer, top-2 routing
    # (0 = dense Llama MLP)
    experts: int = 0

    @property
    def q_dim(self):
        return self.heads * self.head_dim

    @property
    def kv_dim(self):
        return self.kv_heads * self.head_dim


PRESETS = {
    "tiny": LlamaConfig("tiny", hidden=512, layers=2, heads=4, kv_heads=1, ffn=1024),
    "tiny-g2": LlamaConfig("tiny-g2", hidden=512, layers=3, heads=4, kv_heads=2, ffn=1536),
    # the head grouping of one Llama-3-70B shard at TP=8 (8 query heads on 1 KV head)
    "tiny-g8": LlamaConfig("tiny-g8", hidden=1024, layers=2, heads=8, kv_heads=1, ffn=2048),
    "llama-3-8b-l2": LlamaConfig("llama-3-8b-l2", hidden=4096, layers=2, heads=32, kv_heads=8,
                                 ffn=14336),
    "llama-3-8b": LlamaConfig("llama-3-8b", hidden=4096, layers=32, heads=32, kv_heads=8, ffn=14336),
    "llama-3-70b": LlamaConfig("llama-3-70b", hidden=8192, layers=80, heads=64, kv_heads=8,
                               ffn=28672),
    # Mixtral-8x7B architecture (BASELINE config 4): 8 experts, top-2, rope theta 1e6.  The synthetic
    # presets keep the 128256-entry vocabulary of the synthetic tokenizer (a real checkpoint has 32000).
    "tiny-moe": LlamaConfig("tiny-moe", hidden=512, layers=2, heads=4, kv_heads=2, ffn=768, experts=8,
                            rope_theta=1000000.0),
    "mixtral-8x7b-l2": LlamaConfig("mixtral-8x7b-l2", hidden=4096, layers=2, heads=32, kv_heads=8, ffn=14336,
                                   experts=8, rope_theta=1000000.0),
    "mixtral-8x7b": LlamaConfig("mixtral-8x7b", hidden=4096, layers=32, heads=32, kv_heads=8, ffn=14336,
                                experts=8, rope_theta=1000000.0),
}


def rope_inv_freq(cfg: LlamaConfig) -> np.ndarray:
    """fp32 inverse frequencies, computed in double like csrc/model.cu rope_inv_freq(): plain
    theta^(-2i/d), then (rope_scaling) wavelengths above orig_max/low are slowed by `factor`, those
    between orig_max/high and orig_max/low are interpolated (transformers' "llama3" rope type)."""
    half = cfg.head_dim // 2
    f = cfg.rope_theta ** (-(np.arange(half, dtype=np.float64) * 2.0) / cfg.head_dim)
    if cfg.rope_scaling is not None:
        factor, low, high, orig = (float(v) for v in cfg.rope_scaling)
        wavelen = 2.0 * np.pi / f
        low_wl, high_wl = orig / low, orig / high
        smooth = (orig / wavelen - low) / (high - low)
        mid = (1.0 - smooth) * f / factor + smooth * f
        f = np.where(wavelen > low_wl, f / factor, np.where(wavelen < high_wl, f, mid))
    return f.astype(np.float32)


def rope_tables(cfg: LlamaConfig, max_pos: int):
    """cos/sin [max_pos][head_dim/2] fp32 — the same recipe as csrc/model.cu build_rope_table():
    inv_freq = fp32(theta^(-2i/d)) from double; angle = fp32(pos) * inv_freq (fp32 multiply);
    cos/sin evaluated in double on that fp32 angle, rounded to fp32."""
    half = cfg.head_dim // 2
    inv = rope_inv_freq(cfg)
    ang = (np.arange(max_pos, dtype=np.float32)[:, None] * inv[None, :]).astype(np.float32)
    return np.cos(ang.astype(np.float64)).astype(np.float32), np.sin(ang.astype(np.float64)).astype(
        np.float32)


def router_logits(x: np.ndarray, w: np.ndarray) -> np.ndarray:
    """fp32 router logits x[T][H] . w[E][H] in the ENGINE's summation order (csrc/moe.cu
    moe_router_kernel): 32 lanes, lane j accumulates the products of elements j, j+32, j+64, ... in
    that order (separately rounded multiply and add), then the lanes are folded 16, 8, 4, 2, 1."""
    T, H = x.shape
    E = w.shape[0]
    prod = (x.astype(np.float32)[:, None, :] * w.astype(np.float32)[None, :, :]).astype(np.float32)
    prod = prod.reshape(T, E, H // 32, 32)
    acc = np.zeros((T, E, 32), np.float32)
    for i in range(H // 32):
        acc = (acc + prod[:, :, i, :]).astype(np.float32)
    for half in (16, 8, 4, 2, 1):
        acc = (acc[:, :, :half] + acc[:, :, half:2 * half]).astype(np.float32)
    return acc[:, :, 0]


class Weights:
    """fp32 copies of the synthetic bf16 tensors (generated lazily per layer)."""

    def __init__(self, cfg: LlamaConfig, seed: int):
        self.cfg, self.seed = cfg, seed
        self._cache = {}

    def _mat(self, tid, rows, cols):
        key = (tid, rows, cols)
        if key not in self._cache:
            self._cache[key] = bits_to_f32(synth.synth_matrix(self.seed, tid, rows, cols,
                                                             self.cfg.w_std))
        return self._cache[key]

    def _gain(self, tid, n):
        key = (tid, n)
        if key not in self._cache:
            self._cache[key] = bits_to_f32(synth.synth_bits(self.seed, tid, n, 0.1, plus_one=True))
        return self._cache[key]

    def embed_rows(self, toks):
        return bits_to_f32(synth.synth_rows(self.seed, synth.TID_EMBED, np.asarray(toks),
                                            self.cfg.hidden, self.cfg.w_std))

    def lm_head(self):
        return self._mat(synth.TID_LM_HEAD, self.cfg.vocab, self.cfg.hidden)

    def final_norm(self):
        return self._gain(synth.TID_FINAL_NORM, self.cfg.hidden)

    def wqkv(self, l):
        c = self.cfg
        return self._mat(synth.layer_tid(l, synth.TID_WQKV), c.q_dim + 2 * c.kv_dim, c.hidden)

    def wo(self, l):
        return self._mat(synth.layer_tid(l, synth.TID_WO), self.cfg.hidden, self.cfg.q_dim)

    def wgu(self, l):
        return self._mat(synth.layer_tid(l, synth.TID_WGU), 2 * self.cfg.ffn, self.cfg.hidden)

    def wdown(self, l):
        return self._mat(synth.layer_tid(l, synth.TID_WDOWN), self.cfg.hidden, self.cfg.ffn)

    def router(self, l):
        return self._mat(synth.layer_tid(l, synth.TID_ROUTER), self.cfg.experts, self.cfg.hidden)

    def expert_gu(self, l, e):
        return self._mat(synth.expert_tid(l, e, synth.TID_EXPERT_GU), 2 * self.cfg.ffn, self.cfg.hidden)

    def expert_down(self, l, e):
        return self._mat(synth.expert_tid(l, e, synth.TID_EXPERT_DOWN), self.cfg.hidden, self.cfg.ffn)

    def attn_norm(self, l):
        return self._gain(synth.layer_tid(l, synth.TID_ATTN_NORM), self.cfg.hidden)

    def ffn_norm(self, l):
        return self._gain(synth.layer_tid(l, synth.TID_FFN_NORM), self.cfg.hidden)


_WEIGHTS_CACHE: dict = {}


def shared_weights(cfg: LlamaConfig, seed: int) -> Weights:
    """One Weights object per (config, seed): the 128256-row LM head takes seconds to generate."""
    key = (cfg, seed)
    if key not in _WEIGHTS_CACHE:
        _WEIGHTS_CACHE[key] = Weights(cfg, seed)
    return _WEIGHTS_CACHE[key]


class LlamaOracle:
    """One sequence, KV cached.  mode='bf16' mirrors the engine's rounding points, 'fp32' has none
    (that mode is what is pinned against HuggingFace)."""

    def __init__(self, cfg: LlamaConfig, seed: int, mode: str = "bf16", weights: Weights | None = None):
        assert mode in ("bf16", "fp32")
        self.cfg, self.mode = cfg, mode
        self.w = weights or shared_weights(cfg, seed)
        self.cos, self.sin = rope_tables(cfg, cfg.max_pos)
        self.k = [np.zeros((0, cfg.kv_heads, cfg.head_dim), np.float32) for _ in range(cfg.layers)]
        self.v = [np.zeros((0, cfg.kv_heads, cfg.head_dim), np.float32) for _ in range(cfg.layers)]
        self.pos = 0

    def _r(self, x):
        return bf16_round(x) if self.mode == "bf16" else x.astype(np.float32)

    def _rmsnorm(self, x, g):
        var = np.mean(x.astype(np.float32) ** 2, axis=-1, keepdims=True, dtype=np.float32)
        rstd = (1.0 / np.sqrt(var + np.float32(self.cfg.eps))).astype(np.float32)
        return self._r(g * self._r(x * rstd))

    def _rope(self, x, pos):
        # x: [T][H][d]; rotate-half convention (HF Llama): pairs (i, i + d/2)
        half = self.cfg.head_dim // 2
        c = self.cos[pos][:, None, :]
        s = self.sin[pos][:, None, :]
        x1, x2 = x[..., :half], x[..., half:]
        return self._r(np.concatenate([x1 * c - x2 * s, x2 * c + x1 * s], axis=-1))

    def forward(self, tokens, all_logits: bool = False):
        """Append `tokens` to the sequence; return fp32 logits of the last (or every) position."""
        c = self.cfg
        toks = np.asarray(tokens, dtype=np.int64)
        T = len(toks)
        pos = np.arange(self.pos, self.pos + T)
        x = self.w.embed_rows(toks)  # bf16 values
        scale = np.float32(1.0 / np.sqrt(c.head_dim))
        group = c.heads // c.kv_heads
        for l in range(c.layers):
            xn = self._rmsnorm(x, self.w.attn_norm(l))
            qkv = self._r(xn @ self.w.wqkv(l).T)
            q = qkv[:, :c.q_dim].reshape(T, c.heads, c.head_dim)
            k = qkv[:, c.q_dim:c.q_dim + c.kv_dim].reshape(T, c.kv_heads, c.head_dim)
            v = qkv[:, c.q_dim + c.kv_dim:].reshape(T, c.kv_heads, c.head_dim)
            q = self._rope(q, pos)
            k = self._rope(k, pos)
            self.k[l] = np.concatenate([self.k[l], k], axis=0)
            self.v[l] = np.concatenate([self.v[l], v], axis=0)
            K, V = self.k[l], self.v[l]  # [S][kvh][d]
            S = K.shape[0]
            attn = np.empty((T, c.heads, c.head_dim), np.float32)
            causal = (np.arange(S)[None, :] <= pos[:, None])  # [T][S]
            for h in range(c.heads):
                kh = h // group
                s = (q[:, h, :] @ K[:, kh, :].T) * scale  # [T][S]
                s = np.where(causal, s, -np.inf)
                m = s.max(axis=-1, keepdims=True)
                p = np.exp(s - m)
                attn[:, h, :] = (p @ V[:, kh, :]) / p.sum(axis=-1, keepdims=True)
            attn = self._r(attn.reshape(T, c.q_dim))
            o = self._r(attn @ self.w.wo(l).T)
            x = self._r(x + o)
            xn2 = self._rmsnorm(x, self.w.ffn_norm(l))
            if c.experts:
                d = self._moe(xn2, l)
            else:
                gu = self._r(xn2 @ self.w.wgu(l).T)
                g, u = gu[:, :c.ffn], gu[:, c.ffn:]
                act = self._r(g / (np.float32(1.0) + np.exp(-g)))
                h_ = self._r(act * u)
                d = self._r(h_ @ self.w.wdown(l).T)
            x = self._r(x + d)
        self.pos += T
        xf = self._rmsnorm(x if all_logits else x[-1:], self.w.final_norm())
        return (xf @ self.w.lm_head().T).astype(np.float32)

    def _moe(self, xn2, l):
        """Sparse MoE block of one layer (transformers MixtralSparseMoeBlock: softmax router, top-2,
        renormalised weights, SwiGLU experts), with the engine's rounding points in bf16 mode:
            r      = router_logits(xn2)   fp32, FIXED summation order (router_logits below) so that the
                                          engine and the oracle select the same experts bit for bit
            e0, e1 = the two largest logits (lowest index wins ties)
            w0, w1 = 1/(1+exp(r1-r0)), exp(r1-r0)/(1+exp(r1-r0))     (= softmax renormalised over the top 2)
            d_k    = bf16(h_k @ Wd_k^T),  h_k = bf16(bf16(silu(g)) * u),  [g|u] = bf16(xn2 @ Wgu_k^T)
            out    = bf16(w0*d_0 + w1*d_1)     (two fp32 products, one fp32 add, one rounding)
        The stages are the array-level functions of oracle/moe_oracle.py, which the kernel tests check one by one."""
        from . import moe_oracle
        c = self.cfg
        r = router_logits(xn2, self.w.router(l))
        idx, w = moe_oracle.top2(r)
        self.last_routing = (idx[:, 0], idx[:, 1], w[:, 0], w[:, 1])
        # closest call of the discrete routing so far: gap between the 2nd and 3rd largest router logit.  bf16
        # rounding noise UPSTREAM of the router (the engine and the oracle agree on the router arithmetic bit for
        # bit, not on every bit of its input) can flip the second expert when this gap is inside that noise.
        r3 = np.partition(r, -3, axis=1)
        self.min_router_gap = min(getattr(self, "min_router_gap", np.inf), float(np.min(r3[:, -2] - r3[:, -3])))
        return moe_oracle.moe_block(xn2, idx, w, lambda e: self.w.expert_gu(l, e), lambda e: self.w.expert_down(l, e),
                                    c.experts, self._r)

    def greedy(self, prompt, max_new: int, eos=(), force=None):
        """Greedy decode; returns (token ids, per-step (top1-top2) logit margins).
        `force` (optional list) teacher-forces emitted tokens (the engine's acp_force_tokens)."""
        out, margins = [], []
        logits = self.forward(prompt)[-1]
        for step in range(max_new):
            top2 = np.partition(logits, -2)[-2:]
            margins.append(float(top2[1] - top2[0]))
            tok = int(np.argmax(logits))  # lowest index on ties, like the fused arg-max epilogue
            if force is not None and step < len(force):
                tok = int(force[step])
            out.append(tok)
            if tok in eos or step == max_new - 1:
                break
            logits = self.forward([tok])[-1]
        return out, margins
