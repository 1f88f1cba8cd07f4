"""Long contexts on the GPU: Llama-3.1 presets with prompts of 40K to 120K tokens (max_pages_per_seq up to 4096).

  * parity against tests/torch_oracle.py (bf16 rounding points), teacher-forced over prompt + engine tokens, with
    the attention of the oracle computed in query blocks (a [heads][T][S] score tensor would need ~20 GB here);
  * bit-identical results under chunked prefill, a prefix-cache hit, batching beside short sequences and a rerun;
  * the context limit at max_pages_per_seq * 32 tokens;
  * step uploads that follow the pages in use, not max_pages_per_seq;
  * the wgmma prefill attention kernel over 65536 keys.
"""
import ctypes

import numpy as np
import pytest

from agentcontrolplane_b200 import _lib
from agentcontrolplane_b200.engine import Engine
from oracle.bf16 import bf16_round_to_bits, bits_to_f32
from llama31_presets import LLAMA31

pytestmark = pytest.mark.gpu

SEED = 0xACB200
VOCAB = 128256


def _prompt(n, seed):
    rng = np.random.default_rng(seed)
    return [128000] + [int(t) for t in rng.integers(0, 256, size=n - 1)]


def _engine(model, ctx_tokens, max_batch=8, mtps=8192, pages_per_seq=4096, prefix_cache=False):
    """ctx_tokens: the tokens of every sequence of the test together (the KV pool is sized to them)"""
    pages = (ctx_tokens + 31) // 32 + 16 + max_batch
    return Engine({"model": model, "max_batch": max_batch, "kv_pages": pages, "max_tokens_per_step": mtps,
                   "max_pages_per_seq": pages_per_seq, "prefix_cache": prefix_cache})


def _run(eng, model, prompts, n_new, logits=True):
    ts = [eng.submit({"model": model, "max_tokens": n_new,
                      "acp": {"prompt_token_ids": p, "return_logits": n_new if logits else 0}}) for p in prompts]
    out = []
    for t in ts:
        assert eng.wait(t, 900000)
        lg = eng.logits(t, n_new, VOCAB) if logits else None
        st, body = eng.result(t)
        assert st == 200, body
        out.append((body["acp"]["token_ids"], lg))
    return out


# ---------------------------------------------------------------- parity


def _teacher_forced_logits(weights, tokens, n_last):
    """fp32 logits of the last n_last positions of `tokens`, with TorchLlamaOracle's rounding points; attention is
    computed per block of queries over the keys the block can see, the MLP per block of rows."""
    import torch
    from torch_oracle import TorchLlamaOracle, _mm
    o = TorchLlamaOracle(weights)
    c, dev, _r = o.cfg, weights.device, o._r
    toks = torch.as_tensor(tokens, dtype=torch.int64, device=dev)
    T = toks.numel()
    pos = torch.arange(T, device=dev)
    x = weights.embed[toks].to(torch.float32)
    scale = 1.0 / np.sqrt(c.head_dim)
    G = c.heads // c.kv_heads
    qb = max(64, min(2048, (1 << 31) // (c.heads * T * 4)))   # query block: <= 2 GiB of fp32 scores
    rb = 4096                                                 # row block of the projections
    with torch.no_grad():
        for L in weights.layers:
            attn = torch.empty(T, c.q_dim, device=dev)
            K = torch.empty(T, c.kv_heads, c.head_dim, device=dev)
            V = torch.empty_like(K)
            Q = torch.empty(T, c.heads, c.head_dim, device=dev)
            for r0 in range(0, T, rb):
                r1 = min(T, r0 + rb)
                qkv = _r(_mm(o._rmsnorm(x[r0:r1], L["attn_norm"]), L["wqkv"]))
                n = r1 - r0
                Q[r0:r1] = o._rope(qkv[:, :c.q_dim].reshape(n, c.heads, c.head_dim), pos[r0:r1])
                K[r0:r1] = o._rope(qkv[:, c.q_dim:c.q_dim + c.kv_dim].reshape(n, c.kv_heads, c.head_dim), pos[r0:r1])
                V[r0:r1] = qkv[:, c.q_dim + c.kv_dim:].reshape(n, c.kv_heads, c.head_dim)
            Kh = K.permute(1, 0, 2)                                                 # [kvh][S][d]
            Vh = V.permute(1, 0, 2)
            for q0 in range(0, T, qb):
                q1 = min(T, q0 + qb)
                q = Q[q0:q1].permute(1, 0, 2).reshape(c.kv_heads, G * (q1 - q0), c.head_dim)   # [kvh][G*blk][d]
                s = torch.matmul(q, Kh[:, :q1].transpose(1, 2)) * scale                      # [kvh][G*blk][S]
                s = s.view(c.kv_heads, G, q1 - q0, q1)
                causal = torch.arange(q1, device=dev)[None, :] <= pos[q0:q1, None]
                s = s.masked_fill(~causal[None, None], float("-inf"))
                p = torch.exp(s - s.max(dim=-1, keepdim=True).values)
                a = torch.matmul(p.view(c.kv_heads, G * (q1 - q0), q1), Vh[:, :q1])          # [kvh][G*blk][d]
                a = a.view(c.kv_heads, G, q1 - q0, c.head_dim) / p.sum(dim=-1, keepdim=True)
                attn[q0:q1] = a.permute(2, 0, 1, 3).reshape(q1 - q0, c.q_dim)
                del s, p, a
            attn = _r(attn)
            for r0 in range(0, T, rb):
                r1 = min(T, r0 + rb)
                xr = _r(x[r0:r1] + _r(_mm(attn[r0:r1], L["wo"])))
                gu = _r(_mm(o._rmsnorm(xr, L["ffn_norm"]), L["wgu"]))
                g, u = gu[:, :c.ffn], gu[:, c.ffn:]
                act = _r(g / (1.0 + torch.exp(-g)))
                x[r0:r1] = _r(xr + _r(_mm(_r(act * u), L["wdown"])))
            del attn, K, V, Q, Kh, Vh
        xf = o._rmsnorm(x[T - n_last:], weights.final_norm)
        return _mm(xf, weights.lm_head).cpu().numpy()


@pytest.mark.parametrize("model,prompt_len", [("tiny-3.1", 120000), ("llama-3.1-8b-l2", 65536)])
def test_long_prompt_matches_the_bf16_oracle(model, prompt_len):
    import torch
    from torch_oracle import TorchWeights
    n_new = 8
    prompt = _prompt(prompt_len, prompt_len)
    with _engine(model, prompt_len + n_new) as eng:
        (got, lg), = _run(eng, model, [prompt], n_new)
    assert len(got) == n_new, got      # random byte tokens: no end-of-turn in 8 steps
    weights = TorchWeights(LLAMA31[model], SEED, device="cuda:0")
    ref = _teacher_forced_logits(weights, prompt + got[:-1], n_new)
    del weights
    torch.cuda.empty_cache()
    worst = 0.0
    for j in range(n_new):
        std = float(np.std(ref[j]))
        tol = max(3e-2, 0.08 * std)
        d = float(np.max(np.abs(lg[j] - ref[j])))
        worst = max(worst, d / std)
        assert d < tol, (model, j, d, tol)
        want = int(np.argmax(ref[j]))
        if got[j] != want:
            top2 = np.partition(ref[j], -2)[-2:]
            assert top2[1] - top2[0] < 2 * tol, (model, j, got, want)   # near-tie policy (DESIGN.md §5)
    print(f"{model} at {prompt_len} tokens: max |logit diff| vs bf16 oracle = {worst:.4f} logit std")


# ---------------------------------------------------------------- invariants at ~40K tokens

INV_MODEL, INV_LEN, INV_NEW = "tiny-3.1", 40000, 16


@pytest.fixture(scope="module")
def alone():
    prompt = _prompt(INV_LEN, 7)
    with _engine(INV_MODEL, INV_LEN + INV_NEW, mtps=INV_LEN) as eng:
        out = _run(eng, INV_MODEL, [prompt], INV_NEW)[0]
        again = _run(eng, INV_MODEL, [prompt], INV_NEW)[0]
        assert eng.stats()["prefill_steps"] == 2      # one shot each
    return prompt, out, again


def _same(a, b):
    assert a[0] == b[0]
    assert np.array_equal(a[1], b[1])


def test_rerun_is_bit_identical(alone):
    _, out, again = alone
    _same(out, again)


def test_chunked_prefill_equals_single_shot(alone):
    prompt, out, _ = alone
    with _engine(INV_MODEL, INV_LEN + INV_NEW, mtps=2048) as eng:
        got = _run(eng, INV_MODEL, [prompt], INV_NEW)[0]
        assert eng.stats()["prefill_steps"] == (INV_LEN + 2047) // 2048
    _same(got, out)


def test_prefix_cache_hit_equals_cold_run(alone):
    prompt, out, _ = alone
    with _engine(INV_MODEL, 2 * (INV_LEN + INV_NEW), mtps=INV_LEN, prefix_cache=True) as eng:
        cold = _run(eng, INV_MODEL, [prompt], INV_NEW)[0]
        before = eng.stats()["prefill_tokens"]
        hit = _run(eng, INV_MODEL, [prompt], INV_NEW)[0]
        assert eng.stats()["prefill_tokens"] - before < INV_LEN // 2    # the cached prefix was reused
    _same(cold, out)
    _same(hit, out)


def test_long_sequence_beside_63_short_ones(alone):
    prompt, out, _ = alone
    shorts = [_prompt(300 + 7 * i, 100 + i) for i in range(63)]
    with _engine(INV_MODEL, INV_LEN + INV_NEW + 63 * 800, max_batch=64, mtps=INV_LEN) as eng:
        res = _run(eng, INV_MODEL, [prompt] + shorts, INV_NEW)
    _same(res[0], out)


# ---------------------------------------------------------------- limits and uploads


def test_context_limit_follows_max_pages_per_seq():
    with _engine(INV_MODEL, 100000 + 64) as eng:
        got, _ = _run(eng, INV_MODEL, [_prompt(100000, 3)], 4, logits=False)[0]
        assert len(got) == 4
        st, body = eng.complete({"model": INV_MODEL, "max_tokens": 1,
                                 "acp": {"prompt_token_ids": _prompt(4096 * 32, 4)}}, 60000)
        assert st == 400 and body["error"]["type"] == "context_length_exceeded", body


def test_step_uploads_follow_the_pages_in_use():
    prompts = [_prompt(1500 + 300 * i, 40 + i) for i in range(8)]
    runs = {}
    for pps in (256, 4096):
        with _engine(INV_MODEL, 8 * 4200, pages_per_seq=pps, mtps=2048) as eng:
            # one request at a time: the same steps in both engines (concurrent arrivals batch by timing)
            toks = [_run(eng, INV_MODEL, [p], 12, logits=False)[0][0] for p in prompts]
            s = eng.stats()
            runs[pps] = (toks, s["prefill_steps"], s["decode_steps"], s["h2d_bytes"])
    assert runs[256] == runs[4096], runs


# ---------------------------------------------------------------- kernel


def test_prefill_attention_kernel_over_65536_keys():
    """256 queries at the end of a 65536-key context against the float64 reference and tolerance of
    oracle/attention_oracle.py, with planted keys (at the first key, at 32767 | 32768 -- a page and 64-key tile
    boundary -- and on the first query's diagonal) that a dropped or misread key, page or tile would move by ~1"""
    from oracle import attention_oracle as ao
    heads, kv_heads, q_len, ctx = 32, 8, 256, 65536
    rng = np.random.default_rng(65536)
    q = bits_to_f32(bf16_round_to_bits(rng.standard_normal((q_len, heads, 128)).astype(np.float32)))
    k = bits_to_f32(bf16_round_to_bits(rng.standard_normal((ctx, kv_heads, 128)).astype(np.float32)))
    v = bits_to_f32(bf16_round_to_bits(rng.standard_normal((ctx, kv_heads, 128)).astype(np.float32)))
    pos = np.arange(ctx - q_len, ctx)
    keys = [0, 32767, 32768, ctx - q_len + 1]
    q, k, v = ao.plant_prefill_keys(q, pos, k, v, keys)
    q, k, v = (bf16_round_to_bits(x) for x in (q, k, v))
    lib = _lib.load()
    u16p = ctypes.POINTER(ctypes.c_uint16)
    out = np.zeros((q_len, heads, 128), np.uint16)
    ms = ctypes.c_float(0)
    lib.acp_kernel_attn_prefill.argtypes = [u16p, u16p, u16p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                            ctypes.c_int, u16p, ctypes.c_int, ctypes.POINTER(ctypes.c_float)]
    rc = lib.acp_kernel_attn_prefill(q.ctypes.data_as(u16p), k.ctypes.data_as(u16p), v.ctypes.data_as(u16p), heads,
                                     kv_heads, q_len, ctx, 1, out.ctypes.data_as(u16p), 0, ctypes.byref(ms))
    assert rc == 0
    q, k, v = (bits_to_f32(x) for x in (q, k, v))
    ref, A = ao.attention(q, k, v, pos + 1)
    ao.check_prefill_canaries(q, pos, k, v, keys, ref)
    worst = ao.assert_within(bits_to_f32(out), ref, A)
    print(f"prefill over 65536 keys: worst (|got-ref| - 2^-8|ref|)/A = {worst:.3g}")
