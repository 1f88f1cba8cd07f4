"""End-to-end parity of the CUDA engine (through the C ABI) against the numerical oracle:
token ids bit-exact under greedy decoding, logits within a stated tolerance."""
import numpy as np
import pytest

from agentcontrolplane_b200.engine import Engine
from oracle.llama_oracle import PRESETS, LlamaOracle

pytestmark = pytest.mark.gpu

SEED = 0xACB200
# |engine - oracle(bf16 mode)| on fp32 logits.  Both round to bf16 at the same points; what is
# left is fp32 summation order (tensor-core vs numpy) which can flip single bf16 roundings.  The bound
# is stated relative to the logit scale: 8 % of the standard deviation of the oracle's logit vector,
# never looser than LOGIT_ATOL absolute.
LOGIT_ATOL = 3e-2
LOGIT_RTOL = 8e-2


def logit_tol(ref):
    return max(LOGIT_ATOL, LOGIT_RTOL * float(np.std(ref)))


# Mixture of experts: routing is discrete.  When the oracle's own 2nd / 3rd router logits were closer than this
# anywhere on the sequence's path, upstream bf16 noise may legitimately pick another second expert in the engine;
# the continuations are then compared no further (measured router-input noise ~2e-3 at the tiny-moe preset).
ROUTER_GAP_TOL = 1e-2


def assert_tokens_match(got, want, margins, where="", tol=LOGIT_ATOL, router_gap=None):
    """Bit-exact token ids, with the stated near-tie policy (DESIGN.md §5): a mismatch is only
    tolerated at a step whose oracle top-1/top-2 logit margin is below 2*LOGIT_ATOL (either
    implementation may legitimately pick either candidate there); comparison stops at that step
    because the continuations differ from then on."""
    for i, (g, w) in enumerate(zip(got, want)):
        if g != w:
            if router_gap is not None and router_gap < ROUTER_GAP_TOL:
                return i
            assert margins[i] < 2 * tol, (where, i, got, want, margins, router_gap)
            return i
    assert len(got) == len(want), (where, got, want)
    return len(got)


def _tol_for(cfg):
    """near-tie tolerance of a preset: the logit std is w_std * sqrt(hidden) of a unit-normalised hidden state"""
    return max(LOGIT_ATOL, LOGIT_RTOL * cfg.w_std * float(np.sqrt(cfg.hidden)))


def _greedy(cfg, prompt, n_new):
    """oracle tokens, margins and (MoE presets) its closest router call on this sequence"""
    orc = LlamaOracle(cfg, SEED, mode="bf16")
    want, margins = orc.greedy(prompt, n_new, eos=(128001, 128008, 128009))
    return want, margins, getattr(orc, "min_router_gap", None)


def _prompt(rng, n):
    return [128000] + [int(t) for t in rng.integers(0, 256, size=n - 1)]


# tiny / tiny-g2: hidden 512, G = 4 / 2.  tiny-g8: the head grouping of a Llama-3-70B TP=8 shard (8 query
# heads on 1 KV head).  llama-3-8b-l2: the REAL Llama-3-8B width (hidden 4096, 32 q / 8 kv heads, ffn 14336,
# vocab 128256) at 2 layers, where the numpy oracle still finishes in seconds; full depth is covered by
# tests/test_fulldepth_gpu.py.
# tiny-moe: the Mixtral architecture (8 experts, top-2 routing, grouped expert GEMMs; csrc/moe.cu).
@pytest.fixture(scope="module", params=["tiny", "tiny-g2", "tiny-g8", "tiny-moe", "llama-3-8b-l2"])
def eng(request):
    e = Engine({"model": request.param, "max_batch": 64, "kv_pages": 512, "max_tokens_per_step": 1024})
    e.model_name = request.param
    yield e
    e.close()


def _run(eng, prompt, max_tokens, logits=0, force=None):
    req = {"model": eng.model_name, "max_tokens": max_tokens,
           "acp": {"prompt_token_ids": prompt, "return_logits": logits}}
    if force:
        req["acp"]["force_tokens"] = force
    t = eng.submit(req)
    assert eng.wait(t, 120000)
    lg = eng.logits(t, logits, 128256) if logits else None
    status, body = eng.result(t)
    assert status == 200, body
    return body["acp"]["token_ids"], lg, body


def test_single_sequence_matches_oracle(eng):
    cfg = PRESETS[eng.model_name]
    rng = np.random.default_rng(1)
    prompt = _prompt(rng, 45)
    n_new = 12
    toks, lg, body = _run(eng, prompt, n_new, logits=4)
    orc = LlamaOracle(cfg, SEED, mode="bf16")
    want, margins = orc.greedy(prompt, n_new, eos=(128001, 128008, 128009))
    # logits of the first sampled position (prefill) and three decode steps
    orc2 = LlamaOracle(cfg, SEED, mode="bf16")
    ref0 = orc2.forward(prompt)[-1]
    tol = logit_tol(ref0)
    assert np.max(np.abs(lg[0] - ref0)) < tol
    print("max |logit diff| prefill position:", float(np.max(np.abs(lg[0] - ref0))), "tolerance", tol)
    cur = want[0]
    for i in range(1, 4):
        ref = orc2.forward([cur])[-1]
        assert np.max(np.abs(lg[i] - ref)) < tol, i
        cur = want[i]
    assert_tokens_match(toks, want, margins, tol=tol, router_gap=getattr(orc, "min_router_gap", None))
    assert body["usage"]["prompt_tokens"] == len(prompt)


def test_batched_mixed_lengths_match_oracle(eng):
    """Many concurrent requests of different lengths: every sequence must produce exactly the
    tokens it produces alone (batch invariance) and the oracle's tokens."""
    cfg = PRESETS[eng.model_name]
    rng = np.random.default_rng(2)
    lens = [3, 17, 32, 33, 64, 65, 100, 130, 7, 257]
    prompts = [_prompt(rng, n) for n in lens]
    n_new = 6
    tickets = [eng.submit({"model": eng.model_name, "max_tokens": n_new,
                           "acp": {"prompt_token_ids": p}}) for p in prompts]
    outs = []
    for t in tickets:
        assert eng.wait(t, 120000)
        st, body = eng.result(t)
        assert st == 200
        outs.append(body["acp"]["token_ids"])
    first_ok = 0
    for p, got in zip(prompts, outs):
        want, margins, rgap = _greedy(cfg, p, n_new)
        n_ok = assert_tokens_match(got, want, margins, where=len(p), tol=_tol_for(cfg), router_gap=rgap)   # a mismatch is only accepted at a near tie
        first_ok += int(n_ok >= 1)
    assert first_ok >= len(prompts) - 2      # near ties on the very first token are rare


def test_chunked_prefill_equals_single_shot(eng):
    cfg = PRESETS[eng.model_name]
    rng = np.random.default_rng(3)
    prompt = _prompt(rng, 300)
    a, _, _ = _run(eng, prompt, 5)
    small = Engine({"model": eng.model_name, "max_batch": 8, "kv_pages": 128, "max_tokens_per_step": 64})
    try:
        small.model_name = eng.model_name
        b, _, _ = _run(small, prompt, 5)   # prefilled in 5 chunks of <= 64 tokens
    finally:
        small.close()
    assert a == b
    want, margins, rgap = _greedy(cfg, prompt, 5)
    assert_tokens_match(a, want, margins, tol=_tol_for(cfg), router_gap=rgap)


def test_forced_tokens_and_stop(eng):
    rng = np.random.default_rng(4)
    prompt = _prompt(rng, 20)
    toks, _, body = _run(eng, prompt, 10, force=[65, 66, 128009])
    assert toks == [65, 66, 128009]
    assert body["choices"][0]["finish_reason"] == "stop"
    assert body["choices"][0]["message"]["content"] == "AB"


def test_deterministic_across_runs(eng):
    rng = np.random.default_rng(5)
    prompt = _prompt(rng, 77)
    a, la, _ = _run(eng, prompt, 8, logits=2)
    b, lb, _ = _run(eng, prompt, 8, logits=2)
    assert a == b
    assert np.array_equal(la, lb)


def test_prefix_retention_is_bit_identical_to_recompute(eng):
    """§8(f) rank 1: the second LLM step of a Task re-sends its (append-only) window; the engine
    reuses the K/V pages of the shared prompt prefix and must produce exactly what a cold engine
    produces."""
    rng = np.random.default_rng(11)
    p1 = _prompt(rng, 200)
    p2 = p1 + [int(t) for t in rng.integers(0, 256, size=57)]
    eng.stats_reset()
    a1, _, _ = _run(eng, p1, 4)
    s0 = eng.stats()
    a2, lg2, _ = _run(eng, p2, 6, logits=2)
    s1 = eng.stats()
    assert s1["prefix_hits"] - s0["prefix_hits"] == 1
    assert s1["prefix_tokens_reused"] - s0["prefix_tokens_reused"] == 192      # 6 whole pages of p1
    assert s1["prefill_tokens"] - s0["prefill_tokens"] == len(p2) - 192        # only the delta is prefilled
    cold = Engine({"model": eng.model_name, "max_batch": 8, "kv_pages": 128, "max_tokens_per_step": 1024,
                   "prefix_cache": False})
    try:
        cold.model_name = eng.model_name
        b2, lgb, _ = _run(cold, p2, 6, logits=2)
        assert cold.stats()["prefix_hits"] == 0
    finally:
        cold.close()
    assert a2 == b2
    assert np.array_equal(lg2, lgb)          # bit-identical logits, not just tokens
    # an unrelated prompt does not hit
    _run(eng, _prompt(rng, 100), 2)
    assert eng.stats()["prefix_hits"] == s1["prefix_hits"]


def test_shared_prefix_pages_serve_many_sequences_at_once():
    """§8(f) rank 1, second half: every Task of an Agent starts with the same system prompt + tool
    schemas.  Once that prefix is cached, ANY number of concurrent sequences map the same physical
    pages read-only (reference counted, page-chained by content); each result is bit-identical to a
    cold engine's, only the tails are prefilled, and no page leaks."""
    rng = np.random.default_rng(23)
    base = _prompt(rng, 170)                                        # 5 whole pages + 10 tokens
    tails = [[int(t) for t in rng.integers(0, 256, size=n)] for n in (3, 40, 22, 61, 9, 35, 50, 17, 28, 44, 5, 31)]
    prompts = [base + t for t in tails]
    cfg = {"model": "tiny-g2", "max_batch": 16, "kv_pages": 160, "max_tokens_per_step": 512, "max_pages_per_seq": 16}

    def run_all(e, ps):
        ts = [e.submit({"model": "tiny-g2", "max_tokens": 5, "acp": {"prompt_token_ids": p, "return_logits": 1}}) for p in ps]
        out = []
        for t in ts:
            assert e.wait(t, 120000)
            lg = e.logits(t, 1, 128256)
            st, body = e.result(t)
            assert st == 200, body
            out.append((body["acp"]["token_ids"], lg))
        return out

    with Engine(dict(cfg, prefix_cache=False)) as cold:
        want = run_all(cold, prompts)
    with Engine(cfg) as e:
        run_all(e, [base])                                          # seeds the cache: 5 pages
        s0 = e.stats()
        assert s0["prefix_cache_pages"] == 5
        got = run_all(e, prompts)                                   # 12 sequences share them concurrently
        s1 = e.stats()
        assert s1["prefix_hits"] - s0["prefix_hits"] == 12
        assert s1["prefix_tokens_reused"] - s0["prefix_tokens_reused"] == 12 * 160
        assert s1["prefill_tokens"] - s0["prefill_tokens"] == sum(len(p) for p in prompts) - 12 * 160
        for (a, la), (b, lb) in zip(got, want):
            assert a == b and np.array_equal(la, lb)
        # conservation: every page is either free or held by the cache, and the shared chain was
        # extended by the tails' own whole pages (no duplicates of the 5 common pages)
        assert s1["kv_pages_free"] + s1["prefix_cache_pages"] == s1["kv_pages_total"] and s1["running"] == 0
        assert 5 < s1["prefix_cache_pages"] <= 5 + sum((170 + len(t)) // 32 - 5 for t in tails)
        # a pool too small for everything evicts cached leaves instead of failing
        big = [_prompt(rng, 400) for _ in range(12)]
        run_all(e, big)
        s2 = e.stats()
        assert s2["kv_pages_free"] + s2["prefix_cache_pages"] == s2["kv_pages_total"]


@pytest.mark.parametrize("mode", ["item", "chunked"])
def test_decode_attention_modes_agree(eng, mode):
    """Both decode-attention paths (one CTA per item / chunked + merge) give the oracle's tokens on
    mixed context lengths (auto only picks between them, and they are arithmetically identical)."""
    cfg = PRESETS[eng.model_name]
    rng = np.random.default_rng(21)
    prompts = [_prompt(rng, n) for n in (2, 31, 64, 65, 129, 300, 513)]
    e = Engine({"model": eng.model_name, "max_batch": 16, "kv_pages": 256, "max_tokens_per_step": 2048,
                "attn_decode_mode": mode, "prefix_cache": False})
    try:
        ts = [e.submit({"model": eng.model_name, "max_tokens": 5, "acp": {"prompt_token_ids": p}}) for p in prompts]
        outs = []
        for t in ts:
            assert e.wait(t, 120000)
            st, body = e.result(t)
            assert st == 200
            outs.append(body["acp"]["token_ids"])
    finally:
        e.close()
    for p, got in zip(prompts, outs):
        want, margins, rgap = _greedy(cfg, p, 5)
        assert_tokens_match(got, want, margins, where=(mode, len(p)), tol=_tol_for(cfg), router_gap=rgap)


def test_decode_batch_larger_than_one_n_tile(eng):
    """More than 256 live sequences: the decode GEMMs run two N tiles over the same split-K planes.
    Every sequence must still produce what it produces alone (checked against the oracle on a sample)."""
    cfg = PRESETS[eng.model_name]
    rng = np.random.default_rng(31)
    n = 300
    prompts = [_prompt(rng, int(rng.integers(2, 40))) for _ in range(n)]
    big = Engine({"model": eng.model_name, "max_batch": 320, "kv_pages": 1024, "max_tokens_per_step": 4096,
                  "prefix_cache": False})
    try:
        ts = [big.submit({"model": eng.model_name, "max_tokens": 4, "acp": {"prompt_token_ids": p}}) for p in prompts]
        outs = []
        for t in ts:
            assert big.wait(t, 120000)
            st, body = big.result(t)
            assert st == 200
            outs.append(body["acp"]["token_ids"])
        assert big.stats()["decode_tokens"] >= 3 * 256          # really ran wide decode steps
    finally:
        big.close()
    for i in (0, 1, 128, 255, 256, 257, 299):
        want, margins, rgap = _greedy(cfg, prompts[i], 4)
        assert_tokens_match(outs[i], want, margins, where=i, tol=_tol_for(cfg), router_gap=rgap)


def test_long_context_chunked_prefill(eng):
    """A 2500-token window prefilled in 1024-token chunks, then decoded across page and tile
    boundaries, against the oracle."""
    cfg = PRESETS[eng.model_name]
    rng = np.random.default_rng(41)
    prompt = _prompt(rng, 2500)
    toks, _, _ = _run(eng, prompt, 4)
    want, margins, rgap = _greedy(cfg, prompt, 4)
    assert_tokens_match(toks, want, margins, tol=_tol_for(cfg), router_gap=rgap)
    # context limit: prompt + max_tokens beyond max_pages_per_seq * 32 is a typed 400
    t = eng.submit({"model": eng.model_name, "max_tokens": 8000, "acp": {"prompt_token_ids": prompt}})
    assert eng.wait(t, 10000)
    st, body = eng.result(t)
    assert st == 400 and body["error"]["type"] == "context_length_exceeded"


def test_config1_shape_64_windows_of_512_tokens(eng):
    """BASELINE config 1's batch shape: 64 concurrent Tasks x 512-token windows, greedy.  Every
    sequence is compared with the oracle on its first tokens (a sample at the real 8B width, where one
    oracle pass costs seconds), and all 64 must equal what the same prompt produces alone."""
    cfg = PRESETS[eng.model_name]
    rng = np.random.default_rng(64512)
    prompts = [_prompt(rng, 512) for _ in range(64)]
    n_new = 6
    big = Engine({"model": eng.model_name, "max_batch": 64, "kv_pages": 64 * 18 + 8, "max_tokens_per_step": 4096,
                  "prefix_cache": False})
    try:
        ts = [big.submit({"model": eng.model_name, "max_tokens": n_new, "acp": {"prompt_token_ids": p}}) for p in prompts]
        outs = []
        for t in ts:
            assert big.wait(t, 300000)
            st, body = big.result(t)
            assert st == 200, body
            outs.append(body["acp"]["token_ids"])
        s = big.stats()
        assert s["prefill_tokens"] == 64 * 512 and s["decode_tokens"] >= 64 * (n_new - 1) - 64
        alone, _, _ = _run(eng, prompts[5], n_new)
        assert alone == outs[5]
    finally:
        big.close()
    sample = range(64) if cfg.hidden <= 1024 else (0, 13, 31, 63)
    for i in sample:
        want, margins, rgap = _greedy(cfg, prompts[i], n_new)
        assert_tokens_match(outs[i], want, margins, where=i, tol=_tol_for(cfg), router_gap=rgap)
