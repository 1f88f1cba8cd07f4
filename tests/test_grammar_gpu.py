"""Constrained tool-call decoding on the GPU (tool_choice "required" / named functions, DESIGN.md §3.3):
grammar_mask_kernel against oracle/grammar_oracle.py bit for bit over whole vocabularies, and the engine's
masked logits, tokens and responses across the model families."""
import ctypes
import json
import os

import numpy as np
import pytest

from agentcontrolplane_b200 import _lib, host
from agentcontrolplane_b200.engine import Engine
from oracle import chat_oracle
from oracle import sampling_oracle as S
from oracle.grammar_oracle import MAX_DEPTH, MAX_WS, Grammar, build_trie

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN_TOK = os.path.join(ROOT, "tests", "golden", "llama3_style_tokenizer.json")
VOCAB = 128256
STOPS = (128001, 128008, 128009)
NAMES = ["get_weather", "get_time", "say \"hi\"", "日本"]
TOOLS = [{"type": "function", "function": {"name": n, "parameters": {"type": "object"}}} for n in NAMES]


def synthetic_vocab():
    vocab = [chat_oracle.decode_tokens([i]) for i in range(VOCAB)]
    return vocab, [i in STOPS for i in range(VOCAB)]


def golden_vocab():
    added = {t["id"]: t["content"] for t in json.load(open(GOLDEN_TOK))["added_tokens"]}
    n = max(added) + 1
    vocab = [host.tokenizer_decode([i], GOLDEN_TOK) for i in range(n)]
    stop = [added.get(i) in ("<|end_of_text|>", "<|eom_id|>", "<|eot_id|>") for i in range(n)]
    return vocab, stop


_VOCABS = {}


def vocab_of(which):
    if which not in _VOCABS:
        vocab, stop = synthetic_vocab() if which == "synthetic" else golden_vocab()
        _VOCABS[which] = (vocab, stop, build_trie(vocab, stop))
    return _VOCABS[which]


def device_mask(names, parallel, prefix: bytes, vocab, stop):
    f = _lib.load().acp_kernel_grammar_mask
    f.argtypes = [ctypes.c_char_p, ctypes.c_int, ctypes.c_char_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_char_p,
                  ctypes.c_char_p, ctypes.c_int, ctypes.c_void_p]
    off = np.zeros(len(vocab) + 1, np.int32)
    off[1:] = np.cumsum([len(b) for b in vocab])
    bits = np.zeros((len(vocab) + 7) // 8, np.uint8)
    rc = f(json.dumps(names).encode(), int(parallel), prefix, len(prefix), off.ctypes.data, b"".join(vocab),
           bytes(stop), len(vocab), bits.ctypes.data)
    assert rc == 0
    return np.unpackbits(bits, bitorder="little")[: len(vocab)].astype(bool)


def _walk_prefixes(parallel):
    """prefixes that reach the interesting states: inside names, escapes, multi-byte UTF-8, numbers, the depth
    cap, the whitespace cap, between calls, and seeded random walks"""
    head = b'{"name": "get_time", "parameters": '
    fixed = [b"", b'{"na', b'{"name": "', b'{"name": "get_', b'{"name": "say \\', b'{"name": "\xe6\x97',
             head, head + b"{", head + b'{"a": "x\\', head + b'{"a": "x\\u00', head + b'{"a": "\xf0\x9f',
             head + b'{"a": "\xe0', head + b'{"a": -', head + b'{"a": 0', head + b'{"a": 12.5e', head + b'{"a": 1.5',
             head + b'{"a": [tr', head + b'{"a": ' + b"[" * (MAX_DEPTH - 1), head + b"{" + b" " * MAX_WS,
             head + b'{"a": 1', head + b"{}", head + b"{}}"] + ([head + b"{}}\n"] if parallel else [])
    g = Grammar(NAMES, parallel)
    rng = np.random.default_rng(11)
    walks = []
    for _ in range(6):
        s, data = g.start(), bytearray()
        for _ in range(int(rng.integers(10, 120))):
            opts = [c for c in range(256) if g.step(s.copy(), c)]
            if not opts:
                break
            c = int(rng.choice(opts))
            g.step(s, c)
            data.append(c)
        walks.append(bytes(data))
    return fixed + walks


@pytest.mark.parametrize("which", ["synthetic", "golden"])
@pytest.mark.parametrize("parallel", [True, False])
def test_mask_kernel_equals_oracle_over_every_id(which, parallel):
    vocab, stop, trie = vocab_of(which)
    g = Grammar(NAMES, parallel)
    for prefix in _walk_prefixes(parallel):
        s, _ = g.run(prefix)
        want = np.array(g.allowed(s, vocab, stop, trie))
        got = device_mask(NAMES, parallel, prefix, vocab, stop)
        assert want.any(), prefix
        bad = np.nonzero(got != want)[0]
        assert bad.size == 0, (which, prefix, [(int(i), vocab[i], bool(want[i])) for i in bad[:8]])


# ---- the engine ----
MODELS = ["tiny", "tiny-g2", "tiny-fp8", "tiny-moe", "llama-3-8b-l2"]


@pytest.fixture(scope="module", params=MODELS)
def eng(request):
    e = Engine({"model": request.param, "max_batch": 32, "kv_pages": 512, "max_tokens_per_step": 1024})
    e.model_name = request.param
    yield e
    e.close()


def _prompt(rng, n):
    return [128000] + [int(t) for t in rng.integers(0, 256, size=n)]


def _req(eng, prompt, max_tokens, **kw):
    acp = {"prompt_token_ids": prompt}
    for k in ("return_logits", "force_tokens"):
        if k in kw:
            acp[k] = kw.pop(k)
    return dict({"model": eng.model_name, "max_tokens": max_tokens, "tools": TOOLS, "acp": acp}, **kw)


def _finish(eng, t, logits=0):
    assert eng.wait(t, 300000)
    lg = eng.logits(t, logits, VOCAB) if logits else None
    status, body = eng.result(t)
    return status, body, lg


def _key(s):
    return (s.mode, s.pos, tuple(s.cands), tuple(s.stack), s.ws, s.tok, s.aux, s.u8, s.parallel)


def masked_candidates(l, sampling, step):
    """What the sampler may emit from a masked logit row: the sampling oracle's candidates among the finite ids.
    A masked id has zero weight in the oracle's CDF; sample_kernel never keeps one, not even in the CDF's last step."""
    if sampling:
        T, k, p = sampling["temperature"], sampling.get("top_k", 0), sampling.get("top_p", 1.0)
        cands = S.candidates(l, T, k, p, sampling["seed"], step)
    else:
        cands = {S.sample(l, 0.0, 0, 1.0, 0, step)}
    return {c for c in cands if np.isfinite(l[c])}


def check_constrained_run(g, lg, toks, sampling, cache):
    """At every kept position the -inf pattern is the oracle's mask for the state the emitted prefix reaches, and
    the token is the sampler's on those masked logits.  When the response carries no token ids (a 422 length cut)
    the prefix is followed through every token the sampler may have drawn that leads to the next position's mask."""
    vocab, stop, trie = vocab_of("synthetic")

    def allowed(s):
        k = _key(s)
        if k not in cache:
            cache[k] = np.array(g.allowed(s, vocab, stop, trie))
        return cache[k]

    states = [g.start()]
    for i in range(len(lg)):
        fin = np.isfinite(lg[i])
        assert np.all(lg[i][~fin] == -np.inf)
        states = [s for s in states if np.array_equal(allowed(s), fin)]
        assert states, i
        cands = masked_candidates(lg[i], sampling, i)
        assert cands, i
        if toks is not None:
            assert toks[i] in cands, (i, toks[i], sorted(cands))
            cands = {toks[i]}
        nxt = {}
        for s in states:
            for c in cands:
                if stop[c]:
                    assert g.accepting(s)
                    continue
                t, _ = g.run(vocab[c], s)
                assert t is not None
                nxt[_key(t)] = t
        states = list(nxt.values())
        if not states:
            break


@pytest.mark.parametrize("sampling", [{}, {"temperature": 1.0, "seed": 77}, {"temperature": 0.8, "top_k": 40, "top_p": 0.9, "seed": 5}],
                         ids=["greedy", "t1", "t0.8-k40-p0.9"])
def test_masked_logits_and_tokens_follow_the_oracle(eng, sampling):
    rng = np.random.default_rng(len(sampling) + 3)
    n = 64
    for parallel in (True, False):
        g = Grammar(NAMES, parallel)
        t = eng.submit(_req(eng, _prompt(rng, 40), n, return_logits=n, tool_choice="required",
                            parallel_tool_calls=parallel, **sampling))
        status, body, lg = _finish(eng, t, n)
        if status == 422:
            assert body["error"]["type"] == "truncated_tool_call", body
            assert len(lg) == n
        else:
            assert status == 200, body
        toks = body["acp"]["token_ids"] if status == 200 else None
        check_constrained_run(g, lg, toks, sampling, {})


def test_first_position_finite_logits_equal_the_unconstrained_ones(eng):
    rng = np.random.default_rng(21)
    prompt = _prompt(rng, 50)
    _, _, free = _finish(eng, eng.submit(_req(eng, prompt, 1, return_logits=1)), 1)
    _, _, con = _finish(eng, eng.submit(_req(eng, prompt, 1, return_logits=1, tool_choice="required")), 1)
    keep = np.isfinite(con[0])
    assert keep.sum() == 1 and keep[ord("{")]          # only '{' starts a call
    assert np.array_equal(con[0][keep].view(np.uint32), free[0][keep].view(np.uint32))


def test_unconstrained_requests_beside_constrained_ones_are_unchanged(eng):
    rng = np.random.default_rng(5)
    plain = [_req(eng, _prompt(rng, 30 + 7 * i), 10, **({"temperature": 1.0, "seed": 9 + i} if i % 2 else {}))
             for i in range(4)]
    alone = []
    for r in plain:
        st, body, _ = _finish(eng, eng.submit(r))
        assert st == 200
        alone.append(body["acp"]["token_ids"])
    ts = [eng.submit(r) for r in plain]
    cs = [eng.submit(_req(eng, _prompt(rng, 25), 12, tool_choice="required", **({"temperature": 0.9, "seed": i} if i % 2 else {})))
          for i in range(6)]
    for t, want in zip(ts, alone):
        st, body, _ = _finish(eng, t)
        assert st == 200 and body["acp"]["token_ids"] == want
    for t in cs:
        st, body, _ = _finish(eng, t)
        assert st in (200, 422), body


def test_named_function_with_forced_prefix_completes_to_a_tool_call(eng):
    rng = np.random.default_rng(8)
    forced = list(b'{"name": "get_time", "parameters": {}')
    for parallel in (False, True):
        st, body, _ = _finish(eng, eng.submit(_req(
            eng, _prompt(rng, 20), len(forced) + 2 + (0 if not parallel else 30), force_tokens=forced,
            tool_choice={"type": "function", "function": {"name": "get_time"}}, parallel_tool_calls=parallel)))
        if parallel and st == 422:       # a second call started and was cut by max_tokens
            assert body["error"]["type"] == "truncated_tool_call"
            continue
        assert st == 200, body
        choice = body["choices"][0]
        assert choice["finish_reason"] == "tool_calls"
        calls = choice["message"]["tool_calls"]
        assert calls[0]["function"] == {"name": "get_time", "arguments": "{}"}
        assert all(c["function"]["name"] == "get_time" for c in calls)
        if not parallel:
            assert len(calls) == 1 and body["acp"]["token_ids"][len(forced):] in ([ord("}"), s] for s in STOPS)


def test_required_responses_hold_only_allowed_calls(eng):
    rng = np.random.default_rng(13)
    ts = [eng.submit(_req(eng, _prompt(rng, 20 + i), 24 + 8 * i, tool_choice="required",
                          **({"temperature": 1.0, "seed": 100 + i} if i % 2 else {}))) for i in range(8)]
    for t in ts:
        st, body, _ = _finish(eng, t)
        if st == 422:
            assert body["error"]["type"] == "truncated_tool_call", body
            continue
        assert st == 200, body
        calls = body["choices"][0]["message"]["tool_calls"]
        assert calls and body["choices"][0]["finish_reason"] == "tool_calls"
        for c in calls:
            assert c["function"]["name"] in NAMES
            assert isinstance(json.loads(c["function"]["arguments"]), dict)


def test_forced_tokens_the_grammar_rejects_are_refused(eng):
    for forced in (list(b'{"name": "nope"'), list(b" "), [128009]):
        st, body, _ = _finish(eng, eng.submit(_req(eng, [128000, 72], 8, force_tokens=forced, tool_choice="required")))
        assert st == 400 and "tool_choice" in body["error"]["message"], body
