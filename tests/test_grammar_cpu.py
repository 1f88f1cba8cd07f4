"""The tool-call grammar of `tool_choice: "required"` / named functions on the host (no GPU): the C++ automaton
of csrc/grammar.h (through acp_kernel_grammar_accepts) against oracle/grammar_oracle.py on handwritten cases
and a seeded fuzz, accepted completions against json.loads and the chat oracle's parse_completion, random walks
that never reach a dead end, and the 400s of tool_choice validation."""
import ctypes
import json
import random

import pytest

from agentcontrolplane_b200 import _lib, host
from oracle import chat_oracle
from oracle.grammar_oracle import MAX_DEPTH, MAX_WS, Grammar

NAMES = ["get_weather", "get_time", "get", "say \"hi\"", "naïve\\path", "tab\tname", "ctl\x01x", "日本"]


def _lib_accepts():
    f = _lib.load().acp_kernel_grammar_accepts
    f.argtypes = [ctypes.c_char_p, ctypes.c_int, ctypes.c_char_p, ctypes.c_size_t, ctypes.POINTER(ctypes.c_size_t),
                  ctypes.POINTER(ctypes.c_int)]
    return f


def cpp_run(names, parallel, data: bytes):
    """(bytes accepted, complete) of the C++ automaton"""
    consumed, complete = ctypes.c_size_t(), ctypes.c_int()
    rc = _lib_accepts()(json.dumps(names).encode(), int(parallel), data, len(data), ctypes.byref(consumed),
                        ctypes.byref(complete))
    assert rc == 0
    return consumed.value, bool(complete.value)


def oracle_run(g: Grammar, data: bytes):
    s, n = g.run(data)
    return n, g.accepting(s)


def call(name: str, params: bytes) -> bytes:
    return b'{"name": ' + Grammar([name]).names[0] + b', "parameters": ' + params + b"}"


HANDWRITTEN = [
    call("get_time", b"{}"),
    call("get_weather", b'{"city": "Paris", "days": [1, 2, 3], "x": {"y": null, "z": true, "w": false}}'),
    call("get", b'{"n": -0, "f": 1.5e-3, "g": 2E+10, "h": 0.0, "i": 10}'),
    call("say \"hi\"", b'{"s": "\\u00e9\\n\\"\\\\\\/\\b\\f\\r\\t"}'),
    call("naïve\\path", "{\"é\": \"日本語 \U0001F600\"}".encode()),
    call("tab\tname", b"{}") + b"\n" + call("ctl\x01x", b'{ "a" :\t[ ] , "b":{} }'),
    call("日本", b"{}"),
    # rejections
    b'{"name": "nope", "parameters": {}}',
    b'{"name":"get_time", "parameters": {}}',
    call("get_time", b"[]"),
    call("get_time", b'{"a": 01}'),
    call("get_time", b'{"a": 1.}'),
    call("get_time", b'{"a": 1e}'),
    call("get_time", b'{"a": -}'),
    call("get_time", b'{"a": .5}'),
    call("get_time", b'{"a": NaN}'),
    call("get_time", b'{"a": [1,]}'),
    call("get_time", b'{"a": 1,}'),
    call("get_time", b'{a: 1}'),
    call("get_time", b'{"a": "\x01"}'),
    call("get_time", b'{"a": "\\x"}'),
    call("get_time", b'{"a": "\\u12g4"}'),
    call("get_time", b'{"a": "\xc0\x80"}'),         # overlong
    call("get_time", b'{"a": "\xe0\x80\x80"}'),     # overlong
    call("get_time", b'{"a": "\xed\xa0\x80"}'),     # surrogate
    call("get_time", b'{"a": "\xf4\x90\x80\x80"}'),  # above U+10FFFF
    call("get_time", b'{"a": "\xf5"}'),
    call("get_time", b'{"a": "\xc3"}'),             # cut character
    call("get_time", b'{"a": truth}'),
    call("get_time", b"{}") + b"\n\n" + call("get", b"{}"),
    call("get_time", b"{}") + b" ",
    b" " + call("get_time", b"{}"),
    call("get_time", b"{" + b" " * MAX_WS + b"}"),
    call("get_time", b"{" + b" " * (MAX_WS + 1) + b"}"),
    call("get_time", b'{"a": ' + b"[" * (MAX_DEPTH - 1) + b"]" * (MAX_DEPTH - 1) + b"}"),
    call("get_time", b'{"a": ' + b"[" * MAX_DEPTH + b"]" * MAX_DEPTH + b"}"),
    call("get_time", b'{"a": 1}') + b"}",
    call("get_tim", b"{}"),
    call("get_times", b"{}"),
]


@pytest.mark.parametrize("parallel", [True, False])
@pytest.mark.parametrize("case", range(len(HANDWRITTEN)))
def test_cpp_automaton_equals_oracle_on_handwritten_cases(case, parallel):
    data = HANDWRITTEN[case]
    g = Grammar(NAMES, parallel)
    want = oracle_run(g, data)
    assert cpp_run(NAMES, parallel, data) == want, data
    for cut in range(len(data)):   # every prefix
        assert cpp_run(NAMES, parallel, data[:cut])[0] == min(cut, want[0]), (data, cut)


def test_handwritten_verdicts():
    g = Grammar(NAMES)
    complete = [g.is_complete(d) for d in HANDWRITTEN]
    assert complete[:7] == [True] * 7
    assert not any(complete[7:32])
    assert complete[32] and not complete[33]        # whitespace cap
    assert complete[34] and not complete[35]        # depth cap (the parameters object is level 1)
    assert not any(complete[36:])
    assert not Grammar(NAMES, parallel=False).is_complete(HANDWRITTEN[5])


# ---- a generator of valid OBJECTs, and mutations of them ----
def _ws(rng):
    return rng.choice([b"", b"", b" ", b"\n", b"\t ", b"\r\n  "])


def _string(rng):
    parts = []
    for _ in range(rng.randint(0, 5)):
        k = rng.randint(0, 6)
        if k == 0:
            parts.append(rng.choice([b'\\"', b"\\\\", b"\\/", b"\\b", b"\\f", b"\\n", b"\\r", b"\\t"]))
        elif k == 1:
            parts.append(b"\\u%04x" % rng.randint(0, 0xFFFF))
        elif k == 2:
            parts.append(chr(rng.choice([0xE9, 0x800, 0xFFFD, 0x10000, 0x10FFFF, 0xD7FF, 0xE000])).encode())
        else:
            parts.append(bytes(rng.choice(b"abc xyz:{}[],01") for _ in range(rng.randint(1, 4))))
    return b'"' + b"".join(parts) + b'"'


def _number(rng):
    s = rng.choice([b"", b"-"]) + rng.choice([b"0", b"7", b"42", b"1000"])
    if rng.random() < 0.4:
        s += b"." + rng.choice([b"0", b"5", b"125"])
    if rng.random() < 0.3:
        s += rng.choice([b"e", b"E"]) + rng.choice([b"", b"+", b"-"]) + rng.choice([b"0", b"10"])
    return s


def _value(rng, depth):
    k = rng.randint(0, 7 if depth < MAX_DEPTH else 4)
    if k == 0:
        return _string(rng)
    if k == 1:
        return _number(rng)
    if k == 2:
        return rng.choice([b"true", b"false", b"null"])
    if k in (3, 4):
        return _number(rng) if rng.random() < 0.5 else _string(rng)
    if k in (5, 6):
        return _object(rng, depth + 1)
    items = [_ws(rng) + _value(rng, depth + 1) + _ws(rng) for _ in range(rng.randint(0, 3))]
    return b"[" + b",".join(items) + b"]" if items else b"[" + _ws(rng) + b"]"


def _object(rng, depth=1):
    members = [_ws(rng) + _string(rng) + _ws(rng) + b":" + _ws(rng) + _value(rng, depth) + _ws(rng)
               for _ in range(rng.randint(0, 3))]
    return b"{" + b",".join(members) + b"}" if members else b"{" + _ws(rng) + b"}"


def _completion(rng, names, parallel):
    n = rng.randint(1, 3) if parallel else 1
    return b"\n".join(call(rng.choice(names), _object(rng)) for _ in range(n))


def _mutate(rng, data: bytes) -> bytes:
    b = bytearray(data)
    for _ in range(rng.randint(1, 3)):
        i = rng.randrange(len(b) + 1)
        k = rng.randint(0, 2)
        byte = rng.choice([rng.randrange(256), rng.choice(b'{}[]",:0.eE-+ \n\\u')])
        if k == 0 and i < len(b):
            b[i] = byte
        elif k == 1:
            b.insert(i, byte)
        elif i < len(b):
            del b[i]
    return bytes(b)


def test_seeded_fuzz_cpp_equals_oracle_and_completions_parse():
    rng = random.Random(0xACB200)
    completed = 0
    for it in range(1500):
        parallel = it % 3 != 0
        names = rng.sample(NAMES, rng.randint(1, len(NAMES)))
        g = Grammar(names, parallel)
        data = _completion(rng, names, parallel)
        if it % 2:
            data = _mutate(rng, data)
        got, want = cpp_run(names, parallel, data), oracle_run(g, data)
        assert got == want, (names, parallel, data)
        if not want[1]:
            continue
        completed += 1
        text = data.decode("utf-8")           # strict: well-formed UTF-8 only
        # CALLs are separated by one newline; "}\n{" never occurs inside an OBJECT (it needs a ',' there)
        lines = text.replace('}\n{"name": ', '}\x00{"name": ').split("\x00")
        assert parallel or len(lines) == 1
        for line in lines:                    # every CALL is a JSON object naming an allowed tool
            obj = json.loads(line, parse_constant=lambda c: pytest.fail("constant " + c))
            assert obj["name"] in names and isinstance(obj["parameters"], dict)
        tools = [{"type": "function", "function": {"name": n}} for n in names]
        parsed = chat_oracle.parse_completion(text, tools)
        assert len(parsed["tool_calls"]) == len(lines)
        for line, tc in zip(lines, parsed["tool_calls"]):
            assert tc["function"]["name"] == json.loads(line)["name"]
            head = b'{"name": ' + Grammar([tc["function"]["name"]]).names[0] + b', "parameters": '
            assert tc["function"]["arguments"].encode() == line.encode()[len(head):-1]   # byte-identical OBJECT
        # the engine's own parser agrees (what the response's tool_calls are built from)
        assert host.parse_completion(text, tools)["tool_calls"] == parsed["tool_calls"]
    assert completed > 500


def test_random_walks_reach_no_dead_end():
    """From every state a walk reaches, some byte continues or a stop token is allowed; the C++ automaton
    accepts every walk, and the walks visit the depth cap, the whitespace cap, names, escapes, UTF-8 and numbers."""
    rng = random.Random(7)
    favoured = list(b'{}[]",:0123456789-.eE+ \n\tu\\tfnrl') + [0xC3, 0xA9, 0xE2, 0x82, 0xAC, 0xF0, 0x9F, 0x98, 0x80]
    seen = set()
    for w in range(60):
        parallel = w % 2 == 0
        names = rng.sample(NAMES, rng.randint(1, 4))
        g = Grammar(names, parallel)
        s, data = g.start(), bytearray()
        open_bias = 0.9 if w % 5 == 0 else 0.3
        for _ in range(400):
            options = [c for c in range(256) if g.step(s.copy(), c)]
            assert options or g.accepting(s), bytes(data)
            if not options:
                break
            pref = [c for c in options if c in favoured]
            if w % 5 == 0 and ord("[") in options and rng.random() < open_bias:
                c = ord("[")
            elif w % 7 == 0 and ord(" ") in options:
                c = ord(" ")
            else:
                c = rng.choice(pref if pref and rng.random() < 0.8 else options)
            g.step(s, c)
            data.append(c)
            if s.mode == "json":
                seen.add(("depth", len(s.stack)))
                seen.add(("ws", s.ws))
                seen.add(("tok", s.tok))
            seen.add(("mode", s.mode))
        assert cpp_run(names, parallel, bytes(data))[0] == len(data)
    assert ("depth", MAX_DEPTH) in seen and ("ws", MAX_WS) in seen
    for tok in ("string", "escape", "hex", "utf8", "num_frac", "num_exp", "literal"):
        assert ("tok", tok) in seen, tok
    assert ("mode", "name") in seen and ("mode", "after") in seen


# ---- tool_choice validation (section 1 of DESIGN.md §3.4) ----
BASE = {"model": "m", "messages": [{"role": "user", "content": "hi"}]}
TOOLS = [{"type": "function", "function": {"name": n, "parameters": {"type": "object"}}} for n in ("get_time", "get_weather")]


@pytest.mark.parametrize("extra", [
    {"tool_choice": "required"},
    {"tool_choice": "required", "tools": []},
    {"tool_choice": {"type": "function", "function": {"name": "get_time"}}},
    {"tool_choice": {"type": "function", "function": {"name": "nope"}}, "tools": TOOLS},
    {"tool_choice": {"type": "function"}, "tools": TOOLS},
    {"tool_choice": {"type": "function", "function": {"name": ""}}, "tools": TOOLS},
    {"tool_choice": {"type": "function", "function": {"name": 3}}, "tools": TOOLS},
    {"tool_choice": {"type": "tool", "function": {"name": "get_time"}}, "tools": TOOLS},
    {"tool_choice": {"function": "get_time"}, "tools": TOOLS},
    {"tool_choice": "none", "tools": TOOLS},
    {"tool_choice": "any", "tools": TOOLS},
    {"tool_choice": 1, "tools": TOOLS},
    {"tool_choice": "required", "tools": [{"type": "function", "function": {"name": f"t{i}"}} for i in range(129)]},
    {"tool_choice": "required", "tools": [{"type": "function", "function": {"name": "x" * 2100 + str(i)}} for i in range(4)]},
])
def test_tool_choice_refusals(extra):
    r = host.render_prompt(dict(BASE, **extra))
    assert r.get("status") == 400 and "tool_choice" in r["error"], (extra, r)


@pytest.mark.parametrize("extra", [
    {"tool_choice": "required", "tools": TOOLS},
    {"tool_choice": "required", "tools": TOOLS, "parallel_tool_calls": False},
    {"tool_choice": {"type": "function", "function": {"name": "get_weather"}}, "tools": TOOLS},
    {"tool_choice": "required", "tools": [{"type": "function", "function": {"name": f"t{i}"}} for i in range(128)]},
    {"tool_choice": "auto", "tools": TOOLS},
])
def test_tool_choice_served(extra):
    r = host.render_prompt(dict(BASE, **extra))
    assert "status" not in r, (extra, r)
    # the prompt is the one "auto" renders: the constraint acts on sampling only
    assert r == host.render_prompt(dict(BASE, tools=extra["tools"]))


def test_hook_rejects_bad_name_lists():
    consumed, complete = ctypes.c_size_t(), ctypes.c_int()
    for bad in (b"[]", b"{}", b"[1]", b"not json"):
        assert _lib_accepts()(bad, 1, b"", 0, ctypes.byref(consumed), ctypes.byref(complete)) != 0
