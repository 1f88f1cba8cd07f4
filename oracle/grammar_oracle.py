"""Python restatement of the tool-call grammar of `tool_choice: "required"` / named functions
(agentcontrolplane_b200/csrc/grammar.h, DESIGN.md §3.3).

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

    COMPLETION := CALL ( "\\n" CALL )* STOP          (parallel_tool_calls false: CALL STOP)
    CALL       := '{"name": ' NAME ', "parameters": ' OBJECT '}'
    NAME       := the bytes Json::escape_to writes for an allowed tool name, quotes included
    OBJECT     := an RFC 8259 object; strings well-formed UTF-8; at most 32 levels; whitespace runs <= 32 bytes
    STOP       := a stop token, allowed only right after a complete CALL

The automaton here is written as a pushdown recogniser over bytes with an explicit container stack
(a Python list), independent of the C++ packing of the state into a fixed-size struct.
`allowed(state, vocab)` walks a byte trie of the vocabulary, so a rejected prefix prunes every token
that starts with it.
"""
from __future__ import annotations

MAX_DEPTH = 32
MAX_WS = 32
PREFIX = b'{"name": '
MID = b', "parameters": '
WS = b" \t\n\r"
DIGITS = b"0123456789"
HEX = b"0123456789abcdefABCDEF"


def escape_name(name: str) -> bytes:
    """Json::escape_to (csrc/json.h) for a valid UTF-8 string."""
    out = bytearray(b'"')
    for ch in name:
        c = ord(ch)
        if ch == '"':
            out += b'\\"'
        elif ch == "\\":
            out += b"\\\\"
        elif ch == "\n":
            out += b"\\n"
        elif ch == "\r":
            out += b"\\r"
        elif ch == "\t":
            out += b"\\t"
        elif c < 0x20:
            out += b"\\u%04x" % c
        else:
            out += ch.encode("utf-8")
    out += b'"'
    return bytes(out)


def utf8_next_range(lead: int):
    """(continuation bytes, allowed range of the first one) after a UTF-8 lead byte, or None."""
    if 0xC2 <= lead <= 0xDF:
        return 1, (0x80, 0xBF)
    if lead == 0xE0:
        return 2, (0xA0, 0xBF)
    if lead == 0xED:
        return 2, (0x80, 0x9F)
    if 0xE1 <= lead <= 0xEF:
        return 2, (0x80, 0xBF)
    if lead == 0xF0:
        return 3, (0x90, 0xBF)
    if 0xF1 <= lead <= 0xF3:
        return 3, (0x80, 0xBF)
    if lead == 0xF4:
        return 3, (0x80, 0x8F)
    return None


class State:
    """Mutable recogniser state; copy() before trying alternatives."""
    __slots__ = ("mode", "pos", "cands", "stack", "ws", "tok", "aux", "u8", "parallel")

    def __init__(self, names: list[bytes], parallel: bool):
        self.mode = "prefix"      # prefix | name | mid | root | json | close | after
        self.pos = 0              # offset inside the current literal / name
        self.cands = names        # escaped names consistent with the NAME bytes so far
        self.stack: list[str] = []  # "{" / "[" per open container
        self.ws = 0
        self.tok = "value"        # inside json: what comes next
        self.aux = None           # is-key flag of a string / (literal, offset)
        self.u8 = None            # inside a UTF-8 sequence: (continuation bytes left, lo, hi) of the next one
        self.parallel = parallel

    def copy(self) -> "State":
        s = State.__new__(State)
        s.mode, s.pos, s.cands, s.stack = self.mode, self.pos, self.cands, list(self.stack)
        s.ws, s.tok, s.aux, s.u8, s.parallel = self.ws, self.tok, self.aux, self.u8, self.parallel
        return s


class Grammar:
    def __init__(self, tool_names: list[str], parallel: bool = True):
        self.names = sorted(set(escape_name(n) for n in tool_names))
        self.parallel = parallel

    def start(self) -> State:
        return State(self.names, self.parallel)

    # ---- one byte ----
    def step(self, s: State, c: int) -> bool:
        m = s.mode
        if m == "prefix" or m == "mid":
            lit = PREFIX if m == "prefix" else MID
            if c != lit[s.pos]:
                return False
            s.pos += 1
            if s.pos == len(lit):
                s.mode, s.pos = ("name", 0) if m == "prefix" else ("root", 0)
                s.cands = self.names
            return True
        if m == "name":
            cands = [n for n in s.cands if n[s.pos] == c]
            if not cands:
                return False
            s.pos += 1
            s.cands = cands
            if len(cands[0]) == s.pos:
                s.mode, s.pos = "mid", 0
            return True
        if m == "root":
            if c != ord("{"):
                return False
            s.mode, s.stack, s.tok, s.ws = "json", ["{"], "first_key", 0
            return True
        if m == "close":
            if c != ord("}"):
                return False
            s.mode = "after"
            return True
        if m == "after":
            if c == ord("\n") and s.parallel:
                s.mode, s.pos = "prefix", 0
                return True
            return False
        return self._json(s, c)

    def _close(self, s: State):
        s.stack.pop()
        if not s.stack:
            s.mode = "close"
        else:
            s.tok = "after_value"

    def _json(self, s: State, c: int) -> bool:
        t = s.tok
        if t == "string":
            if c == ord('"'):
                s.tok = "colon" if s.aux else "after_value"
                return True
            if c == ord("\\"):
                s.tok = "escape"
                return True
            if c < 0x20:
                return False
            if c < 0x80:
                return True
            r = utf8_next_range(c)
            if r is None:
                return False
            s.tok, s.u8 = "utf8", (r[0], r[1][0], r[1][1])
            return True
        if t == "utf8":
            left, lo, hi = s.u8
            if not lo <= c <= hi:
                return False
            if left == 1:
                s.tok, s.u8 = "string", None
            else:
                s.u8 = (left - 1, 0x80, 0xBF)
            return True
        if t == "escape":
            if c == ord("u"):
                s.tok, s.pos = "hex", 4
                return True
            if c in b'"\\/bfnrt':
                s.tok = "string"
                return True
            return False
        if t == "hex":
            if c not in HEX:
                return False
            s.pos -= 1
            if s.pos == 0:
                s.tok = "string"
            return True
        if t == "literal":
            lit, i = s.aux
            if c != lit[i]:
                return False
            if i + 1 == len(lit):
                s.tok = "after_value"
            else:
                s.aux = (lit, i + 1)
            return True
        if t.startswith("num_"):
            nxt = self._number(t, c)
            if nxt is not None:
                s.tok = nxt
                return True
            if t in ("num_minus", "num_dot", "num_e", "num_esign"):
                return False
            s.tok = "after_value"          # the number ended before c
            return self._json(s, c)
        # structural positions: whitespace first
        if c in WS:
            if s.ws >= MAX_WS:
                return False
            s.ws += 1
            return True
        s.ws = 0
        if t == "first_key" and c == ord("}"):
            self._close(s)
            return True
        if t in ("first_key", "key"):
            if c != ord('"'):
                return False
            s.tok, s.aux = "string", True
            return True
        if t == "colon":
            if c != ord(":"):
                return False
            s.tok = "value"
            return True
        if t == "after_value":
            top = s.stack[-1]
            if c == ord(","):
                s.tok = "key" if top == "{" else "value"
                return True
            if c == ord("}" if top == "{" else "]"):
                self._close(s)
                return True
            return False
        if t == "first_value" and c == ord("]"):
            self._close(s)
            return True
        # a value (t is "value" or "first_value")
        if c in b"{[":
            if len(s.stack) >= MAX_DEPTH:
                return False
            s.stack.append(chr(c))
            s.tok = "first_key" if c == ord("{") else "first_value"
            return True
        if c == ord('"'):
            s.tok, s.aux = "string", False
            return True
        for lit in (b"true", b"false", b"null"):
            if c == lit[0]:
                s.tok, s.aux = "literal", (lit, 1)
                return True
        if c == ord("-"):
            s.tok = "num_minus"
            return True
        if c == ord("0"):
            s.tok = "num_zero"
            return True
        if c in DIGITS:
            s.tok = "num_int"
            return True
        return False

    @staticmethod
    def _number(t: str, c: int):
        """next number state after c, or None when c does not continue the number"""
        d = c in DIGITS
        if t == "num_minus":
            return "num_zero" if c == ord("0") else ("num_int" if d else None)
        if t == "num_zero":
            return "num_dot" if c == ord(".") else ("num_e" if c in b"eE" else None)
        if t == "num_int":
            return "num_int" if d else ("num_dot" if c == ord(".") else ("num_e" if c in b"eE" else None))
        if t == "num_dot":
            return "num_frac" if d else None
        if t == "num_frac":
            return "num_frac" if d else ("num_e" if c in b"eE" else None)
        if t == "num_e":
            return "num_esign" if c in b"+-" else ("num_exp" if d else None)
        if t in ("num_esign", "num_exp"):
            return "num_exp" if d else None
        return None

    # ---- strings of bytes ----
    def run(self, data: bytes, s: State | None = None):
        """(state after data, number of bytes accepted); the state is None when a byte was rejected"""
        s = self.start() if s is None else s.copy()
        for i, c in enumerate(data):
            if not self.step(s, c):
                return None, i
        return s, len(data)

    def accepts_prefix(self, data: bytes) -> bool:
        return self.run(data)[0] is not None

    @staticmethod
    def accepting(s: State) -> bool:
        return s is not None and s.mode == "after"

    def is_complete(self, data: bytes) -> bool:
        """data followed by a stop token is a COMPLETION"""
        return self.accepting(self.run(data)[0])

    # ---- a vocabulary ----
    def allowed(self, s: State, vocab: list[bytes], stop: list[bool], trie=None) -> list[bool]:
        """allowed[id] for every id: byte strings through the grammar from s; empty ids never, stop ids
        exactly in an accepting state"""
        trie = trie if trie is not None else build_trie(vocab, stop)
        out = [False] * len(vocab)
        acc = self.accepting(s)
        for i, st in enumerate(stop):
            if st:
                out[i] = acc
        todo = [(trie, s)]
        while todo:
            node, st = todo.pop()
            for c, child in node[1].items():
                t = st.copy()
                if not self.step(t, c):
                    continue
                for i in child[0]:
                    out[i] = True
                if child[1]:
                    todo.append((child, t))
        return out


def build_trie(vocab: list[bytes], stop: list[bool]):
    """node = (ids ending here, {byte: node}); stop ids and empty ids are left out"""
    root = ([], {})
    for i, b in enumerate(vocab):
        if stop[i] or not b:
            continue
        node = root
        for c in b:
            node = node[1].setdefault(c, ([], {}))
        node[0].append(i)
    return root
