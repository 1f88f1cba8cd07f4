// grammar.h — the byte-level tool-call grammar that `tool_choice: "required"` and named-function requests are
// constrained to (DESIGN.md §3.3).  One definition, compiled for the host (the scheduler advances each
// constrained sequence by the bytes of the token it emitted) and for the device (grammar_mask_kernel runs every
// vocabulary entry's bytes from the row's state).  Header-only: no CUDA runtime calls, plain inline under g++.
//
//   COMPLETION := CALL ( "\n" CALL )* STOP          (parallel_tool_calls false: CALL STOP)
//   CALL       := '{"name": ' NAME ', "parameters": ' OBJECT '}'
//   NAME       := the bytes Json::escape_to writes for an allowed tool name, quotes included
//   OBJECT     := an RFC 8259 object: strings of well-formed UTF-8 (no overlong forms, no surrogates, nothing
//                 above U+10FFFF), RFC numbers, at most GRAMMAR_MAX_DEPTH levels, whitespace runs of at most
//                 GRAMMAR_MAX_WS bytes
//   STOP       := a stop token (Tokenizer::is_stop), allowed only right after a complete CALL
//
// Every state the step function can reach is completable: numbers have no length cap, the depth cap only
// removes '{' and '[', and the whitespace cap only removes whitespace.
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define ACP_HD __host__ __device__ __forceinline__
#else
#define ACP_HD inline
#endif

namespace acp {

constexpr int GRAMMAR_MAX_TOOLS = 128;
constexpr int GRAMMAR_MAX_NAME_BYTES = 8192;   // escaped names, quotes included, all tools together
constexpr int GRAMMAR_MAX_DEPTH = 32;
constexpr int GRAMMAR_MAX_WS = 32;

// The allowed names of one request, escaped and sorted bytewise (no duplicates).  Names consistent with the
// bytes of a NAME so far are then a contiguous index range.
struct GrammarNames {
  int32_t n;
  uint16_t off[GRAMMAR_MAX_TOOLS + 1];          // name i = bytes[off[i], off[i + 1])
  uint8_t bytes[GRAMMAR_MAX_NAME_BYTES];
};

enum : uint8_t { G_PREFIX, G_NAME, G_MID, G_ROOT, G_JSON, G_CLOSE, G_AFTER };
enum : uint8_t {
  J_VALUE, J_OBJ_FIRST, J_OBJ_KEY, J_COLON, J_AFTER, J_ARR_FIRST, J_STR, J_ESC, J_HEX, J_UTF8, J_LIT,
  J_NUM_MINUS, J_NUM_ZERO, J_NUM_INT, J_NUM_DOT, J_NUM_FRAC, J_NUM_E, J_NUM_ESIGN, J_NUM_EXP
};
enum : uint8_t { GF_PARALLEL = 1, GF_KEY = 2 };

struct GrammarState {
  uint8_t phase, js;   // G_* ; J_* while phase == G_JSON
  uint8_t depth, ws;   // open containers; length of the current whitespace run
  uint8_t cnt;         // literal offset / hex digits left / UTF-8 continuation bytes left
  uint8_t lo8, hi8;    // range of the next UTF-8 continuation byte
  uint8_t flags;       // GF_*
  uint8_t lit, pad_;   // J_LIT: 0 true, 1 false, 2 null
  uint16_t lo, hi, off;  // G_NAME: names [lo, hi) match the `off` bytes seen so far
  uint32_t stack;      // bit d: container at level d is an object (else an array)
};

ACP_HD void grammar_init(GrammarState* s, int n_names, bool parallel) {
  *s = GrammarState();
  s->phase = G_PREFIX;
  s->hi = (uint16_t)n_names;
  s->flags = parallel ? GF_PARALLEL : 0;
}

// A stop token is allowed exactly here.
ACP_HD bool grammar_accepting(const GrammarState& s) { return s.phase == G_AFTER; }

ACP_HD bool grammar_is_ws(uint8_t c) { return c == ' ' || c == '\n' || c == '\t' || c == '\r'; }
ACP_HD bool grammar_is_digit(uint8_t c) { return c >= '0' && c <= '9'; }

// Closes the innermost container.
ACP_HD void grammar_pop(GrammarState& s) {
  --s.depth;
  if (s.depth == 0) s.phase = G_CLOSE;
  else s.js = J_AFTER;
}

// A value starts with c (J_VALUE, or J_ARR_FIRST on anything but ']').
ACP_HD bool grammar_value(GrammarState& s, uint8_t c) {
  switch (c) {
    case '{':
    case '[':
      if (s.depth >= GRAMMAR_MAX_DEPTH) return false;
      if (c == '{') s.stack |= 1u << s.depth; else s.stack &= ~(1u << s.depth);
      ++s.depth;
      s.js = c == '{' ? J_OBJ_FIRST : J_ARR_FIRST;
      return true;
    case '"': s.js = J_STR; s.flags &= ~GF_KEY; return true;
    case 't': s.js = J_LIT; s.lit = 0; s.cnt = 1; return true;
    case 'f': s.js = J_LIT; s.lit = 1; s.cnt = 1; return true;
    case 'n': s.js = J_LIT; s.lit = 2; s.cnt = 1; return true;
    case '-': s.js = J_NUM_MINUS; return true;
    case '0': s.js = J_NUM_ZERO; return true;
    default:
      if (c >= '1' && c <= '9') { s.js = J_NUM_INT; return true; }
      return false;
  }
}

// The structural states: whitespace, values, ',', ':', closers.
ACP_HD bool grammar_struct(GrammarState& s, uint8_t c) {
  if (grammar_is_ws(c)) {
    if (s.ws >= GRAMMAR_MAX_WS) return false;
    ++s.ws;
    return true;
  }
  s.ws = 0;
  switch (s.js) {
    case J_VALUE: return grammar_value(s, c);
    case J_ARR_FIRST:
      if (c == ']') { grammar_pop(s); return true; }
      return grammar_value(s, c);
    case J_OBJ_FIRST:
      if (c == '}') { grammar_pop(s); return true; }
      if (c == '"') { s.js = J_STR; s.flags |= GF_KEY; return true; }
      return false;
    case J_OBJ_KEY:
      if (c == '"') { s.js = J_STR; s.flags |= GF_KEY; return true; }
      return false;
    case J_COLON:
      if (c == ':') { s.js = J_VALUE; return true; }
      return false;
    default: {  // J_AFTER
      const bool obj = (s.stack >> (s.depth - 1)) & 1u;
      if (c == ',') { s.js = obj ? J_OBJ_KEY : J_VALUE; return true; }
      if (c == (obj ? '}' : ']')) { grammar_pop(s); return true; }
      return false;
    }
  }
}

// Advances s by one byte; false = the byte is not allowed here (s is then unspecified).
ACP_HD bool grammar_step(GrammarState& s, uint8_t c, const GrammarNames& names) {
  switch (s.phase) {
    case G_PREFIX: {
      const char* lit = "{\"name\": ";
      if (c != (uint8_t)lit[s.cnt]) return false;
      if (++s.cnt == 9) { s.phase = G_NAME; s.off = 0; s.lo = 0; s.hi = (uint16_t)names.n; s.cnt = 0; }
      return true;
    }
    case G_NAME: {
      // every name in [lo, hi) is longer than off; keep those whose byte at off is c
      int lo = s.lo, hi = s.hi;
      while (lo < hi && names.bytes[names.off[lo] + s.off] < c) ++lo;
      int e = lo;
      while (e < hi && names.bytes[names.off[e] + s.off] == c) ++e;
      if (e == lo) return false;
      s.lo = (uint16_t)lo; s.hi = (uint16_t)e;
      ++s.off;
      // the closing quote is the only unescaped quote of an escaped name: a name that ends here is the only match
      if (names.off[lo + 1] - names.off[lo] == s.off) { s.phase = G_MID; s.cnt = 0; }
      return true;
    }
    case G_MID: {
      const char* lit = ", \"parameters\": ";
      if (c != (uint8_t)lit[s.cnt]) return false;
      if (++s.cnt == 16) { s.phase = G_ROOT; s.cnt = 0; }
      return true;
    }
    case G_ROOT:
      if (c != '{') return false;
      s.phase = G_JSON; s.js = J_OBJ_FIRST; s.depth = 1; s.stack = 1u; s.ws = 0;
      return true;
    case G_CLOSE:
      if (c != '}') return false;
      s.phase = G_AFTER;
      return true;
    case G_AFTER:
      if (c != '\n' || !(s.flags & GF_PARALLEL)) return false;
      s.phase = G_PREFIX; s.cnt = 0;
      return true;
    case G_JSON: break;
    default: return false;
  }
  switch (s.js) {
    case J_STR:
      if (c == '"') { s.js = (s.flags & GF_KEY) ? J_COLON : J_AFTER; return true; }
      if (c == '\\') { s.js = J_ESC; return true; }
      if (c < 0x20) return false;
      if (c < 0x80) return true;
      s.lo8 = 0x80; s.hi8 = 0xBF;
      if (c >= 0xC2 && c <= 0xDF) s.cnt = 1;
      else if (c >= 0xE0 && c <= 0xEF) {
        s.cnt = 2;
        if (c == 0xE0) s.lo8 = 0xA0;        // no overlong 3-byte forms
        else if (c == 0xED) s.hi8 = 0x9F;   // no surrogates
      } else if (c >= 0xF0 && c <= 0xF4) {
        s.cnt = 3;
        if (c == 0xF0) s.lo8 = 0x90;        // no overlong 4-byte forms
        else if (c == 0xF4) s.hi8 = 0x8F;   // nothing above U+10FFFF
      } else return false;
      s.js = J_UTF8;
      return true;
    case J_UTF8:
      if (c < s.lo8 || c > s.hi8) return false;
      s.lo8 = 0x80; s.hi8 = 0xBF;
      if (--s.cnt == 0) s.js = J_STR;
      return true;
    case J_ESC:
      if (c == 'u') { s.js = J_HEX; s.cnt = 4; return true; }
      if (c == '"' || c == '\\' || c == '/' || c == 'b' || c == 'f' || c == 'n' || c == 'r' || c == 't') { s.js = J_STR; return true; }
      return false;
    case J_HEX:
      if (!(grammar_is_digit(c) || (c >= 'a' && c <= 'f') || (c >= 'A' && c <= 'F'))) return false;
      if (--s.cnt == 0) s.js = J_STR;
      return true;
    case J_LIT: {
      const char* lit = s.lit == 0 ? "true" : s.lit == 1 ? "false" : "null";
      if (c != (uint8_t)lit[s.cnt]) return false;
      ++s.cnt;
      if (lit[s.cnt] == 0) s.js = J_AFTER;
      return true;
    }
    case J_NUM_MINUS:
      if (c == '0') { s.js = J_NUM_ZERO; return true; }
      if (c >= '1' && c <= '9') { s.js = J_NUM_INT; return true; }
      return false;
    case J_NUM_DOT:
      if (grammar_is_digit(c)) { s.js = J_NUM_FRAC; return true; }
      return false;
    case J_NUM_E:
      if (c == '+' || c == '-') { s.js = J_NUM_ESIGN; return true; }
      if (grammar_is_digit(c)) { s.js = J_NUM_EXP; return true; }
      return false;
    case J_NUM_ESIGN:
      if (grammar_is_digit(c)) { s.js = J_NUM_EXP; return true; }
      return false;
    case J_NUM_ZERO:
    case J_NUM_INT:
    case J_NUM_FRAC:
    case J_NUM_EXP:
      if (grammar_is_digit(c) && s.js != J_NUM_ZERO) return true;
      if (c == '.' && (s.js == J_NUM_ZERO || s.js == J_NUM_INT)) { s.js = J_NUM_DOT; return true; }
      if ((c == 'e' || c == 'E') && s.js != J_NUM_EXP) { s.js = J_NUM_E; return true; }
      s.js = J_AFTER;   // the number ended: c is the byte after it
      return grammar_struct(s, c);
    default:
      return grammar_struct(s, c);
  }
}

// Host and device view of the vocabulary: id -> the bytes Tokenizer::decode({id}) gives; stop ids flagged.
struct GrammarVocab {
  int vocab = 0;
  const int32_t* off = nullptr;    // [vocab + 1]
  const uint8_t* bytes = nullptr;  // [off[vocab]]
  const uint8_t* stop = nullptr;   // [vocab]
};

// Whether token `id` may follow state s.  Ids that decode to nothing are never allowed, except stop ids in an
// accepting state.
ACP_HD bool grammar_token_allowed(const GrammarState& s, const GrammarVocab& v, int id, const GrammarNames& names) {
  if (v.stop[id]) return grammar_accepting(s);
  const int b = v.off[id], e = v.off[id + 1];
  if (b == e) return false;
  GrammarState t = s;
  for (int i = b; i < e; ++i)
    if (!grammar_step(t, v.bytes[i], names)) return false;
  return true;
}

// One constrained row of a step: which sampled row, which name table, and the state its emitted prefix reached.
struct GrammarRow {
  int32_t row;    // index into the step's sampled rows
  int32_t slot;   // name-table slot of the sequence
  GrammarState state;
};

}  // namespace acp
