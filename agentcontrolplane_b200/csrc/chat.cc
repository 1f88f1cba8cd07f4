// chat.cc — see chat.h.  Host-only code (no CUDA).
#include "chat.h"
#include <string.h>
#include <time.h>
#include <algorithm>

namespace acp {

static const char* kToolPreamble =
    "Given the following functions, please respond with a JSON for a function call with its "
    "proper arguments that best answers the given prompt.\n\nRespond in the format {\"name\": "
    "function name, \"parameters\": dictionary of argument name and its value}. Do not use "
    "variables.\n\n";

// ---------------------------------------------------------------------------------
// request parsing
// ---------------------------------------------------------------------------------
static std::string content_to_text(const Json& c) {
  if (c.is_string()) return c.as_string();
  if (c.is_array()) {  // OpenAI content parts: concatenate the text parts
    std::string out;
    for (const Json& part : c.items()) {
      if (part.is_object() && part.get("type").as_string() == "text") out += part.get("text").as_string();
      else if (part.is_string()) out += part.as_string();
    }
    return out;
  }
  return std::string();  // null / absent
}

int parse_chat_request(const char* json, size_t len, ChatRequest* out, std::string* err) {
  Json root;
  std::string perr;
  if (!Json::parse(json, len, &root, &perr)) { *err = "invalid JSON body: " + perr; return 400; }
  if (!root.is_object()) { *err = "request body must be a JSON object"; return 400; }
  ChatRequest r;
  r.model = root.get("model").as_string();
  if (root.get("stream").as_bool(false)) { *err = "stream=true is not supported by provider local"; return 400; }
  if (root.find("n") && root.get("n").as_int(1) != 1) { *err = "n must be 1"; return 400; }
  // Parameters that would change the completion but are not implemented are refused, never silently
  // ignored (the reference's SendRequest sets none of them: langchaingo_client.go:83-102).
  {
    const Json& stop = root.get("stop");
    if ((stop.is_string() && !stop.as_string().empty()) || (stop.is_array() && stop.size() > 0)) {
      *err = "stop sequences are not supported by provider local";
      return 400;
    }
    if (root.get("logprobs").as_bool(false)) { *err = "logprobs are not supported by provider local"; return 400; }
    for (const char* pen : {"frequency_penalty", "presence_penalty"})
      if (root.get(pen).as_double(0.0) != 0.0) { *err = std::string(pen) + " is not supported by provider local"; return 400; }
    const Json& rf = root.get("response_format");
    if (rf.is_object() && !rf.get("type").as_string().empty() && rf.get("type").as_string() != "text") {
      *err = "response_format other than text is not supported by provider local";
      return 400;
    }
  }

  const Json& acp = root.get("acp");
  if (acp.is_object()) {
    const Json& pti = acp.get("prompt_token_ids");
    if (pti.is_array()) {
      r.has_prompt_ids = true;
      for (const Json& t : pti.items()) r.prompt_token_ids.push_back((int)t.as_int(-1));
    }
    for (const Json& t : acp.get("force_tokens").items()) r.force_tokens.push_back((int)t.as_int(-1));
    r.return_logits = (int)acp.get("return_logits").as_int(0);
  }

  const Json& msgs = root.get("messages");
  if (!msgs.is_array() || msgs.size() == 0) {
    if (!r.has_prompt_ids) { *err = "messages must be a non-empty array"; return 400; }
  }
  for (const Json& m : msgs.items()) {
    if (!m.is_object()) { *err = "each message must be an object"; return 400; }
    ChatMessage cm;
    cm.role = m.get("role").as_string();
    if (cm.role.empty()) { *err = "message.role is required"; return 400; }
    cm.content = content_to_text(m.get("content"));
    cm.tool_call_id = m.get("tool_call_id").as_string();
    cm.name = m.get("name").as_string();
    for (const Json& tc : m.get("tool_calls").items()) {
      ToolCallMsg t;
      t.id = tc.get("id").as_string();
      t.type = tc.get("type").as_string();
      const Json& fn = tc.get("function");
      t.name = fn.get("name").as_string();
      const Json& args = fn.get("arguments");
      t.arguments = args.is_string() ? args.as_string() : (args.is_null() ? std::string() : args.dump());
      cm.tool_calls.push_back(std::move(t));
    }
    r.messages.push_back(std::move(cm));
  }
  for (const Json& t : root.get("tools").items()) {
    if (!t.is_object()) { *err = "each tool must be an object"; return 400; }
    ToolDef td;
    td.type = t.get("type").as_string();
    if (td.type.empty()) td.type = "function";
    const Json& fn = t.get("function");
    td.name = fn.get("name").as_string();
    if (td.name.empty()) { *err = "tool.function.name is required"; return 400; }
    td.description = fn.get("description").as_string();
    td.parameters = fn.get("parameters");
    r.tools.push_back(std::move(td));
  }
  // tool_choice: "auto" (or none) samples freely; "required" and a named function constrain the completion to
  // tool calls with a grammar enforced on the GPU (grammar.h, DESIGN.md §3.3)
  {
    const Json& tc = root.get("tool_choice");
    std::vector<std::string> allowed;
    const bool constrained = !(tc.is_null() || (tc.is_string() && tc.as_string() == "auto"));
    if (!constrained) {
    } else if (tc.is_string() && tc.as_string() == "required") {
      for (const ToolDef& t : r.tools) allowed.push_back(t.name);
    } else if (tc.is_object()) {
      const Json& fn = tc.get("function");
      if (tc.get("type").as_string() != "function" || !fn.is_object() || !fn.get("name").is_string() ||
          fn.get("name").as_string().empty()) {
        *err = "tool_choice object must be {\"type\": \"function\", \"function\": {\"name\": <tool name>}}";
        return 400;
      }
      const std::string name = fn.get("name").as_string();
      bool known = false;
      for (const ToolDef& t : r.tools) known = known || t.name == name;
      if (!r.tools.empty() && !known) { *err = "tool_choice names function '" + name + "', which is not among the request's tools"; return 400; }
      allowed.push_back(name);
    } else {
      *err = "tool_choice " + tc.dump() + " is not supported by provider local (served: \"auto\", \"required\", a named function)";
      return 400;
    }
    if (constrained) {
      if (r.tools.empty()) { *err = "tool_choice other than \"auto\" needs a non-empty tools list"; return 400; }
      auto names = std::make_shared<GrammarNames>();
      std::string gerr;
      if (!build_grammar_names(allowed, names.get(), &gerr)) { *err = "tool_choice: " + gerr; return 400; }
      r.grammar_names = std::move(names);
      r.parallel_tool_calls = root.get("parallel_tool_calls").as_bool(true);
    }
  }
  SamplingParams& sp = r.sampling;
  for (const char* key : {"max_completion_tokens", "max_tokens"}) {
    const Json* mt = root.find(key);
    if (!mt || mt->is_null()) continue;
    const long long v = mt->as_int(0);
    if (v <= 0) { *err = "max_tokens must be positive"; return 400; }
    sp.max_tokens = (int)(v > 1000000000LL ? 1000000000LL : v);
  }
  if (root.find("temperature") && !root.get("temperature").is_null()) sp.temperature = (float)root.get("temperature").as_double(0.0);
  if (sp.temperature < 0.f) { *err = "temperature must be >= 0"; return 400; }
  if (root.find("top_p") && !root.get("top_p").is_null()) sp.top_p = (float)root.get("top_p").as_double(1.0);
  if (sp.top_p <= 0.f || sp.top_p > 1.f) { *err = "top_p must be in (0, 1]"; return 400; }
  if (root.find("top_k") && !root.get("top_k").is_null()) sp.top_k = (int)root.get("top_k").as_int(0);
  if (root.find("seed") && !root.get("seed").is_null()) sp.seed = (uint64_t)root.get("seed").as_int(0);
  *out = std::move(r);
  return 0;
}

bool build_grammar_names(const std::vector<std::string>& names, GrammarNames* out, std::string* err) {
  std::vector<std::string> esc;
  for (const std::string& n : names) {
    std::string e;
    Json::escape_to(n, e);
    Json back;
    std::string perr;
    if (!Json::parse(e, &back, &perr) || back.as_string() != n) { *err = "tool name is not valid UTF-8"; return false; }
    esc.push_back(std::move(e));
  }
  std::sort(esc.begin(), esc.end());
  esc.erase(std::unique(esc.begin(), esc.end()), esc.end());
  if ((int)esc.size() > GRAMMAR_MAX_TOOLS) {
    *err = std::to_string(esc.size()) + " tool names exceed the limit of " + std::to_string(GRAMMAR_MAX_TOOLS);
    return false;
  }
  size_t total = 0;
  for (const std::string& e : esc) total += e.size();
  if (total > (size_t)GRAMMAR_MAX_NAME_BYTES) {
    *err = "tool names take " + std::to_string(total) + " bytes escaped, over the limit of " + std::to_string(GRAMMAR_MAX_NAME_BYTES);
    return false;
  }
  memset(out, 0, sizeof *out);
  out->n = (int32_t)esc.size();
  size_t at = 0;
  for (size_t i = 0; i < esc.size(); ++i) {
    out->off[i] = (uint16_t)at;
    memcpy(out->bytes + at, esc[i].data(), esc[i].size());
    at += esc[i].size();
  }
  out->off[esc.size()] = (uint16_t)at;
  return true;
}

// ---------------------------------------------------------------------------------
// tokenizer
// ---------------------------------------------------------------------------------
void encode_text(const std::string& text, std::vector<int>* ids) { synthetic_tokenizer().encode(text, ids); }
std::string decode_tokens(const std::vector<int>& ids) { return synthetic_tokenizer().decode(ids); }

// ---------------------------------------------------------------------------------
// chat template
// ---------------------------------------------------------------------------------
namespace {
struct Emitter {
  std::vector<int>* ids;   // either token ids ...
  std::string* text;       // ... or the spelled-out string
  const Tokenizer* tok;
  std::string pending;     // ordinary text since the last special token: encoded as ONE string, as a
                           // tokenizer that splits the rendered prompt at special tokens would
  void flush() {
    if (ids && !pending.empty()) tok->encode(pending, ids);
    pending.clear();
  }
  void special(int id, const char* spelled) {
    flush();
    if (ids) ids->push_back(id);
    if (text) *text += spelled;
  }
  void bytes(const std::string& s) {
    if (ids) pending += s;
    if (text) *text += s;
  }
  void header(const char* role) {
    special(tok->special().start_header, "<|start_header_id|>");
    bytes(role);
    special(tok->special().end_header, "<|end_header_id|>");
    bytes("\n\n");
  }
  void eot() { special(tok->special().eot, "<|eot_id|>"); }
};

std::string tool_json(const ToolDef& t) {
  Json fn = Json::object();
  fn.set("name", Json(t.name));
  fn.set("description", Json(t.description));
  fn.set("parameters", t.parameters.is_null() ? Json::object() : t.parameters);
  Json o = Json::object();
  o.set("type", Json(t.type));
  o.set("function", fn);
  return o.dump();
}

void render(const ChatRequest& req, Emitter& e) {
  e.special(e.tok->special().begin_of_text, "<|begin_of_text|>");
  size_t idx = 0;
  std::string sys;
  if (!req.messages.empty() && req.messages[0].role == "system") { sys = req.messages[0].content; idx = 1; }
  const bool has_tools = !req.tools.empty();
  if (!sys.empty() || has_tools) {
    e.header("system");
    e.bytes(std::string(has_tools ? "Environment: ipython\n\n" : "") + sys);
    e.eot();
  }
  bool first_user = true;
  for (; idx < req.messages.size(); ++idx) {
    const ChatMessage& m = req.messages[idx];
    if (m.role == "assistant") {
      e.header("assistant");
      if (!m.tool_calls.empty()) {
        std::string body;
        for (size_t i = 0; i < m.tool_calls.size(); ++i) {
          if (i) body += "\n";
          std::string name_json;
          Json::escape_to(m.tool_calls[i].name, name_json);
          body += "{\"name\": " + name_json + ", \"parameters\": " +
                  (m.tool_calls[i].arguments.empty() ? std::string("{}") : m.tool_calls[i].arguments) + "}";
        }
        e.bytes(body);
      } else {
        e.bytes(m.content);
      }
      e.eot();
    } else if (m.role == "tool") {
      e.header("ipython");
      e.bytes(m.content);
      e.eot();
    } else if (m.role == "system") {
      e.header("system");
      e.bytes(m.content);
      e.eot();
    } else {  // "user", and unknown roles map to user like convertToLangchainMessages' default arm
      e.header("user");
      if (has_tools && first_user) {
        std::string body = kToolPreamble;
        for (size_t i = 0; i < req.tools.size(); ++i) body += tool_json(req.tools[i]) + "\n\n";
        body += m.content;
        e.bytes(body);
      } else {
        e.bytes(m.content);
      }
      first_user = false;
      e.eot();
    }
  }
  e.header("assistant");
  e.flush();
}
}  // namespace

void render_prompt(const ChatRequest& req, std::vector<int>* ids, const Tokenizer& tok) {
  Emitter e{ids, nullptr, &tok, std::string()};
  render(req, e);
}
std::string render_prompt_text(const ChatRequest& req) {
  std::string s;
  Emitter e{nullptr, &s, &synthetic_tokenizer(), std::string()};
  render(req, e);
  return s;
}

// ---------------------------------------------------------------------------------
// completion parsing
// ---------------------------------------------------------------------------------
static bool is_ws(char c) { return c == ' ' || c == '\n' || c == '\t' || c == '\r'; }

ParsedCompletion parse_completion(const std::string& text, const std::vector<ToolDef>& tools,
                                  const std::string& call_id_prefix) {
  ParsedCompletion pc;
  if (!tools.empty()) {
    std::vector<ToolCallMsg> calls;
    size_t pos = 0;
    const size_t n = text.size();
    bool ok = true;
    while (true) {
      while (pos < n && is_ws(text[pos])) ++pos;
      if (pos >= n) break;
      if (text[pos] != '{') { ok = false; break; }
      Json obj;
      std::string err;
      size_t end = 0;
      std::vector<Json::MemberSpan> spans;
      if (!Json::parse(text.data() + pos, n - pos, &obj, &err, &end, true, &spans) || !obj.is_object()) { ok = false; break; }
      const std::string name = obj.get("name").as_string();
      bool known = false;
      for (const ToolDef& t : tools) if (t.name == name) known = true;
      const char* key = obj.find("parameters") ? "parameters" : "arguments";
      const Json& params = obj.get(key);
      if (!known || !params.is_object()) { ok = false; break; }
      ToolCallMsg tc;
      tc.type = "function";
      tc.name = name;
      for (const auto& sp : spans)
        if (sp.key == key) tc.arguments = text.substr(pos + sp.begin, sp.end - sp.begin);  // verbatim
      tc.id = call_id_prefix + std::to_string(calls.size());
      calls.push_back(std::move(tc));
      pos += end;
    }
    if (ok && !calls.empty()) { pc.tool_calls = std::move(calls); return pc; }
  }
  pc.content = text;
  return pc;
}

// ---------------------------------------------------------------------------------
// responses
// ---------------------------------------------------------------------------------
std::string build_chat_response(uint64_t ticket, const std::string& model, const ParsedCompletion& pc,
                                const std::string& finish_reason, int prompt_tokens,
                                const std::vector<int>& completion_ids, double queue_ms,
                                double prefill_ms, double decode_ms) {
  Json msg = Json::object();
  msg.set("role", Json("assistant"));
  if (!pc.tool_calls.empty()) {
    msg.set("content", Json());
    Json tcs = Json::array();
    for (const ToolCallMsg& t : pc.tool_calls) {
      Json fn = Json::object();
      fn.set("name", Json(t.name));
      fn.set("arguments", Json(t.arguments));
      Json o = Json::object();
      o.set("id", Json(t.id));
      o.set("type", Json("function"));
      o.set("function", fn);
      tcs.push(o);
    }
    msg.set("tool_calls", tcs);
  } else {
    msg.set("content", Json(pc.content));
  }
  Json choice = Json::object();
  choice.set("index", Json(0));
  choice.set("message", msg);
  choice.set("finish_reason", Json(pc.tool_calls.empty() ? finish_reason : std::string("tool_calls")));
  Json choices = Json::array();
  choices.push(choice);
  Json usage = Json::object();
  usage.set("prompt_tokens", Json(prompt_tokens));
  usage.set("completion_tokens", Json((int)completion_ids.size()));
  usage.set("total_tokens", Json(prompt_tokens + (int)completion_ids.size()));
  Json ext = Json::object();
  Json ids = Json::array();
  for (int t : completion_ids) ids.push(Json(t));
  ext.set("token_ids", ids);
  ext.set("queue_ms", Json(queue_ms));
  ext.set("prefill_ms", Json(prefill_ms));
  ext.set("decode_ms", Json(decode_ms));
  Json root = Json::object();
  root.set("id", Json("chatcmpl-" + std::to_string(ticket)));
  root.set("object", Json("chat.completion"));
  root.set("created", Json((long long)time(nullptr)));
  root.set("model", Json(model));
  root.set("choices", choices);
  root.set("usage", usage);
  root.set("acp", ext);
  return root.dump();
}

std::string build_error_response(int status, const std::string& type, const std::string& message) {
  Json e = Json::object();
  e.set("message", Json(message));
  e.set("type", Json(type));
  e.set("code", Json(status));
  Json root = Json::object();
  root.set("error", e);
  return root.dump();
}

}  // namespace acp
