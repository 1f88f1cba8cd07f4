// chat.h — the text side of the local provider: OpenAI chat-completions request parsing, the
// Llama-3 chat template, the (synthetic byte-level) tokenizer, tool-call extraction and the
// OpenAI-shaped response.  The reference outsources ALL of this to the hosted provider behind
// langchaingo (acp/internal/llmclient/langchaingo_client.go:102); the definitions used here are
// written down in DESIGN.md §3 and restated for the tests in oracle/chat_oracle.py.
#pragma once
#include <stdint.h>
#include <memory>
#include <string>
#include <vector>
#include "grammar.h"
#include "json.h"
#include "tokenizer.h"

namespace acp {

// Llama-3 special token ids (the synthetic vocabulary keeps them at their real ids)
constexpr int TOK_BEGIN_OF_TEXT = 128000;
constexpr int TOK_END_OF_TEXT = 128001;
constexpr int TOK_START_HEADER = 128006;
constexpr int TOK_END_HEADER = 128007;
constexpr int TOK_EOM = 128008;
constexpr int TOK_EOT = 128009;
constexpr int TOK_PYTHON_TAG = 128010;

struct ToolCallMsg {  // acp.MessageToolCall (acp/api/v1alpha1/task_types.go:79-97)
  std::string id, type, name, arguments;
};
struct ChatMessage {  // acp.Message (task_types.go:57-76) in its OpenAI wire form
  std::string role, content, tool_call_id, name;
  std::vector<ToolCallMsg> tool_calls;
};
struct ToolDef {  // llmclient.Tool (acp/internal/llmclient/llm_client.go:33-50)
  std::string type, name, description;
  Json parameters;
};

struct SamplingParams {
  int max_tokens = 0;       // 0 = the request set none: the engine fills in its default (engine.cc submit)
  float temperature = 0.f;  // the reference path sends temperature 0 (SURVEY.md §8c) => greedy
  int top_k = 0;
  float top_p = 1.f;
  uint64_t seed = 0;
};

struct ChatRequest {
  std::string model;
  std::vector<ChatMessage> messages;
  std::vector<ToolDef> tools;
  SamplingParams sampling;
  // "acp" extension block (test / bench hooks; never sent by the reference)
  std::vector<int> prompt_token_ids;  // bypass template + tokenizer
  std::vector<int> force_tokens;      // teacher-force the first generated tokens
  int return_logits = 0;              // keep fp32 logits of the first n sampled positions
  bool has_prompt_ids = false;
  // tool_choice "required" or {"type": "function", "function": {"name": N}}: the completion is constrained to
  // tool calls (grammar.h) of these names; null for "auto" / no tool_choice
  std::shared_ptr<const GrammarNames> grammar_names;
  bool parallel_tool_calls = true;    // false: exactly one call
};

// Parses an OpenAI chat-completions body.  Returns 0 or an HTTP-like 4xx status with *err set.
int parse_chat_request(const char* json, size_t len, ChatRequest* out, std::string* err);

// The grammar's name table for these tool names: each escaped as Json::escape_to writes it, sorted bytewise,
// duplicates dropped.  False + *err when a limit (GRAMMAR_MAX_TOOLS, GRAMMAR_MAX_NAME_BYTES) is exceeded or a
// name is not valid UTF-8 (its escaped form would not name the tool).
bool build_grammar_names(const std::vector<std::string>& names, GrammarNames* out, std::string* err);

// ---- tokenizer: see tokenizer.h; these two are the synthetic byte-level vocabulary (DESIGN.md §3.2) ----
void encode_text(const std::string& text, std::vector<int>* ids);  // one id per UTF-8 byte
std::string decode_tokens(const std::vector<int>& ids);            // total over [0, vocab)

// ---- chat template (Llama-3 headers; Llama-3.1 JSON tool calling) ----
void render_prompt(const ChatRequest& req, std::vector<int>* ids, const Tokenizer& tok = synthetic_tokenizer());
std::string render_prompt_text(const ChatRequest& req);  // specials spelled out, for tests

// ---- completion text -> assistant message ----
struct ParsedCompletion {
  std::string content;
  std::vector<ToolCallMsg> tool_calls;
};
// Tool calls are recognised as one JSON object per line: {"name": <tool>, "parameters": {...}}
// (optionally preceded by <|python_tag|>).  `arguments` is the VERBATIM substring of the
// generated text that spells the parameters object.
ParsedCompletion parse_completion(const std::string& text, const std::vector<ToolDef>& tools,
                                  const std::string& call_id_prefix);

std::string build_chat_response(uint64_t ticket, const std::string& model, const ParsedCompletion& pc,
                                const std::string& finish_reason, int prompt_tokens,
                                const std::vector<int>& completion_ids, double queue_ms,
                                double prefill_ms, double decode_ms);
std::string build_error_response(int status, const std::string& type, const std::string& message);

}  // namespace acp
