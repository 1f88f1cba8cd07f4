/* acp_host.h — C entry points of the HOST-side mirror of the reference's Go code on this path
 * (agentcontrolplane_b200/csrc/host/: llmclient + Task LLM step), plus the reconcile-loop
 * simulator used by bench.py.  JSON in, malloc'ed JSON out (release with acp_host_free).
 *
 * These live in their OWN shared library, libacp_host.so (pure C++, no CUDA, not linked against
 * libacp_infer.so): the reference arm of bench.py and the cpu_baseline load it alone.  Only provider
 * "local" reaches the engine, through the acp_infer_* C ABI looked up with dlsym at first use.
 *
 * Why this exists: the reference's host language is Go and this image has no Go toolchain, so
 * the caller side of the boundary (what acp/internal/llmclient and
 * acp/internal/controller/task do around SendRequest) is restated in C++ and exercised through
 * these hooks; the Go sources a maintainer would add are in integration/go/ (see INTEGRATION.md).
 * Nothing here needs a GPU unless an engine handle is passed.
 */
#ifndef ACP_HOST_H
#define ACP_HOST_H
#include <stddef.h>
#include "acp_infer.h"
#ifdef __cplusplus
extern "C" {
#endif

/* Releases any buffer returned by the functions below. */
void acp_host_free(void* p);

/* Chat template + tokenizer: {"text": <prompt with specials spelled out>, "token_ids": [...]}
 * for an OpenAI chat-completions body, or {"status": 4xx, "error": "..."} . */
int acp_host_render_prompt(const char* chat_request_json, size_t len, char** out_json);

/* Completion text -> assistant message: {"content": "..."} or {"tool_calls": [{id,type,
 * function:{name,arguments}}]}; tools_json = OpenAI tools array (may be NULL / "[]"). */
int acp_host_parse_completion(const char* text, size_t len, const char* tools_json,
                              const char* call_id_prefix, char** out_json);

/* Detokenizer of the synthetic vocabulary. */
int acp_host_decode_tokens(const int* ids, int n, char** out_text, size_t* out_len);

/* convertToLangchainMessages/-Tools + wire serialisation (langchaingo_client.go:118-203):
 * CRD-shaped messages + llmclient tools -> OpenAI chat-completions body. */
int acp_host_build_chat_request(const char* model, const char* messages_crd_json,
                                const char* tools_json, char** out_json);

/* convertFromLangchainResponse (langchaingo_client.go:208-282): OpenAI chat.completion body ->
 * CRD-shaped acp.Message JSON. */
int acp_host_convert_response(const char* response_json, char** out_message_crd_json);

/* One Task state-machine operation against an in-memory object store.  input_json:
 *   {"op": "sendLLMRequest" | "checkToolCalls" | "sendLLMRequestFromCluster" (validateTaskAndAgent +
 *          getLLMAndCredentials + CreateClient from the LLM CR + collectTools + the LLM step; needs
 *          "objects": [{"kind": "Agent"|"LLM"|"Secret"|"ContactChannel", "object": <CR JSON>}] and
 *          "mcp": {<server>: [<MCP tool>...]}) | "collectTools" ("agent": <Agent CR JSON>),
 *    "task": <Task CR JSON>, "tools": [<llmclient.Tool + "acpToolType">...],
 *    "toolcalls": [<ToolCall CR JSON>...]            (pre-existing objects for checkToolCalls)
 *    "llm": {"provider": "mock" | "local" | "openai" | <anything: unsupported>,
 *            "model": "...", "baseURL": "...", "maxTokens": n, "acp": {...extension...},
 *            "mock": {"message": <acp.Message>} | {"error": "text"} |
 *                    {"request_error": {"status": 400, "message": "..."}}}}
 * out_json: {"task":…, "result":{"requeue":b,"requeueAfter":s}, "error":"…", "events":[…],
 *            "toolcalls":[…], "store_writes":n, "request_json": "..." (mock/local only)} */
int acp_host_task_step(acp_engine* engine_or_null, const char* input_json, char** out_json);

/* Loopback HTTP/1.1 stub completion server (the reference tests' httptest.NewServer,
 * acp/test/e2e/getting_started/test_getting_started.go:251-262): answers every POST with `body`
 * (NULL = the reference's fixture {"id":"test-id","choices":[{"message":{"content":"test"}}]}).
 * Returns a handle >= 0 and the bound port. */
int acp_host_stub_server_start(const char* body, int* port);
void acp_host_stub_server_stop(int handle);

/* Reconcile-loop simulator: N Task CRs in phase ReadyForLLM driven through sendLLMRequest (and
 * the checkToolCalls fold-back when the scripted reply is a tool call) by `workers` concurrent
 * reconcile workers.  config_json:
 *   {"tasks": n, "workers": w, "provider": "local" | "openai", "model": "...", "baseURL": "...",
 *    "max_tokens": 64, "prompt_tokens": 512 (window rendered to exactly this many tokens),
 *    "tools": k (number of synthetic MCP tools attached), "tool_loop": bool, "seed": s,
 *    "emulate_lease": true}
 * result_json: {"reconciles": n, "wall_s": t, "reconciles_per_s": r, "step_ms_p50": …,
 *               "step_ms_p99": …, "store_writes": n, "final_phases": {...}, "digest": "…"} */
int acp_hostsim_run(acp_engine* engine_or_null, const char* config_json, char** result_json);

/* Tokenizer hooks (no GPU).  tokenizer_path = a HuggingFace tokenizer.json (or its directory);
 * NULL / "" / "synthetic" = the built-in synthetic byte-level vocabulary.
 *   encode: {"ids":[…], "pieces":[Llama-3 pre-tokenizer split of the text], "kind":…, "vocab_size":n,
 *            "special":{"begin_of_text":id, …}}   or {"error":…} with ACP_ERR_INVALID
 *   decode: raw bytes of the ids (special / unknown ids decode to nothing)
 *   render_prompt_with: acp_host_render_prompt through that tokenizer. */
int acp_host_tokenizer_encode(const char* tokenizer_path, const char* text, size_t len, char** out_json);
int acp_host_tokenizer_decode(const char* tokenizer_path, const int* ids, int n, char** out_text, size_t* out_len);
int acp_host_render_prompt_with(const char* tokenizer_path, const char* chat_request_json, size_t len, char** out_json);

/* Checkpoint inspection (no GPU): opens a HuggingFace Llama checkpoint directory the way
 * acp_infer_init {"weights": dir} does and reports
 *   {"dir":…, "config":{…config.json…}, "tensors":{"name":{"dtype","shape","nbytes"}},
 *    "model":{"hidden":…, "layers":…, "heads":…, "kv_heads":…, "ffn":…, "vocab":…, "rope_theta":…,
 *             "eps":…, "tied_embeddings":…, "max_pos":…, "experts":…,
 *             "rope_scaling": [factor, low_freq_factor, high_freq_factor, original_max_pos] | null,
 *             "weight_dtype": "bf16" | "fp8_e4m3", "rope_inv_freq":[64 floats]}}
 * max_pos is the checkpoint's max_position_embeddings (the engine serves min(max_pos, max_pages_per_seq * 32)).
 * A quantization_config other than compressed-tensors FP8_DYNAMIC (DESIGN.md §2) is refused with the field named.
 * or {"error": "..."} with return code ACP_ERR_INVALID. */
int acp_host_checkpoint_index(const char* path, char** out_json);
/* The synthetic preset `name` of acp_infer_init {"model": name} as {"model": {…the fields above…}};
 * ACP_ERR_NOT_FOUND for an unknown name. */
int acp_host_model_preset(const char* name, char** out_json);

/* The engine's split-K rule for decode GEMMs (csrc/model_config.cc, pure host logic): the number of fp32 planes of
 * out[N][M] = X[N][K] W[M][K]^T, and the workspace bytes that hold the planes of ANY step of up to max_batch rows. */
int acp_host_splitk_factor(int M, int K, int N, int target_ctas, int strict_batch_invariance);
size_t acp_host_splitk_workspace_bytes(int M, int K, int max_batch, int target_ctas, int strict_batch_invariance);
/* The same for the FP8 (e4m3) GEMMs of FP8 models, whose k-blocks hold 128 codes; K in elements. */
int acp_host_splitk_factor_fp8(int M, int K, int N, int target_ctas, int strict_batch_invariance);
size_t acp_host_splitk_workspace_bytes_fp8(int M, int K, int max_batch, int target_ctas, int strict_batch_invariance);
/* One tensor of the checkpoint as the bf16 bits the loader uploads (BF16 verbatim; F16 / F32 rounded
 * to nearest even).  out == NULL: only *n_elems is set.  ACP_ERR_NOT_FOUND: no such tensor. */
int acp_host_checkpoint_tensor_bf16(const char* path, const char* name, uint16_t* out, size_t max_elems,
                                    size_t* n_elems);

#ifdef __cplusplus
}
#endif
#endif
