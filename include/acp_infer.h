/* acp_infer.h — C ABI of libacp_infer.so, the H100-native `provider: local` for ACP.
 *
 * This is the drop-in boundary for ONE path of humanlayer/agentcontrolplane: the Task reconciler's
 * per-step LLM call.  Everything the reference sends over HTTPS at
 *     acp/internal/llmclient/langchaingo_client.go:102   (c.model.GenerateContent)
 * crosses this header instead; the Go side keeps `llmclient.LLMClient.SendRequest`
 * (acp/internal/llmclient/llm_client.go:11-14) unchanged.  INTEGRATION.md shows the cgo shim
 * (acp/internal/inference) and the `case "local"` arm of NewLangchainClient
 * (langchaingo_client.go:31-73) that bind these symbols.
 *
 * Wire format: the request is the SAME OpenAI chat-completions JSON body langchaingo's openai
 * provider POSTs to {baseURL}/chat/completions (model, messages[{role, content, tool_calls,
 * tool_call_id}], tools[], tool_choice, parallel_tool_calls, temperature, max_tokens, top_p, seed); the response is an OpenAI
 * chat.completion JSON (choices[0].message.{content | tool_calls}, usage) plus an "acp" object
 * with the emitted token ids.  Status codes follow HTTP: 200 ok, 4xx = request is invalid and
 * must not be retried (maps to llmclient.LLMRequestError, llm_client.go:18-30, which
 * handleLLMError turns into phase Failed, controller/task/state_machine.go:733-790), 5xx =
 * transient (plain error => requeue after 5 s).
 *
 * Conventions: every function except acp_infer_shutdown is thread-safe and callable from any OS
 * thread (cgo); acp_infer_shutdown frees the handle and must not overlap any other call on it
 * (stop the poller first: integration/go/inference Shutdown); no function
 * throws; return value 0 = success, negative = ACP_ERR_*; out-buffers are malloc'ed by the
 * library and released with acp_infer_free(); the library never keeps a caller pointer after
 * the call returns (cgo pointer-passing rule).  There is NO CPU fallback: without a usable CUDA
 * device acp_infer_init fails with ACP_ERR_CUDA.
 */
#ifndef ACP_INFER_H
#define ACP_INFER_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define ACP_OK 0
#define ACP_ERR_INVALID (-1)    /* bad argument / malformed config                            */
#define ACP_ERR_NOT_FOUND (-2)  /* unknown ticket                                             */
#define ACP_ERR_TIMEOUT (-3)    /* wait/poll timed out (not an error of the request)          */
#define ACP_ERR_NOMEM (-4)      /* host or device allocation failed                           */
#define ACP_ERR_CUDA (-5)       /* CUDA runtime / device failure, or no device                */
#define ACP_ERR_SHUTDOWN (-6)   /* engine is shutting down                                    */
#define ACP_ERR_PENDING (-7)    /* result requested before the ticket finished                */

typedef struct acp_engine acp_engine;

/* Once per process (per GPU): generate/load weights into HBM, allocate the paged KV pool, start
 * the scheduler thread.  Replaces per-reconcile client construction in
 * llmclient.NewLangchainClient (langchaingo_client.go:27-80): the Go `local` client is a
 * zero-cost handle onto this singleton.  config_json keys (all optional):
 *   "model": "llama-3-8b" | "llama-3-8b-l2" | "llama-3-70b" | "tiny" | "tiny-g2"
 *            | "<dense single-GPU preset>-fp8" (llama-3-8b-fp8, llama-3-8b-l2-fp8, tiny-fp8, tiny-g2-fp8,
 *              tiny-g8-fp8): the same synthetic weights with the four layer projections quantised to e4m3
 *              (per-row weight scales, per-token activation scales; DESIGN.md §5); acp_infer_stats reports
 *              "weight_dtype"
 *            | "tiny-3.1" | "llama-3.1-8b-l2" | "llama-3.1-8b" (and their -fp8 forms): the shapes and weights of
 *              tiny / llama-3-8b-l2 / llama-3-8b with Llama-3.1's "llama3" RoPE scaling (factor 8, low 1,
 *              high 4, original 8192) and a 131072-token window
 *   "weights": "synthetic" (seeded generator, default) | "<dir>" = HuggingFace Llama checkpoint
 *              (config.json + model.safetensors or model.safetensors.index.json + shards; BF16/F16/F32;
 *              or compressed-tensors FP8_DYNAMIC: F8_E4M3 projections with per-channel or per-tensor
 *              weight_scale, served on the FP8 GEMMs, one GPU; DESIGN.md §2;
 *              "model" is then just the name requests must carry, default = the directory name)
 *   "seed": 11317760                  (0xACB200)
 *   "device": 0, "max_batch": 256, "max_tokens_per_step": 8192, "kv_pages": 2048,
 *   "max_pages_per_seq": 256 (KV pages of 32 tokens one sequence may hold: its context, prompt + max_tokens, is
 *              limited to min(max_pages_per_seq * 32, the model's max_position_embeddings), beyond which a request
 *              gets 400 context_length_exceeded; 4096 serves Llama-3.1's 131072 tokens.  Raise kv_pages with it:
 *              the pool is shared by all sequences.  The decode attention workspace grows with
 *              max_batch x max_pages_per_seq, DESIGN.md §2),
 *   "prefix_cache": true, "tp": 1 (tensor-parallel GPUs of THIS process),
 *   "tp_comm": "p2p" | "nccl", "layers": n (truncated depth, dev only),
 *   "request_timeout_ms": n (0 = none): a request older than this, queued or running, ends with status 504
 *              (transient: plain error upstream => the Task is requeued, state_machine.go:757-789),
 *   "replicas": n (1..16): n data-parallel engines on GPUs device, device+tp, ... behind THIS handle;
 *              requests are routed stickily (OpenAI `user` field, else a hash of the first two
 *              messages, else round-robin) so a Task's turns find their retained K/V; tickets are
 *              global; acp_infer_stats sums the additive counters and lists per-replica objects */
int acp_infer_init(const char* config_json, acp_engine** out);

/* Non-blocking submit of one chat-completions request (what SendRequest does at
 * langchaingo_client.go:83-102).  On success *ticket identifies the request.  Requests that are
 * invalid still get a ticket; their result carries the 4xx status. */
int acp_infer_submit(acp_engine* e, const char* chat_request_json, size_t len, uint64_t* ticket);

/* Block until `ticket` finishes or timeout_ms elapses (timeout_ms < 0: forever). */
int acp_infer_wait(acp_engine* e, uint64_t ticket, int timeout_ms);

/* Collect up to `max` finished tickets that no poll has reported yet; returns the count
 * (possibly 0 after timeout_ms).  One Go poller goroutine can serve every blocked SendRequest
 * without pinning an OS thread per request. */
int acp_infer_poll(acp_engine* e, uint64_t* tickets, int max, int timeout_ms);

/* Fetch the finished response: *chat_response_json (malloc'ed, NUL-terminated), *len,
 * *http_like_status.  The ticket is consumed. */
int acp_infer_result(acp_engine* e, uint64_t ticket, char** chat_response_json, size_t* len,
                     int* http_like_status);

/* fp32 logits kept for the first `acp.return_logits` sampled positions of a finished ticket
 * (parity tests).  Must be called BEFORE acp_infer_result.  Returns the number of positions
 * copied (each `vocab` floats) or a negative error.  For a request constrained by tool_choice
 * "required" or a named function these are the MASKED logits the sampler saw: -inf for every id
 * the tool-call grammar rejects at that position (DESIGN.md §3.3). */
int acp_infer_result_logits(acp_engine* e, uint64_t ticket, float* out, int max_positions);

/* ctx.Done(): drop a queued or running request; its result reports status 499. */
void acp_infer_cancel(acp_engine* e, uint64_t ticket);

/* Engine counters as JSON (malloc'ed): steps, tokens, device-timed decode/prefill milliseconds,
 * kernel launches, algorithmic bytes per decode step, KV pool occupancy. */
int acp_infer_stats(acp_engine* e, char** json);
/* Zero the counters (bench warm-up boundary). */
void acp_infer_stats_reset(acp_engine* e);

void acp_infer_free(void* p);
/* Ends every queued / running request with status 503 (each is reported once more through
 * acp_infer_poll so that parked waiters wake), joins the scheduler, frees device memory and the
 * handle.  Must not run concurrently with any other call on `e`. */
void acp_infer_shutdown(acp_engine* e);

/* Library build info: "acp_infer <version> sm_90a". */
const char* acp_infer_version(void);

#ifdef __cplusplus
}
#endif
#endif /* ACP_INFER_H */
