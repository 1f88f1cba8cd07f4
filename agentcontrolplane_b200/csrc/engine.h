// engine.h — continuous-batching scheduler of the local provider (one per GPU).
//
// Many concurrent LLMClient.SendRequest callers (Task.Reconcile goroutines in the reference,
// acp/internal/controller/task/state_machine.go:238) submit chat requests; ONE scheduler thread
// coalesces them into prefill / decode steps over the paged KV pool and runs Model::forward.
// Multi-producer (submit/cancel/wait from any thread), single consumer (the scheduler).
#pragma once
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <deque>
#include <memory>
#include <mutex>
#include <thread>
#include <unordered_map>
#include <vector>
#include "chat.h"
#include "model.h"
#include "safetensors.h"

namespace acp {

struct Sequence {
  uint64_t ticket = 0;
  std::vector<ToolDef> tools;
  SamplingParams sampling;
  std::vector<int> force_tokens;
  int return_logits = 0;
  std::vector<int> tokens;   // prompt + generated
  int prompt_len = 0;
  int n_cached = 0;          // tokens whose K/V are in the cache
  std::vector<int> pages;
  std::vector<int> shared;   // prefix-cache entries behind pages[0 .. shared.size()): not ours to free
  std::atomic<bool> cancelled{false};
  bool done = false, reported = false;
  int status = 0;            // HTTP-like, valid when done
  std::string error_type, error_msg, finish_reason;
  std::vector<float> logits; // return_logits x vocab
  int logits_kept = 0;
  // tool_choice "required" / named function: the grammar's names and the state the emitted tokens reached
  std::shared_ptr<const GrammarNames> grammar_names;
  GrammarState gstate;
  int gslot = -1;            // name-table slot on the device while running
  bool gnames_sent = false;
  std::chrono::steady_clock::time_point t_submit, t_admit, t_first, t_done;
};

// KV retained after a sequence finishes and SHARED between sequences (SURVEY.md §8f rank 1): the
// context window of a Task is append-only, so its next LLM step starts with the same tokens; and
// every Task of an Agent starts with the same system prompt + tool schemas.  The cache is a chain
// of whole PROMPT pages keyed by (parent page, the page's 32 tokens): a new sequence walks the
// chain from its first token and maps every page it finds into its own page table — read-only,
// reference-counted, any number of sequences at once.  Only prompt-path K/V is cached (prefill
// arithmetic, batch invariant), so a hit is bit-identical to recomputing.
struct CachedPage {
  int page = -1;        // physical KV page (owned by the cache)
  int parent = -1;      // entry index of the previous page of the chain, -1 for position 0
  int children = 0;     // cached pages whose parent is this one
  int active = 0;       // running sequences that map this page
  uint64_t key = 0;
  uint64_t last_use = 0;
  int tokens[32];       // KV_PAGE tokens (exact match on lookup: the hash only routes)
};

struct EngineStats {
  long long prefix_hits = 0, prefix_tokens_reused = 0, prefix_deferrals = 0;
  long long decode_steps = 0, decode_tokens = 0, decode_ctx_tokens = 0;
  long long prefill_steps = 0, prefill_tokens = 0;
  double decode_ms = 0, prefill_ms = 0;
  double prefill_flops = 0, decode_flops = 0;   // algorithmic FLOPs (SURVEY.md §8d): GEMMs + causal attention + LM head
  long long requests_done = 0, requests_failed = 0;
  std::vector<float> decode_step_ms;
};

// Every id's bytes (Tokenizer::decode({id})) and stop flag, for the grammar on the host and, once, on the device.
struct GrammarVocabTable {
  std::vector<int32_t> off;
  std::vector<uint8_t> bytes, stop;
  GrammarVocab view;
};

class Engine {
 public:
  Engine() = default;
  ~Engine();
  int init(const char* config_json);
  int submit(const char* json, size_t len, uint64_t* ticket);
  int wait(uint64_t ticket, int timeout_ms);
  int poll(uint64_t* tickets, int max, int timeout_ms);
  int result(uint64_t ticket, std::string* body, int* status);
  int result_logits(uint64_t ticket, float* out, int max_positions);
  void cancel(uint64_t ticket);
  std::string stats_json();
  void stats_reset();
  void shutdown();

 private:
  void run();
  void admit_locked();
  bool step();  // returns false when there was nothing to do
  void finish(const std::shared_ptr<Sequence>& s, int status, const std::string& type,
              const std::string& msg, const std::string& finish_reason);
  void fail_all_running(const std::string& msg);
  void release_pages(Sequence& s);

  bool grammar_advance(GrammarState& st, const GrammarNames& names, int tok) const;
  int run_forward(const StepInput& in);
  void tp_worker(int idx);

  std::unique_ptr<Tokenizer> tok_owned_;         // "tokenizer": tokenizer.json (byte-level BPE)
  const Tokenizer* tok_ = &synthetic_tokenizer();
  std::unique_ptr<Checkpoint> ckpt_;             // "weights": <dir> — mmap'ed until the shards are loaded
  GrammarVocabTable gvocab_;                     // tp == 1 only
  std::vector<int> free_gslots_;
  std::vector<GrammarRow> grows_;                // step(): the constrained rows and the name tables to upload
  std::vector<int> gup_slot_;
  std::vector<const GrammarNames*> gup_names_;
  Model model_;                                  // shard 0 (the only one when tp == 1)
  std::vector<std::unique_ptr<Model>> extra_;    // tensor-parallel shards 1..tp-1, one GPU each
  std::vector<NcclComm> comms_;
  std::vector<std::thread> tp_threads_;
  std::mutex tp_mu_;
  std::condition_variable tp_cv_, tp_done_cv_;
  uint64_t tp_gen_ = 0;
  int tp_pending_ = 0, tp_rc_ = 0;
  const StepInput* tp_in_ = nullptr;
  bool tp_stop_ = false;
  int tp_ = 1;
  std::string model_name_;
  std::thread thread_;
  std::mutex mu_;
  std::condition_variable cv_work_, cv_done_;
  std::deque<std::shared_ptr<Sequence>> waiting_;
  std::vector<std::shared_ptr<Sequence>> running_;
  std::unordered_map<uint64_t, std::shared_ptr<Sequence>> all_;
  std::deque<uint64_t> finished_unreported_;
  std::vector<int> free_pages_;
  std::vector<CachedPage> pcache_;               // entries; holes are chained through free_entries_
  std::vector<int> free_entries_;
  std::unordered_multimap<uint64_t, int> pcache_index_;   // chain key -> entry
  int pcache_pages_ = 0;
  uint64_t use_clock_ = 0;
  bool prefix_cache_on_ = true;
  double request_timeout_ms_ = 0;   // "request_timeout_ms": 0 = none
  int pcache_find_locked(int parent, const int* tokens) const;
  int pcache_insert_locked(int parent, const int* tokens, int page);
  void publish_prefix_locked(Sequence& s);
  bool evict_locked(int want);
  void retain_prefix_locked(Sequence& s);
  std::atomic<bool> stop_{false};
  bool broken_ = false;
  uint64_t next_ticket_ = 1;
  EngineStats stats_;
  cudaEvent_t ev0_ = nullptr, ev1_ = nullptr;
  int max_ctx_tokens_ = 0;
  int decode_interleave_ = 0, prefill_steps_since_decode_ = 0;   // scheduling policy, see Engine::init
  int default_max_tokens_ = 1024;  // completion budget of a request that sets no max_tokens ("default_max_tokens")
};

}  // namespace acp
