// c_api.cc — extern "C" surface declared in include/acp_infer.h.  Nothing throws across it.
#include "acp_infer.h"
#include <atomic>
#include <chrono>
#include <memory>
#include <new>
#include <stdlib.h>
#include <string.h>
#include "engine.h"

// One handle = one engine, or — config "replicas": n — n data-parallel engines on consecutive GPUs
// behind the same handle (SURVEY.md §8e: Llama-3-8B shards at REQUEST level, no collective).  The
// ACP manager is ONE process: with 8 GPUs it wants 8 replicas behind one LLMClient.  Requests are
// routed STICKILY so that a Task's turns land on the replica that retains its K/V: by the OpenAI
// `user` field when the caller sets one, else by a hash of the first two messages (system prompt +
// first user message: a Task's context window is append-only, so every turn of a Task carries the
// same two — SendRequest has no Task identity to pass, llm_client.go:11-14); requests with neither
// go round-robin.  Global ticket = local ticket * 16 + replica.  With one replica the handle is a
// plain pass-through.
struct acp_engine {
  std::vector<std::unique_ptr<acp::Engine>> replicas;
  std::atomic<uint64_t> round_robin{0};
  acp::Engine& only() { return *replicas[0]; }
  bool multi() const { return replicas.size() > 1; }
};
constexpr int kReplicaBits = 4;   // up to 16 replicas per handle

static uint64_t fnv1a(const std::string& s) {
  uint64_t h = 1469598103934665603ull;
  for (unsigned char c : s) { h ^= c; h *= 1099511628211ull; }
  return h;
}

static char* dup_string(const std::string& s, size_t* len) {
  char* p = (char*)malloc(s.size() + 1);
  if (!p) return nullptr;
  memcpy(p, s.data(), s.size());
  p[s.size()] = 0;
  if (len) *len = s.size();
  return p;
}

extern "C" {

const char* acp_infer_version(void) { return "acp_infer 0.1.0 sm_90a"; }

int acp_infer_init(const char* config_json, acp_engine** out) {
  if (!out) return ACP_ERR_INVALID;
  *out = nullptr;
  acp_engine* e = nullptr;
  try {
    e = new (std::nothrow) acp_engine();
    if (!e) return ACP_ERR_NOMEM;
    acp::Json cfg;
    std::string perr;
    const std::string text = config_json && *config_json ? config_json : "{}";
    int n = 1;
    if (acp::Json::parse(text, &cfg, &perr) && cfg.is_object()) n = (int)cfg.get("replicas").as_int(1);
    if (n < 1 || n > (1 << kReplicaBits)) { delete e; return ACP_ERR_INVALID; }
    if (n == 1) {
      e->replicas.emplace_back(new acp::Engine());
      int rc = e->only().init(config_json);
      if (rc != 0) { delete e; return rc; }
    } else {
      // replica i runs on devices [device + i*tp, device + (i+1)*tp)
      const int dev0 = (int)cfg.get("device").as_int(0), tp = (int)cfg.get("tp").as_int(1);
      for (int i = 0; i < n; ++i) {
        acp::Json c = cfg;
        c.set("device", acp::Json(dev0 + i * (tp < 1 ? 1 : tp)));
        c.set("replicas", acp::Json(1));
        e->replicas.emplace_back(new acp::Engine());
        int rc = e->replicas.back()->init(c.dump().c_str());
        if (rc != 0) { delete e; return rc; }
      }
    }
    *out = e;
    return ACP_OK;
  } catch (const std::bad_alloc&) {
    try { delete e; } catch (...) {}
    return ACP_ERR_NOMEM;
  } catch (...) {
    try { delete e; } catch (...) {}
    return ACP_ERR_INVALID;
  }
}

int acp_infer_submit(acp_engine* e, const char* chat_request_json, size_t len, uint64_t* ticket) {
  if (!e || !chat_request_json || !ticket) return ACP_ERR_INVALID;
  try {
    if (!e->multi()) return e->only().submit(chat_request_json, len, ticket);
    // sticky routing key: the OpenAI `user` field (malformed bodies still get a ticket: replica 0 reports the 400)
    size_t r = 0;
    acp::Json req;
    std::string perr;
    if (acp::Json::parse(chat_request_json, len, &req, &perr) && req.is_object()) {
      std::string key = req.get("user").as_string();
      if (key.empty()) {
        const acp::Json& msgs = req.get("messages");
        for (size_t i = 0; i < msgs.size() && i < 2; ++i) {
          const acp::Json& c = msgs.items()[i].get("content");
          key += c.is_string() ? c.as_string() : c.dump();
          key.push_back('\x1f');
        }
        if (msgs.size() == 0) key.clear();
      }
      r = key.empty() ? (size_t)(e->round_robin.fetch_add(1) % e->replicas.size()) : (size_t)(fnv1a(key) % e->replicas.size());
    }
    uint64_t local = 0;
    const int rc = e->replicas[r]->submit(chat_request_json, len, &local);
    *ticket = (local << kReplicaBits) | (uint64_t)r;
    return rc;
  } catch (...) { return ACP_ERR_NOMEM; }
}

int acp_infer_wait(acp_engine* e, uint64_t ticket, int timeout_ms) {
  if (!e) return ACP_ERR_INVALID;
  try {
    if (!e->multi()) return e->only().wait(ticket, timeout_ms);
    const size_t r = (size_t)(ticket & ((1u << kReplicaBits) - 1));
    if (r >= e->replicas.size()) return ACP_ERR_NOT_FOUND;
    return e->replicas[r]->wait(ticket >> kReplicaBits, timeout_ms);
  } catch (...) { return ACP_ERR_INVALID; }
}

int acp_infer_poll(acp_engine* e, uint64_t* tickets, int max, int timeout_ms) {
  if (!e) return ACP_ERR_INVALID;
  try {
    if (!e->multi()) return e->only().poll(tickets, max, timeout_ms);
    // sweep the replicas without blocking; when nothing is ready, block in short slices on each in turn
    const auto deadline = std::chrono::steady_clock::now() + std::chrono::milliseconds(timeout_ms < 0 ? 0 : timeout_ms);
    size_t turn = 0;
    while (true) {
      int n = 0;
      for (size_t r = 0; r < e->replicas.size() && n < max; ++r) {
        const int got = e->replicas[r]->poll(tickets + n, max - n, 0);
        for (int i = 0; i < got; ++i) tickets[n + i] = (tickets[n + i] << kReplicaBits) | (uint64_t)r;
        if (got > 0) n += got;
      }
      if (n > 0 || timeout_ms == 0) return n;
      if (timeout_ms > 0 && std::chrono::steady_clock::now() >= deadline) return 0;
      const size_t r = turn++ % e->replicas.size();
      const int got = e->replicas[r]->poll(tickets, max, 1);     // 1 ms slice
      if (got > 0) {
        for (int i = 0; i < got; ++i) tickets[i] = (tickets[i] << kReplicaBits) | (uint64_t)r;
        return got;
      }
    }
  } catch (...) { return ACP_ERR_INVALID; }
}

int acp_infer_result(acp_engine* e, uint64_t ticket, char** chat_response_json, size_t* len,
                     int* http_like_status) {
  if (!e || !chat_response_json || !http_like_status) return ACP_ERR_INVALID;
  try {
    std::string body;
    int rc;
    if (!e->multi()) rc = e->only().result(ticket, &body, http_like_status);
    else {
      const size_t r = (size_t)(ticket & ((1u << kReplicaBits) - 1));
      if (r >= e->replicas.size()) return ACP_ERR_NOT_FOUND;
      rc = e->replicas[r]->result(ticket >> kReplicaBits, &body, http_like_status);
    }
    if (rc != 0) return rc;
    *chat_response_json = dup_string(body, len);
    return *chat_response_json ? ACP_OK : ACP_ERR_NOMEM;
  } catch (...) {
    return ACP_ERR_NOMEM;
  }
}

int acp_infer_result_logits(acp_engine* e, uint64_t ticket, float* out, int max_positions) {
  if (!e) return ACP_ERR_INVALID;
  try {
    if (!e->multi()) return e->only().result_logits(ticket, out, max_positions);
    const size_t r = (size_t)(ticket & ((1u << kReplicaBits) - 1));
    if (r >= e->replicas.size()) return ACP_ERR_NOT_FOUND;
    return e->replicas[r]->result_logits(ticket >> kReplicaBits, out, max_positions);
  } catch (...) { return ACP_ERR_INVALID; }
}

void acp_infer_cancel(acp_engine* e, uint64_t ticket) {
  if (!e) return;
  try {
    if (!e->multi()) { e->only().cancel(ticket); return; }
    const size_t r = (size_t)(ticket & ((1u << kReplicaBits) - 1));
    if (r < e->replicas.size()) e->replicas[r]->cancel(ticket >> kReplicaBits);
  } catch (...) {}
}

int acp_infer_stats(acp_engine* e, char** json) {
  if (!e || !json) return ACP_ERR_INVALID;
  try {
    if (!e->multi()) {
      *json = dup_string(e->only().stats_json(), nullptr);
      return *json ? ACP_OK : ACP_ERR_NOMEM;
    }
    // per-replica objects + the additive counters summed at the top level
    acp::Json out = acp::Json::object(), arr = acp::Json::array();
    static const char* kSum[] = {"decode_steps", "decode_tokens", "prefill_steps", "prefill_tokens", "requests_done", "requests_failed",
                                 "prefix_hits", "prefix_tokens_reused", "prefix_deferrals", "prefix_cache_pages", "kv_pages_free",
                                 "kv_pages_total", "kernel_launches", "h2d_bytes", "d2h_bytes", "running", "waiting"};
    std::vector<long long> sums(sizeof kSum / sizeof *kSum, 0);
    for (auto& r : e->replicas) {
      acp::Json j;
      std::string perr;
      if (!acp::Json::parse(r->stats_json(), &j, &perr)) continue;
      for (size_t k = 0; k < sums.size(); ++k) sums[k] += j.get(kSum[k]).as_int(0);
      arr.push(j);
    }
    out.set("replica_count", acp::Json((int)e->replicas.size()));
    for (size_t k = 0; k < sums.size(); ++k) out.set(kSum[k], acp::Json(sums[k]));
    out.set("replicas", arr);
    *json = dup_string(out.dump(), nullptr);
    return *json ? ACP_OK : ACP_ERR_NOMEM;
  } catch (...) {
    return ACP_ERR_NOMEM;
  }
}

void acp_infer_stats_reset(acp_engine* e) {
  if (e) for (auto& r : e->replicas) r->stats_reset();
}

void acp_infer_free(void* p) { free(p); }

void acp_infer_shutdown(acp_engine* e) {
  if (!e) return;
  try { for (auto& r : e->replicas) r->shutdown(); } catch (...) {}
  delete e;
}

}  // extern "C"
