// engine.cc — see engine.h.
#include "engine.h"
#include <algorithm>
#include <stdio.h>

namespace acp {

using clk = std::chrono::steady_clock;
static double ms_between(clk::time_point a, clk::time_point b) {
  return std::chrono::duration<double, std::milli>(b - a).count();
}

Engine::~Engine() { shutdown(); }

int Engine::init(const char* config_json) {
  Json cfg;
  std::string err;
  const std::string text = config_json && *config_json ? config_json : "{}";
  if (!Json::parse(text, &cfg, &err) || !cfg.is_object()) {
    fprintf(stderr, "[acp_infer] bad config JSON: %s\n", err.c_str());
    return -1;
  }
  ModelConfig mc;
  std::string name = cfg.get("model").as_string();
  const std::string weights = cfg.get("weights").as_string();
  if (!weights.empty() && weights != "synthetic") {
    // a HuggingFace Llama checkpoint directory (config.json + safetensors); "model" is then only
    // the name requests must carry (LLM.spec.parameters.model), default = the directory name
    std::string err;
    ckpt_.reset(new Checkpoint());
    if (!ckpt_->open(weights, &err)) { fprintf(stderr, "[acp_infer] weights: %s\n", err.c_str()); return -1; }
    if (!ckpt_->has_config()) { fprintf(stderr, "[acp_infer] weights: no config.json in %s\n", ckpt_->dir().c_str()); return -1; }
    if (!model_config_from_hf(ckpt_->config(), &mc, &err)) { fprintf(stderr, "[acp_infer] weights: %s\n", err.c_str()); return -1; }
    if (name.empty()) {
      const std::string& d = ckpt_->dir();
      const size_t e = d.find_last_not_of('/');
      const size_t b = d.find_last_of('/', e);
      name = d.substr(b == std::string::npos ? 0 : b + 1, e == std::string::npos ? std::string::npos : e - (b == std::string::npos ? 0 : b + 1) + 1);
      if (name.empty()) name = "checkpoint";
    }
    mc.name = name;
  } else {
    if (name.empty()) name = "tiny";
    if (!model_preset(name, &mc)) {
      fprintf(stderr, "[acp_infer] unknown model preset '%s'\n", name.c_str());
      return -1;
    }
  }
  {  // vocabulary: explicit "tokenizer", else the checkpoint's tokenizer.json, else the synthetic one
    std::string tpath = cfg.get("tokenizer").as_string();
    if (tpath.empty() && ckpt_) {
      const std::string cand = ckpt_->dir() + "/tokenizer.json";
      if (FILE* f = fopen(cand.c_str(), "rb")) { fclose(f); tpath = cand; }
    }
    if (!tpath.empty() && tpath != "synthetic") {
      std::string err;
      tok_owned_ = load_tokenizer_json(tpath, &err);
      if (!tok_owned_) { fprintf(stderr, "[acp_infer] tokenizer: %s\n", err.c_str()); return -1; }
      tok_ = tok_owned_.get();
      if (tok_->vocab_size() > mc.vocab) {
        fprintf(stderr, "[acp_infer] tokenizer has %d ids but the model's vocabulary is %d\n", tok_->vocab_size(), mc.vocab);
        return -1;
      }
    } else if (mc.vocab < synthetic_tokenizer().vocab_size()) {
      fprintf(stderr, "[acp_infer] the synthetic tokenizer needs a model vocabulary of %d (got %d): pass \"tokenizer\"\n",
              synthetic_tokenizer().vocab_size(), mc.vocab);
      return -1;
    }
  }
  if (cfg.find("seed")) mc.seed = (uint64_t)cfg.get("seed").as_int((long long)mc.seed);
  if (cfg.find("layers")) mc.layers = (int)cfg.get("layers").as_int(mc.layers);  // truncated-depth runs
  // std of the seeded synthetic matrices (oracle/synth.py); the default 0.02 makes every layer's
  // update ~85x the embedding's scale, a chaotic regime in which bf16 rounding noise grows layer by
  // layer — tests/test_fulldepth_gpu.py also runs a damped setting where it does not
  if (cfg.find("w_std") && !ckpt_) mc.w_std = cfg.get("w_std").as_double(mc.w_std);
  if (!(mc.w_std > 0.0 && mc.w_std < 1.0)) { fprintf(stderr, "[acp_infer] w_std out of range\n"); return -1; }
  if (mc.layers < 1 || mc.layers > 1024 || mc.hidden < 128 || mc.ffn < 64 || mc.vocab < 128 || mc.heads < 1 || mc.kv_heads < 1) {
    fprintf(stderr, "[acp_infer] invalid model dimensions (layers=%d hidden=%d ffn=%d vocab=%d heads=%d kv_heads=%d)\n",
            mc.layers, mc.hidden, mc.ffn, mc.vocab, mc.heads, mc.kv_heads);
    return -1;
  }
  ModelLimits lim;
  lim.max_batch = (int)cfg.get("max_batch").as_int(lim.max_batch);
  lim.max_tokens = (int)cfg.get("max_tokens_per_step").as_int(lim.max_tokens);
  lim.num_pages = (int)cfg.get("kv_pages").as_int(lim.num_pages);
  lim.max_pages_per_seq = (int)cfg.get("max_pages_per_seq").as_int(lim.max_pages_per_seq);
  {
    const std::string am = cfg.get("attn_decode_mode").as_string();
    lim.attn_decode_mode = am == "item" ? 1 : (am == "chunked" || am == "flat") ? 2 : 0;
  }
  lim.strict_batch_invariance = cfg.get("strict_batch_invariance").as_bool(false);
  if (cfg.find("prefix_cache")) prefix_cache_on_ = cfg.get("prefix_cache").as_bool(true);
  request_timeout_ms_ = (double)cfg.get("request_timeout_ms").as_int(0);
  if (cfg.find("splitk_target_ctas")) lim.splitk_target_ctas = (int)cfg.get("splitk_target_ctas").as_int(lim.splitk_target_ctas);
  if (lim.max_batch < 1 || lim.max_tokens < 16 || lim.num_pages < 2 || lim.max_pages_per_seq < 1 ||
      lim.max_batch > (1 << 16) || lim.max_tokens > (1 << 20) || lim.max_pages_per_seq > (1 << 16)) {
    fprintf(stderr, "[acp_infer] invalid engine limits\n");
    return -1;
  }
  // a decode step has one token row per running sequence: the row budget of a step can never be
  // smaller than the batch (prefill chunking is result-invariant, so raising it changes no output)
  if (lim.max_tokens < lim.max_batch) {
    fprintf(stderr, "[acp_infer] max_tokens_per_step %d < max_batch %d: raised to %d\n", lim.max_tokens, lim.max_batch, lim.max_batch);
    lim.max_tokens = lim.max_batch;
  }
  // Scheduling policy when prompts are pending AND sequences are decoding (VERDICT r1 weak item 15):
  //   0 (default)  prefill first — best throughput for a burst of Tasks (bench.py): decoding sequences wait
  //                until every pending prompt token is cached;
  //   k > 0        latency bound — after every k prefill steps (each <= max_tokens_per_step rows) ONE decode
  //                step runs for the sequences that are already generating, so a decoding Task never waits
  //                longer than k prefill chunks for its next token.
  // Prompt tokens still take the prefill arithmetic and generated tokens the decode arithmetic (a mixed
  // step would put decode rows through the non-split GEMM path and change their fp32 summation order),
  // so results are bit-identical under either policy.
  decode_interleave_ = (int)cfg.get("decode_interleave").as_int(0);
  if (decode_interleave_ < 0) decode_interleave_ = 0;
  default_max_tokens_ = (int)cfg.get("default_max_tokens").as_int(default_max_tokens_);
  if (default_max_tokens_ < 1) default_max_tokens_ = 1;
  const int device = (int)cfg.get("device").as_int(0);
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) {
    fprintf(stderr, "[acp_infer] no CUDA device available: provider local cannot start (no CPU fallback)\n");
    return -5;
  }
  if (device < 0 || device >= ndev) {
    fprintf(stderr, "[acp_infer] device %d out of range (%d visible)\n", device, ndev);
    return -1;
  }
  model_name_ = name;
  tp_ = (int)cfg.get("tp").as_int(1);
  if (mc.fp8 && tp_ != 1) {
    fprintf(stderr, "[acp_infer] tp=%d: FP8 models run on one GPU (tp must be 1)\n", tp_);
    return -1;
  }
  if (tp_ < 1 || device + tp_ > ndev) {
    fprintf(stderr, "[acp_infer] tp=%d needs devices %d..%d but %d are visible\n", tp_, device, device + tp_ - 1, ndev);
    return -1;
  }
  int rc = 0;
  if (tp_ == 1) {
    // the vocabulary as bytes for tool_choice grammars (constrained requests are served on one GPU)
    gvocab_.off.assign((size_t)mc.vocab + 1, 0);
    gvocab_.stop.assign((size_t)mc.vocab, 0);
    std::vector<int> one(1);
    for (int id = 0; id < mc.vocab; ++id) {
      if (id < tok_->vocab_size()) {
        one[0] = id;
        const std::string b = tok_->decode(one);
        gvocab_.bytes.insert(gvocab_.bytes.end(), b.begin(), b.end());
        gvocab_.stop[(size_t)id] = tok_->is_stop(id) ? 1 : 0;
      }
      gvocab_.off[(size_t)id + 1] = (int32_t)gvocab_.bytes.size();
    }
    gvocab_.view.vocab = mc.vocab;
    gvocab_.view.off = gvocab_.off.data();
    gvocab_.view.bytes = gvocab_.bytes.data();
    gvocab_.view.stop = gvocab_.stop.data();
    lim.grammar_vocab = &gvocab_.view;
    for (int i = lim.max_batch - 1; i >= 0; --i) free_gslots_.push_back(i);
    rc = model_.init(mc, lim, device, 0, 1, nullptr, nullptr, ckpt_.get());
    if (rc != 0) return rc;
  } else {
    // tensor parallel inside ONE process: a communicator and a host thread per GPU
    const NcclApi& nc = nccl_api();
    if (!nc.ok) { fprintf(stderr, "[acp_infer] tp > 1 needs libnccl.so.2\n"); return -5; }
    std::vector<int> devs;
    for (int i = 0; i < tp_; ++i) devs.push_back(device + i);
    comms_.resize(tp_);
    int nrc = nc.CommInitAll(comms_.data(), tp_, devs.data());
    if (nrc != 0) { fprintf(stderr, "[acp_infer] ncclCommInitAll: %s\n", nc.GetErrorString(nrc)); return -5; }
    // shards initialise concurrently (weight generation is per GPU)
    std::vector<int> rcs(tp_, 0);
    std::vector<std::thread> inits;
    for (int i = 1; i < tp_; ++i) extra_.emplace_back(new Model());
    for (int i = 0; i < tp_; ++i)
      inits.emplace_back([&, i] {
        Model* m = i == 0 ? &model_ : extra_[i - 1].get();
        // an exception escaping a std::thread is std::terminate: report it as an init failure instead
        try { rcs[i] = m->init(mc, lim, devs[i], i, tp_, comms_[i], i == 0 ? nullptr : &model_, ckpt_.get()); }
        catch (...) { rcs[i] = -4; }
      });
    for (auto& t : inits) t.join();
    for (int r : rcs) if (r != 0) return r;
    // peer-memory exchange (default): every shard may load/store every other shard's buffers
    const std::string comm = cfg.get("tp_comm").as_string();
    if (comm != "nccl") {
      bool ok = (tp_ == 2 || tp_ == 4 || tp_ == 8);  // the exchange kernel is instantiated for these
      for (int i = 0; i < tp_ && ok; ++i) {
        cudaSetDevice(devs[i]);
        for (int j = 0; j < tp_; ++j) {
          if (i == j) continue;
          int can = 0;
          cudaDeviceCanAccessPeer(&can, devs[i], devs[j]);
          if (!can) { ok = false; break; }
          cudaError_t e = cudaDeviceEnablePeerAccess(devs[j], 0);
          if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) { ok = false; break; }
          cudaGetLastError();
        }
      }
      if (ok) {
        TpPeers peers;
        peers.size = tp_;
        for (int p = 0; p < TP_MAX; ++p) {
          Model* m = p == 0 ? &model_ : (p < tp_ ? extra_[p - 1].get() : &model_);
          peers.ar[p] = m->ar_buffer(); peers.x[p] = m->x_buffer(); peers.xn[p] = m->xn_buffer();
          peers.flags[p] = m->tp_flags();
        }
        for (int i = 0; i < tp_; ++i) {
          peers.rank = i;
          (i == 0 ? &model_ : extra_[i - 1].get())->set_peers(peers);
        }
      } else {
        fprintf(stderr, "[acp_infer] peer access unavailable: tensor-parallel exchange falls back to NCCL all-reduce\n");
      }
      cudaSetDevice(device);
    }
    if (const char* xb = getenv("ACP_TP_EXCHANGE_BENCH")) {  // dev: time the bare exchange (no GEMM)
      const int iters = std::max(1, atoi(xb));
      // diag bits (wrong results, timing only): 1 = volatile instead of .nc loads, 2 = no remote pushes,
      // 4 = no remote pulls
      for (int diag : {0, 1, 2, 4, 6})
        for (int T : {64, 256, 2048}) {
          if (T > lim.max_tokens) continue;
          std::vector<float> us(tp_, 0.f);
          std::vector<std::thread> th;
          for (int i = 0; i < tp_; ++i)
            th.emplace_back([&, i] { (i == 0 ? &model_ : extra_[i - 1].get())->bench_exchange(T, iters, &us[i], diag); });
          for (auto& t : th) t.join();
          fprintf(stderr, "[acp_infer] tp=%d bare exchange diag=%d T=%d: %.2f us\n", tp_, diag, T, us[0]);
        }
    }
    for (int i = 1; i < tp_; ++i) tp_threads_.emplace_back([this, i] { tp_worker(i - 1); });
  }
  cudaSetDevice(device);
  if (cudaEventCreate(&ev0_) != cudaSuccess || cudaEventCreate(&ev1_) != cudaSuccess) return -5;
  max_ctx_tokens_ = std::min(lim.max_pages_per_seq * KV_PAGE, mc.max_pos);
  for (int p = lim.num_pages - 1; p >= 1; --p) free_pages_.push_back(p);  // page 0 reserved
  ckpt_.reset();  // weights are in HBM: drop the file mappings
  thread_ = std::thread([this] { run(); });
  return 0;
}

void Engine::shutdown() {
  {
    std::lock_guard<std::mutex> lk(mu_);
    stop_ = true;  // idempotent: a second shutdown() finds nothing left to join or free
  }
  cv_work_.notify_all();
  if (thread_.joinable()) thread_.join();
  {
    std::lock_guard<std::mutex> lk(tp_mu_);
    tp_stop_ = true;
  }
  tp_cv_.notify_all();
  for (auto& t : tp_threads_) if (t.joinable()) t.join();
  tp_threads_.clear();
  extra_.clear();
  if (!comms_.empty()) {
    const NcclApi& nc = nccl_api();
    for (NcclComm c : comms_) if (c) nc.CommDestroy(c);
    comms_.clear();
  }
  std::lock_guard<std::mutex> lk(mu_);
  for (auto& kv : all_) {
    if (!kv.second->done) {
      kv.second->done = true;
      kv.second->status = 503;
      kv.second->error_type = "engine_shutdown";
      kv.second->error_msg = "engine is shutting down";
      finished_unreported_.push_back(kv.first);   // a poller (integration/go/inference) must see them
    }
  }
  running_.clear();
  waiting_.clear();
  cv_done_.notify_all();
  if (ev0_) { cudaEventDestroy(ev0_); ev0_ = nullptr; }
  if (ev1_) { cudaEventDestroy(ev1_); ev1_ = nullptr; }
}

int Engine::submit(const char* json, size_t len, uint64_t* ticket) {
  if (!json || !ticket) return -1;
  auto s = std::make_shared<Sequence>();
  s->t_submit = clk::now();
  ChatRequest req;
  std::string err;
  int status = parse_chat_request(json, len, &req, &err);
  std::string etype = "invalid_request_error";
  if (status == 0) {
    if (!req.model.empty() && req.model != model_name_) {
      status = 404; etype = "model_not_found";
      err = "model '" + req.model + "' is not served by this engine (serving '" + model_name_ + "')";
    }
  }
  if (status == 0) {
    if (req.has_prompt_ids) s->tokens = req.prompt_token_ids;
    else render_prompt(req, &s->tokens, *tok_);
    const int vocab = model_.config().vocab;
    for (int t : s->tokens)
      if (t < 0 || t >= vocab) { status = 400; err = "prompt token id out of range"; break; }
    for (int t : req.force_tokens)
      if (t < 0 || t >= vocab) { status = 400; err = "force token id out of range"; break; }
    if (status == 0 && s->tokens.empty()) { status = 400; err = "empty prompt"; }
  }
  if (status == 0) {
    s->prompt_len = (int)s->tokens.size();
    s->sampling = req.sampling;
    if (s->sampling.max_tokens <= 0) {
      // The reference sends no max_tokens unless LLM.spec.parameters.maxTokens is set
      // (langchaingo_client.go:83-115) and the provider then generates until it stops by itself.
      // Here: everything the context still holds, capped by "default_max_tokens" because KV pages for
      // prompt + max_tokens are reserved at admission.
      const long long left = (long long)max_ctx_tokens_ - s->prompt_len;
      s->sampling.max_tokens = (int)std::max(1LL, std::min<long long>(left, default_max_tokens_));
    }
    if (status == 0 && req.grammar_names) {
      if (tp_ > 1) {
        status = 400;
        err = "tool_choice other than \"auto\" is served on single-GPU engines (tp = 1; use replicas), this one has tp = " +
              std::to_string(tp_);
      } else {
        s->grammar_names = req.grammar_names;
        grammar_init(&s->gstate, s->grammar_names->n, req.parallel_tool_calls);
        GrammarState st = s->gstate;
        for (size_t i = 0; i < req.force_tokens.size() && status == 0; ++i) {
          if (!grammar_advance(st, *s->grammar_names, req.force_tokens[i])) {
            status = 400;
            err = "acp.force_tokens[" + std::to_string(i) + "] is not allowed by the tool_choice grammar";
          }
          if (tok_->is_stop(req.force_tokens[i])) break;
        }
      }
    }
    s->tools = std::move(req.tools);
    s->force_tokens = std::move(req.force_tokens);
    s->return_logits = std::max(0, std::min(req.return_logits, 64));
    const long long need = (long long)s->prompt_len + s->sampling.max_tokens;
    if (need > max_ctx_tokens_) {
      status = 400; etype = "context_length_exceeded";
      err = "prompt (" + std::to_string(s->prompt_len) + " tokens) + max_tokens (" +
            std::to_string(s->sampling.max_tokens) + ") exceeds the engine context limit of " +
            std::to_string(max_ctx_tokens_) + " tokens";
    }
    const long long pages_needed = (need + KV_PAGE - 1) / KV_PAGE;
    if (status == 0 && pages_needed > model_.limits().num_pages - 1) {
      status = 400; etype = "context_length_exceeded";
      err = "request needs more KV pages than the pool holds";
    }
  }
  std::lock_guard<std::mutex> lk(mu_);
  if (stop_) return -6;
  s->ticket = next_ticket_++;
  *ticket = s->ticket;
  all_[s->ticket] = s;
  if (status != 0) {
    s->done = true; s->status = status; s->error_type = etype; s->error_msg = err;
    s->t_done = clk::now();
    finished_unreported_.push_back(s->ticket);
    ++stats_.requests_failed;
    cv_done_.notify_all();
    return 0;
  }
  if (broken_) {
    s->done = true; s->status = 500; s->error_type = "engine_error";
    s->error_msg = "engine stopped after a CUDA failure";
    finished_unreported_.push_back(s->ticket);
    cv_done_.notify_all();
    return 0;
  }
  waiting_.push_back(s);
  cv_work_.notify_one();
  return 0;
}

int Engine::wait(uint64_t ticket, int timeout_ms) {
  std::unique_lock<std::mutex> lk(mu_);
  auto it = all_.find(ticket);
  if (it == all_.end()) return -2;
  auto s = it->second;
  auto pred = [&] { return s->done; };
  if (timeout_ms < 0) cv_done_.wait(lk, pred);
  else if (!cv_done_.wait_for(lk, std::chrono::milliseconds(timeout_ms), pred)) return -3;
  return 0;
}

int Engine::poll(uint64_t* tickets, int max, int timeout_ms) {
  if (!tickets || max <= 0) return -1;
  std::unique_lock<std::mutex> lk(mu_);
  auto pred = [&] { return !finished_unreported_.empty() || stop_.load(); };
  if (timeout_ms < 0) cv_done_.wait(lk, pred);
  else if (timeout_ms > 0) cv_done_.wait_for(lk, std::chrono::milliseconds(timeout_ms), pred);
  int n = 0;
  while (n < max && !finished_unreported_.empty()) {
    tickets[n++] = finished_unreported_.front();
    finished_unreported_.pop_front();
  }
  return n;
}

int Engine::result_logits(uint64_t ticket, float* out, int max_positions) {
  std::lock_guard<std::mutex> lk(mu_);
  auto it = all_.find(ticket);
  if (it == all_.end()) return -2;
  if (!it->second->done) return -7;
  const int vocab = model_.config().vocab;
  const int n = std::min(max_positions, it->second->logits_kept);
  if (n > 0 && out) memcpy(out, it->second->logits.data(), (size_t)n * vocab * sizeof(float));
  return n;
}

int Engine::result(uint64_t ticket, std::string* body, int* status) {
  std::shared_ptr<Sequence> s;
  {
    std::lock_guard<std::mutex> lk(mu_);
    auto it = all_.find(ticket);
    if (it == all_.end()) return -2;
    if (!it->second->done) return -7;
    s = it->second;
    all_.erase(it);
    for (auto f = finished_unreported_.begin(); f != finished_unreported_.end(); ++f)
      if (*f == ticket) { finished_unreported_.erase(f); break; }
  }
  *status = s->status;
  if (s->status != 200) {
    *body = build_error_response(s->status, s->error_type, s->error_msg);
    return 0;
  }
  // detokenise + tool-call extraction happen here, on the caller's thread, not on the scheduler
  std::vector<int> gen(s->tokens.begin() + s->prompt_len, s->tokens.end());
  std::vector<int> text_ids = gen;
  if (s->finish_reason == "stop" && !text_ids.empty()) text_ids.pop_back();  // drop the stop token
  const std::string text = tok_->decode(text_ids);
  ParsedCompletion pc = parse_completion(text, s->tools, "call_" + std::to_string(ticket) + "_");
  if (s->finish_reason == "length" && !s->tools.empty() && pc.tool_calls.empty()) {
    size_t p = 0;
    while (p < text.size() && (text[p] == ' ' || text[p] == '\n' || text[p] == '\t' || text[p] == '\r')) ++p;
    if (p < text.size() && text[p] == '{') {
      // A tool call cut by the completion budget would otherwise be recorded by the Task controller
      // as a successful FinalAnswer holding half a JSON object (processLLMResponse,
      // state_machine.go:608): surface a terminal 4xx instead (retrying gives the same cut).
      *status = 422;
      *body = build_error_response(422, "truncated_tool_call",
                                   "completion reached max_tokens (" + std::to_string(s->sampling.max_tokens) +
                                       ") inside a tool call; raise LLM.spec.parameters.maxTokens");
      return 0;
    }
  }
  if (pc.tool_calls.empty() && pc.content.empty()) {
    // The Task controller loops forever on an empty assistant message
    // (state_machine.go:608/641 + checkToolCalls with zero ToolCalls): surface a terminal 4xx.
    *status = 422;
    *body = build_error_response(422, "empty_completion", "model produced an empty completion");
    return 0;
  }
  *body = build_chat_response(ticket, model_name_, pc, s->finish_reason, s->prompt_len, gen,
                              ms_between(s->t_submit, s->t_admit), ms_between(s->t_admit, s->t_first),
                              ms_between(s->t_first, s->t_done));
  return 0;
}

void Engine::cancel(uint64_t ticket) {
  std::lock_guard<std::mutex> lk(mu_);
  auto it = all_.find(ticket);
  if (it == all_.end() || it->second->done) return;
  it->second->cancelled = true;
  cv_work_.notify_one();
}

// caller holds mu_.  Pages mapped from the prefix cache go back to it (one user fewer), the
// sequence's own pages to the free list.
void Engine::release_pages(Sequence& s) {
  for (size_t i = 0; i < s.pages.size(); ++i) {
    if (i < s.shared.size()) --pcache_[(size_t)s.shared[i]].active;
    else free_pages_.push_back(s.pages[i]);
  }
  s.pages.clear();
  s.shared.clear();
}

static uint64_t chain_key(uint64_t parent_key, const int* tokens) {
  uint64_t h = parent_key * 0x9E3779B97F4A7C15ull + 0xD1B54A32D192ED03ull;
  for (int i = 0; i < KV_PAGE; ++i) {
    h ^= (uint64_t)(uint32_t)tokens[i] + 0x9E3779B97F4A7C15ull + (h << 6) + (h >> 2);
    h *= 0xFF51AFD7ED558CCDull;
    h ^= h >> 33;
  }
  return h;
}

// entry holding the page (parent, tokens[0..32)) or -1; caller holds mu_
int Engine::pcache_find_locked(int parent, const int* tokens) const {
  const uint64_t key = chain_key(parent < 0 ? 0 : pcache_[(size_t)parent].key, tokens);
  auto range = pcache_index_.equal_range(key);
  for (auto it = range.first; it != range.second; ++it) {
    const CachedPage& e = pcache_[(size_t)it->second];
    if (e.parent == parent && memcmp(e.tokens, tokens, sizeof e.tokens) == 0) return it->second;
  }
  return -1;
}

// caller holds mu_.  Frees cached pages that nobody maps and nothing chains from (leaves first, so
// a chain shrinks from its tail), least recently used first, until `want` pages are free or
// nothing is evictable.
bool Engine::evict_locked(int want) {
  bool any = false;
  while ((int)free_pages_.size() < want) {
    std::vector<std::pair<uint64_t, int>> cand;
    for (size_t i = 0; i < pcache_.size(); ++i) {
      const CachedPage& e = pcache_[i];
      if (e.page >= 0 && e.active == 0 && e.children == 0) cand.emplace_back(e.last_use, (int)i);
    }
    if (cand.empty()) break;
    std::sort(cand.begin(), cand.end());
    for (const auto& c : cand) {
      if ((int)free_pages_.size() >= want) break;
      CachedPage& e = pcache_[(size_t)c.second];
      auto range = pcache_index_.equal_range(e.key);
      for (auto it = range.first; it != range.second; ++it)
        if (it->second == c.second) { pcache_index_.erase(it); break; }
      if (e.parent >= 0) --pcache_[(size_t)e.parent].children;
      free_pages_.push_back(e.page);
      e.page = -1;
      free_entries_.push_back(c.second);
      --pcache_pages_;
      any = true;
    }
  }
  return any;
}

// caller holds mu_.  New cache entry for `page` holding `toks` behind `parent` (-1: position 0).
int Engine::pcache_insert_locked(int parent, const int* toks, int page) {
  int idx;
  if (!free_entries_.empty()) { idx = free_entries_.back(); free_entries_.pop_back(); }
  else { idx = (int)pcache_.size(); pcache_.emplace_back(); }
  CachedPage& e = pcache_[(size_t)idx];
  e.page = page;
  e.parent = parent;
  e.children = 0;
  e.active = 0;
  e.key = chain_key(parent < 0 ? 0 : pcache_[(size_t)parent].key, toks);
  e.last_use = use_clock_;
  memcpy(e.tokens, toks, sizeof e.tokens);
  if (parent >= 0) ++pcache_[(size_t)parent].children;
  pcache_index_.emplace(e.key, idx);
  ++pcache_pages_;
  return idx;
}

// caller holds mu_.  Publishes the whole PROMPT pages of a running sequence whose K/V the last
// prefill step completed: from now on any admitted request maps them (the owner keeps using them
// through its page table like any other shared page).  If an identical page was published by a
// twin in the meantime, the sequence switches to the cached page and frees its own — both hold the
// same bits (prompt K/V is batch invariant).
void Engine::publish_prefix_locked(Sequence& s) {
  if (!prefix_cache_on_) return;
  const int whole = std::min(s.prompt_len, s.n_cached) / KV_PAGE;
  if ((int)s.shared.size() >= whole) return;
  ++use_clock_;
  for (int i = (int)s.shared.size(); i < whole && i < (int)s.pages.size(); ++i) {
    const int parent = i == 0 ? -1 : s.shared[(size_t)i - 1];
    const int* toks = s.tokens.data() + (size_t)i * KV_PAGE;
    int e = pcache_find_locked(parent, toks);
    if (e >= 0) {
      free_pages_.push_back(s.pages[(size_t)i]);
      s.pages[(size_t)i] = pcache_[(size_t)e].page;
    } else {
      e = pcache_insert_locked(parent, toks, s.pages[(size_t)i]);
    }
    ++pcache_[(size_t)e].active;
    pcache_[(size_t)e].last_use = use_clock_;
    s.shared.push_back(e);
  }
}

// caller holds mu_.  Donates the whole pages that hold the PROMPT's K/V to the prefix cache (pages
// whose content is already cached are simply freed); everything else goes back to the free list.
void Engine::retain_prefix_locked(Sequence& s) {
  const int keep_tokens = std::min(s.prompt_len, s.n_cached);
  const int keep_pages = keep_tokens / KV_PAGE;  // whole pages only
  if (!prefix_cache_on_ || keep_pages < 1 || (int)s.pages.size() < keep_pages) { release_pages(s); return; }
  ++use_clock_;
  int parent = -1;
  for (int i = 0; i < (int)s.pages.size(); ++i) {
    if (i < (int)s.shared.size()) {          // mapped from the cache: hand it back, keep walking the chain
      parent = s.shared[(size_t)i];
      --pcache_[(size_t)parent].active;
      pcache_[(size_t)parent].last_use = use_clock_;
      continue;
    }
    if (i >= keep_pages) { free_pages_.push_back(s.pages[(size_t)i]); continue; }
    const int* toks = s.tokens.data() + (size_t)i * KV_PAGE;
    const int have = pcache_find_locked(parent, toks);
    if (have >= 0) {                          // same content cached meanwhile by another sequence
      free_pages_.push_back(s.pages[(size_t)i]);
      pcache_[(size_t)have].last_use = use_clock_;
      parent = have;
      continue;
    }
    const int idx = pcache_insert_locked(parent, toks, s.pages[(size_t)i]);
    parent = idx;
  }
  s.pages.clear();
  s.shared.clear();
}

// Advances a constrained sequence's grammar state by token `tok`; false = the grammar rejects it.
bool Engine::grammar_advance(GrammarState& st, const GrammarNames& names, int tok) const {
  if (tok < 0 || tok >= gvocab_.view.vocab) return false;
  if (gvocab_.stop[(size_t)tok]) return grammar_accepting(st);
  const int b = gvocab_.off[(size_t)tok], e = gvocab_.off[(size_t)tok + 1];
  if (b == e) return false;
  for (int i = b; i < e; ++i)
    if (!grammar_step(st, gvocab_.bytes[(size_t)i], names)) return false;
  return true;
}

void Engine::finish(const std::shared_ptr<Sequence>& s, int status, const std::string& type,
                    const std::string& msg, const std::string& finish_reason) {
  if (status == 200) retain_prefix_locked(*s); else release_pages(*s);
  if (s->gslot >= 0) { free_gslots_.push_back(s->gslot); s->gslot = -1; }
  s->done = true;
  s->status = status;
  s->error_type = type;
  s->error_msg = msg;
  s->finish_reason = finish_reason;
  s->t_done = clk::now();
  if (status == 200) ++stats_.requests_done; else ++stats_.requests_failed;
  finished_unreported_.push_back(s->ticket);
  cv_done_.notify_all();
}

void Engine::fail_all_running(const std::string& msg) {
  std::lock_guard<std::mutex> lk(mu_);
  broken_ = true;
  for (auto& s : running_) finish(s, 500, "engine_error", msg, "");
  running_.clear();
  while (!waiting_.empty()) { finish(waiting_.front(), 500, "engine_error", msg, ""); waiting_.pop_front(); }
  cv_done_.notify_all();
}

// caller holds mu_
void Engine::admit_locked() {
  const int max_batch = model_.limits().max_batch;
  // drop cancelled requests that never started
  const auto now = clk::now();
  for (auto it = waiting_.begin(); it != waiting_.end();) {
    if ((*it)->cancelled) { finish(*it, 499, "cancelled", "request cancelled", ""); it = waiting_.erase(it); }
    else if (request_timeout_ms_ > 0 && ms_between((*it)->t_submit, now) > request_timeout_ms_) {
      // the reference declares LLMRequestTimeout (task_controller.go:25) and never applies it; here a request
      // that outlives the configured budget ends as a TRANSIENT 504: plain error upstream => requeue in 5 s
      finish(*it, 504, "timeout", "request exceeded request_timeout_ms in the queue", "");
      it = waiting_.erase(it);
    } else ++it;
  }
  while (!waiting_.empty() && (int)running_.size() < max_batch) {
    auto& s = waiting_.front();
    const int need = (s->prompt_len + s->sampling.max_tokens + KV_PAGE - 1) / KV_PAGE;
    // longest cached chain of whole prompt pages (at least one prompt token is always recomputed
    // so that there are logits to sample from); the pages are MAPPED, not moved: any number of
    // running sequences read the same physical pages
    std::vector<int> chain;
    if (prefix_cache_on_) {
      const int max_pages = (s->prompt_len - 1) / KV_PAGE;
      int parent = -1;
      for (int i = 0; i < max_pages; ++i) {
        const int e = pcache_find_locked(parent, s->tokens.data() + (size_t)i * KV_PAGE);
        if (e < 0) break;
        chain.push_back(e);
        parent = e;
      }
    }
    // in-flight dedup: if a RUNNING sequence is about to publish the very next page of this prompt
    // (same tokens up to and including it, not yet published), wait for it instead of prefilling a
    // copy — a burst of Tasks of one Agent then computes the shared system prompt + tool schemas
    // once.  FIFO is kept (everything behind waits too); the owner publishes after its next prefill
    // step, or leaves running_ (finished / cancelled), so the condition clears by itself.
    if (prefix_cache_on_) {
      const int c = (int)chain.size();
      const int next_end = (c + 1) * KV_PAGE;
      bool in_flight = false;
      if (next_end <= s->prompt_len - 1)
        for (const auto& r : running_) {
          if (r->prompt_len < next_end || (int)r->shared.size() > c || r->n_cached >= r->prompt_len) continue;
          if (memcmp(r->tokens.data(), s->tokens.data(), (size_t)next_end * sizeof(int)) == 0) { in_flight = true; break; }
        }
      if (in_flight) { ++stats_.prefix_deferrals; break; }
    }
    const int fresh = need - (int)chain.size();
    // pin the chain while evicting to make room (an entry with users is never evicted)
    for (int e : chain) ++pcache_[(size_t)e].active;
    if (fresh > (int)free_pages_.size()) evict_locked(fresh);
    if (fresh > (int)free_pages_.size()) {    // FIFO: wait for pages to come back
      for (int e : chain) --pcache_[(size_t)e].active;
      break;
    }
    if (!chain.empty()) {
      ++use_clock_;
      for (int e : chain) {
        s->pages.push_back(pcache_[(size_t)e].page);
        pcache_[(size_t)e].last_use = use_clock_;
      }
      s->shared = chain;
      s->n_cached = (int)chain.size() * KV_PAGE;
      ++stats_.prefix_hits;
      stats_.prefix_tokens_reused += s->n_cached;
    }
    for (int i = 0; i < fresh; ++i) { s->pages.push_back(free_pages_.back()); free_pages_.pop_back(); }
    if (s->grammar_names) { s->gslot = free_gslots_.back(); free_gslots_.pop_back(); }   // running_ < max_batch slots
    s->t_admit = clk::now();
    running_.push_back(s);
    waiting_.pop_front();
  }
}

void Engine::run() {
  cudaSetDevice(model_.device());
  while (true) {
    {
      std::unique_lock<std::mutex> lk(mu_);
      if (stop_) break;
      admit_locked();
      // cancelled while running
      bool any_cancel = false;
      const auto now = clk::now();
      for (auto it = running_.begin(); it != running_.end();) {
        if ((*it)->cancelled) { finish(*it, 499, "cancelled", "request cancelled", ""); it = running_.erase(it); any_cancel = true; }
        else if (request_timeout_ms_ > 0 && ms_between((*it)->t_submit, now) > request_timeout_ms_) {
          finish(*it, 504, "timeout", "request exceeded request_timeout_ms", "");
          it = running_.erase(it);
          any_cancel = true;
        } else ++it;
      }
      if (any_cancel) { cv_done_.notify_all(); admit_locked(); }
      if (running_.empty()) {
        cv_done_.notify_all();
        cv_work_.wait(lk, [&] { return stop_.load() || !waiting_.empty(); });
        continue;
      }
    }
    if (!step()) std::this_thread::yield();
  }
}

bool Engine::step() {
  const ModelLimits& lim = model_.limits();
  const int vocab = model_.config().vocab;
  // running_ is only mutated by this thread
  std::vector<Sequence*> part;   // sequences in this step
  std::vector<int> take;
  bool prefill = false;
  // A sequence is in prefill while prompt tokens remain un-cached (even a single one): prompt
  // tokens always take the prefill arithmetic path, generated tokens always the decode path, so a
  // sequence's result never depends on batch composition or chunk boundaries.
  bool any_decoding = false;
  for (auto& s : running_) {
    if (s->n_cached < s->prompt_len) prefill = true;
    else any_decoding = true;
  }
  if (prefill && any_decoding && decode_interleave_ > 0 && prefill_steps_since_decode_ >= decode_interleave_)
    prefill = false;   // latency bound: the decoding sequences get a step now, the pending prompts right after
  prefill_steps_since_decode_ = prefill ? prefill_steps_since_decode_ + 1 : 0;
  int T = 0, n_blocks = 0;
  const int blk_tokens = attn_prefill_block_tokens(model_.config().heads, model_.config().kv_heads);
  if (prefill) {
    int budget = lim.max_tokens;
    for (auto& s : running_) {
      const int pending = s->prompt_len - s->n_cached;
      if (pending <= 0) continue;
      if (budget == 0 || (int)part.size() == lim.max_batch) break;
      const int t = std::min(pending, budget);
      part.push_back(s.get());
      take.push_back(t);
      budget -= t;
      T += t;
      n_blocks += (t + blk_tokens - 1) / blk_tokens;
    }
  } else {
    for (auto& s : running_) {
      if (s->n_cached < s->prompt_len) continue;   // still prefilling (only possible under decode_interleave)
      part.push_back(s.get());
      take.push_back(1);
    }
    T = (int)part.size();
  }
  if (part.empty()) return false;
  const int B = (int)part.size();
  StepInput& in = model_.stage_begin(T, B, n_blocks);
  in.decode = !prefill;
  int row = 0, nb = 0, ns = 0, max_ctx = 0;
  bool all_greedy = true, want_logits = false;
  std::vector<int> sample_seq;  // index into part for each sampled row
  grows_.clear(); gup_slot_.clear(); gup_names_.clear();
  for (int b = 0; b < B; ++b) {
    Sequence& s = *part[b];
    const int q = take[b];
    in.q_start[b] = row;
    in.q_len[b] = q;
    in.ctx_len[b] = s.n_cached + q;
    max_ctx = std::max(max_ctx, s.n_cached + q);
    for (int i = 0; i < q; ++i) {
      in.tok[row + i] = s.tokens[s.n_cached + i];
      in.pos[row + i] = s.n_cached + i;
      in.seq_of_row[row + i] = b;
    }
    if (prefill)
      for (int t0 = 0; t0 < q; t0 += blk_tokens) { in.blk_seq[nb] = b; in.blk_tok0[nb] = t0; ++nb; }
    // the pages that hold this step's context (Model::forward uploads these); the rest of the row is never read
    int* pt = in.page_table + (size_t)b * lim.max_pages_per_seq;
    const int used = std::min((s.n_cached + q + KV_PAGE - 1) / KV_PAGE, lim.max_pages_per_seq);
    const int np = std::min((int)s.pages.size(), used);
    for (int i = 0; i < np; ++i) pt[i] = s.pages[i];
    for (int i = np; i < used; ++i) pt[i] = 0;
    if (s.n_cached + q == (int)s.tokens.size()) {  // reaches the end of known tokens: sample
      in.sample_rows[ns] = row + q - 1;
      const int gen_idx = (int)s.tokens.size() - s.prompt_len;
      SampleParams& sp = in.sample_params[ns];
      sp.temperature = s.sampling.temperature;
      sp.top_k = s.sampling.top_k;
      sp.top_p = s.sampling.top_p;
      // OpenAI `seed`: same seed + same request => same sample; without one, a per-ticket stream
      sp.seed = s.sampling.seed ? s.sampling.seed : (s.ticket * 0x9E3779B97F4A7C15ull);
      sp.step = (uint32_t)gen_idx;
      if (s.sampling.temperature > 0.f) all_greedy = false;
      if (gen_idx < s.return_logits) want_logits = true;
      if (s.grammar_names) {
        GrammarRow gr;
        gr.row = ns; gr.slot = s.gslot; gr.state = s.gstate;
        grows_.push_back(gr);
        if (!s.gnames_sent) { gup_slot_.push_back(s.gslot); gup_names_.push_back(s.grammar_names.get()); s.gnames_sent = true; }
      }
      sample_seq.push_back(b);
      ++ns;
    }
    row += q;
  }
  in.tile_cum[0] = 0;
  for (int b = 0; b < B; ++b) in.tile_cum[b + 1] = in.tile_cum[b] + attn_decode_chunks(in.ctx_len[b]);
  in.n_sample = ns;
  in.all_greedy = all_greedy;
  in.want_logits = want_logits;
  in.max_ctx = max_ctx;
  in.n_constrained = (int)grows_.size();
  in.g_rows = grows_.data();
  in.n_name_uploads = (int)gup_slot_.size();
  in.g_upload_slot = gup_slot_.data();
  in.g_upload_names = gup_names_.data();

  int rc = run_forward(in);
  if (rc != 0) { fail_all_running("CUDA step failed (see stderr)"); return true; }
  float step_ms = 0.f;
  cudaEventElapsedTime(&step_ms, ev0_, ev1_);

  const int* toks = model_.host_tokens();
  const auto now = clk::now();
  std::lock_guard<std::mutex> lk(mu_);
  double qk_pairs = 0;   // (query token, visible key) pairs of this step
  for (int b = 0; b < B; ++b) {
    const double c0 = part[b]->n_cached, q = take[b];
    qk_pairs += q * c0 + q * (q + 1) / 2;
  }
  const double flops = model_.config().step_flops(T, ns, qk_pairs);
  if (prefill) { ++stats_.prefill_steps; stats_.prefill_tokens += T; stats_.prefill_ms += step_ms; stats_.prefill_flops += flops; }
  else {
    ++stats_.decode_steps; stats_.decode_tokens += B; stats_.decode_ms += step_ms; stats_.decode_flops += flops;
    for (int b = 0; b < B; ++b) stats_.decode_ctx_tokens += part[b]->n_cached;  // keys read (excl. own)
    if (stats_.decode_step_ms.size() < 65536) stats_.decode_step_ms.push_back(step_ms);
  }
  for (int b = 0; b < B; ++b) part[b]->n_cached += take[b];
  if (prefill)
    for (int b = 0; b < B; ++b) publish_prefix_locked(*part[b]);
  bool any_done = false;
  for (int i = 0; i < ns; ++i) {
    Sequence& s = *part[sample_seq[i]];
    int tok = toks[i];
    const int gen_idx = (int)s.tokens.size() - s.prompt_len;
    if (gen_idx < s.return_logits) {
      if (s.logits.empty()) s.logits.resize((size_t)s.return_logits * vocab);
      memcpy(s.logits.data() + (size_t)gen_idx * vocab, model_.host_logits() + (size_t)i * vocab,
             (size_t)vocab * sizeof(float));
      s.logits_kept = gen_idx + 1;
    }
    if (gen_idx < (int)s.force_tokens.size()) tok = s.force_tokens[gen_idx];
    if (gen_idx == 0) s.t_first = now;
    if (s.grammar_names && !grammar_advance(s.gstate, *s.grammar_names, tok)) {
      // the mask allows only tokens the grammar accepts: reaching this is an engine defect, never an answer
      for (auto it = running_.begin(); it != running_.end(); ++it)
        if (it->get() == &s) {
          auto sp = *it;
          running_.erase(it);
          finish(sp, 500, "grammar_violation", "token " + std::to_string(tok) + " violates the tool_choice grammar", "");
          break;
        }
      any_done = true;
      continue;
    }
    s.tokens.push_back(tok);
    const bool stop_tok = tok_->is_stop(tok);
    const bool at_cap = (gen_idx + 1 >= s.sampling.max_tokens);
    if (stop_tok || at_cap) {
      for (auto it = running_.begin(); it != running_.end(); ++it)
        if (it->get() == &s) {
          auto sp = *it;
          running_.erase(it);
          finish(sp, 200, "", "", stop_tok ? "stop" : "length");
          break;
        }
      any_done = true;
    }
  }
  if (any_done) cv_done_.notify_all();
  return true;
}

void Engine::tp_worker(int idx) {
  Model& m = *extra_[idx];
  cudaSetDevice(m.device());
  uint64_t seen = 0;
  while (true) {
    const StepInput* in = nullptr;
    {
      std::unique_lock<std::mutex> lk(tp_mu_);
      tp_cv_.wait(lk, [&] { return tp_stop_ || tp_gen_ != seen; });
      if (tp_stop_) return;
      seen = tp_gen_;
      in = tp_in_;
    }
    int rc = m.forward(*in);
    if (rc == 0) rc = m.sync();
    {
      std::lock_guard<std::mutex> lk(tp_mu_);
      if (rc != 0) tp_rc_ = rc;
      --tp_pending_;
    }
    tp_done_cv_.notify_all();
  }
}

// One engine step on every shard.  Device time is measured on shard 0's stream.
int Engine::run_forward(const StepInput& in) {
  if (tp_ > 1) {
    std::lock_guard<std::mutex> lk(tp_mu_);
    tp_in_ = &in;
    tp_pending_ = (int)extra_.size();
    tp_rc_ = 0;
    ++tp_gen_;
  }
  if (tp_ > 1) tp_cv_.notify_all();
  cudaEventRecord(ev0_, model_.stream());
  int rc = model_.forward(in);
  cudaEventRecord(ev1_, model_.stream());
  if (rc == 0) rc = model_.sync();
  if (tp_ > 1) {
    std::unique_lock<std::mutex> lk(tp_mu_);
    tp_done_cv_.wait(lk, [&] { return tp_pending_ == 0; });
    if (rc == 0) rc = tp_rc_;
  }
  return rc;
}

std::string Engine::stats_json() {
  std::lock_guard<std::mutex> lk(mu_);
  const ModelConfig& c = model_.config();
  Json j = Json::object();
  j.set("model", Json(model_name_));
  j.set("tokenizer", Json(tok_->kind()));
  j.set("layers", Json(c.layers));
  j.set("decode_steps", Json(stats_.decode_steps));
  j.set("decode_tokens", Json(stats_.decode_tokens));
  j.set("decode_ctx_tokens", Json(stats_.decode_ctx_tokens));
  j.set("decode_ms", Json(stats_.decode_ms));
  j.set("prefill_steps", Json(stats_.prefill_steps));
  j.set("prefill_tokens", Json(stats_.prefill_tokens));
  j.set("prefill_ms", Json(stats_.prefill_ms));
  j.set("prefill_flops_algorithmic", Json(stats_.prefill_flops));
  j.set("decode_flops_algorithmic", Json(stats_.decode_flops));
  j.set("requests_done", Json(stats_.requests_done));
  j.set("requests_failed", Json(stats_.requests_failed));
  j.set("kernel_launches", Json(model_.launches()));
  j.set("h2d_bytes", Json(model_.h2d_bytes()));
  j.set("d2h_bytes", Json(model_.d2h_bytes()));
  j.set("tp", Json(tp_));
  j.set("weight_bytes_per_step", Json(c.weight_bytes()));
  j.set("weight_dtype", Json(c.fp8 ? "fp8_e4m3" : "bf16"));
  j.set("kv_bytes_per_token", Json(c.kv_bytes_per_token()));
  // SURVEY.md §8(d): bytes_step = W + sum_seq ctx*K + B*K, summed over the decode steps so far
  // (whole model; with tp > 1 each GPU streams 1/tp of it)
  const double bytes = (double)stats_.decode_steps * c.weight_bytes() +
                       c.kv_bytes_per_token() * ((double)stats_.decode_ctx_tokens + (double)stats_.decode_tokens);
  j.set("decode_bytes_algorithmic", Json(bytes));
  j.set("decode_bytes_algorithmic_per_gpu", Json(bytes / tp_));
  std::vector<float> v = stats_.decode_step_ms;
  if (!v.empty()) {
    std::sort(v.begin(), v.end());
    j.set("decode_step_ms_p50", Json((double)v[v.size() / 2]));
    j.set("decode_step_ms_p99", Json((double)v[std::min(v.size() - 1, (size_t)(v.size() * 0.99))]));
    j.set("decode_step_ms_min", Json((double)v.front()));
    j.set("decode_step_ms_max", Json((double)v.back()));
  }
  j.set("prefix_hits", Json(stats_.prefix_hits));
  j.set("prefix_tokens_reused", Json(stats_.prefix_tokens_reused));
  j.set("prefix_cache_pages", Json(pcache_pages_));
  j.set("prefix_deferrals", Json(stats_.prefix_deferrals));
  j.set("kv_pages_free", Json((int)free_pages_.size()));
  j.set("kv_pages_total", Json(model_.limits().num_pages - 1));
  {
    Json prof;
    std::string perr;
    if (Json::parse(model_.profile_json(), &prof, &perr)) j.set("profile", prof);
  }
  j.set("running", Json((int)running_.size()));
  j.set("waiting", Json((int)waiting_.size()));
  return j.dump();
}

void Engine::stats_reset() {
  std::lock_guard<std::mutex> lk(mu_);
  stats_ = EngineStats();
}

}  // namespace acp
