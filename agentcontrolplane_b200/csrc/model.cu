// model.cu — weights in HBM, activation buffers, and the forward pass of one engine step.
//
// Per step (T token rows, B sequences):
//   embed -> [ rmsnorm -> QKV GEMM -> RoPE + KV scatter -> paged attention -> O GEMM ->
//              add+rmsnorm -> gate/up GEMM -> SwiGLU -> down GEMM -> add+rmsnorm ] x L
//   -> final norm on the sampled rows only -> LM-head GEMM with fused arg-max -> token ids.
// Decode steps (T <= 256) run the GEMMs split-K with fp32 partial planes reduced in fixed order by
// the consumer kernels; prefill steps write bf16 directly.  bf16 rounding points are exactly the
// ones listed in oracle/llama_oracle.py.
#include "model.h"
#include "safetensors.h"
#include "common.cuh"
#include "gemm_wgmma.cuh"
#include <math.h>
#include <stdlib.h>
#include <string.h>

namespace acp {

static bool debug_sync_enabled() {
  static int v = -1;
  if (v < 0) { const char* e = getenv("ACP_DEBUG_SYNC"); v = (e && *e && *e != '0') ? 1 : 0; }
  return v == 1;
}
// ACP_DEBUG_SYNC=1: synchronise after every launch and name the kernel that failed.
#define ACP_TRY(expr)                                                                      \
  do {                                                                                     \
    int _rc = (expr);                                                                      \
    if (_rc != 0) {   /* never fail silently: name the call (one line per frame up the stack) */ \
      fprintf(stderr, "[acp_infer] `%s` failed with %d (%s:%d)\n", #expr, _rc, __FILE__, __LINE__); \
      return _rc;                                                                          \
    }                                                                                      \
    if (debug_sync_enabled() && stream_) {                                                 \
      cudaError_t _e = cudaStreamSynchronize(stream_);                                     \
      if (_e != cudaSuccess) {                                                             \
        fprintf(stderr, "[acp_infer] ACP_DEBUG_SYNC: failure after `%s` (%s:%d): %s\n",    \
                #expr, __FILE__, __LINE__, cudaGetErrorString(_e));                        \
        return -5;                                                                         \
      }                                                                                    \
    }                                                                                      \
  } while (0)

static bool profile_enabled() {
  static int v = -1;
  if (v < 0) { const char* e = getenv("ACP_PROFILE"); v = (e && *e && *e != '0') ? 1 : 0; }
  return v == 1;
}
bool Model::prof_begin(const char* name) {
  if (!profile_enabled()) return false;
  while (prof_pool_.size() < prof_used_ + 2) {
    cudaEvent_t e;
    cudaEventCreate(&e);
    prof_pool_.push_back(e);
  }
  ProfSeg seg{name, prof_pool_[prof_used_], prof_pool_[prof_used_ + 1]};
  prof_used_ += 2;
  cudaEventRecord(seg.a, stream_);
  prof_segs_.push_back(seg);
  return true;
}
void Model::prof_end() { cudaEventRecord(prof_segs_.back().b, stream_); }
void Model::prof_collect(bool decode) {
  auto& acc = prof_acc_[decode ? 1 : 0];
  for (auto& seg : prof_segs_) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, seg.a, seg.b) != cudaSuccess) continue;
    bool found = false;
    for (auto& kv : acc)
      if (kv.first == seg.name) { kv.second.n++; kv.second.ms += ms; found = true; break; }
    if (!found) { ProfAcc a; a.n = 1; a.ms = ms; acc.emplace_back(seg.name, a); }
  }
  prof_segs_.clear();
  prof_used_ = 0;
}
std::string Model::profile_json() {
  std::string out = "{";
  for (int d = 0; d < 2; ++d) {
    out += d ? ",\"decode\":{" : "\"prefill\":{";
    bool first = true;
    for (auto& kv : prof_acc_[d]) {
      char buf[256];
      snprintf(buf, sizeof buf, "%s\"%s\":{\"n\":%lld,\"ms\":%.4f}", first ? "" : ",", kv.first.c_str(), kv.second.n, kv.second.ms);
      out += buf;
      first = false;
    }
    out += "}";
  }
  return out + "}";
}
#define PROF(name, expr)                         \
  do {                                           \
    const bool _p = prof_begin(name);            \
    ACP_TRY(expr);                               \
    if (_p) prof_end();                          \
  } while (0)

Model::~Model() {
  cudaSetDevice(device_);
  if (stream_) cudaStreamSynchronize(stream_);
  for (void* p : allocs_) cudaFree(p);
  if (h_ints_) cudaFreeHost(h_ints_);
  if (h_sparams_) cudaFreeHost(h_sparams_);
  if (h_tokens_) cudaFreeHost(h_tokens_);
  if (h_logits_) cudaFreeHost(h_logits_);
  if (stream_) cudaStreamDestroy(stream_);
}

static int dmalloc(std::vector<void*>& allocs, void** p, size_t bytes, bool zero = false) {
  cudaError_t e = cudaMalloc(p, bytes ? bytes : 16);
  if (e != cudaSuccess) {
    fprintf(stderr, "[acp_infer] cudaMalloc(%zu MiB) failed: %s\n", bytes >> 20, cudaGetErrorString(e));
    return -4;
  }
  allocs.push_back(*p);
  if (zero) {
    e = cudaMemset(*p, 0, bytes ? bytes : 16);
    if (e != cudaSuccess) return -5;
  }
  return 0;
}
template <class T>
static int dmalloc_t(std::vector<void*>& allocs, T** p, size_t count, bool zero = false) {
  return dmalloc(allocs, (void**)p, count * sizeof(T), zero);
}

// Split-K factor of a DECODE-step GEMM.
//   N <= 256 rows (one N tile): depends only on (M, K), never on the batch size, so a sequence's
//   arithmetic does not change with what it happens to be batched with (prefill steps never split:
//   see gemm()) — the batch-invariance the tests check.
//   N > 256 rows (e.g. B = 512): the GEMMs are tensor-bound and 5-7 fp32 planes of
//   512 rows cost more than the MMAs (r1: QKV 0.5, O 0.4 PFLOP/s); there the split only has to give
//   every SM the same share: S minimises ceil(tiles * S / SMs) / S.  Still a fixed function of
//   (M, K, number of N tiles) — deterministic run to run — but a sequence decoded inside a batch of
//   more than 256 sums its K range in different pieces than inside a smaller batch
//   ("strict_batch_invariance": true keeps the one-tile splits everywhere).
int Model::choose_splits(int M, int K, int N) const {
  return splitk_factor(M, K, N, lim_.splitk_target_ctas, lim_.strict_batch_invariance);   // model_config.cc
}

int Model::init(const ModelConfig& cfg, const ModelLimits& lim, int device, int tp_rank, int tp_size,
                NcclComm comm, Model* lead, const Checkpoint* ckpt) {
  cfg_ = cfg;
  lim_ = lim;
  device_ = device;
  tp_rank_ = tp_rank; tp_size_ = tp_size; comm_ = comm; lead_ = lead;
  if (cfg.hidden % 128 || cfg.ffn % 64 || cfg.vocab % 128 || cfg.heads % cfg.kv_heads) {
    fprintf(stderr, "[acp_infer] unsupported model dims\n");
    return -1;
  }
  if (cfg.heads % tp_size || cfg.kv_heads % tp_size || cfg.ffn % (64 * tp_size)) {
    fprintf(stderr, "[acp_infer] tp=%d does not divide heads=%d / kv_heads=%d / ffn=%d\n", tp_size,
            cfg.heads, cfg.kv_heads, cfg.ffn);
    return -1;
  }
  heads_l_ = cfg.heads / tp_size; kvh_l_ = cfg.kv_heads / tp_size;
  qdim_l_ = heads_l_ * HEAD_DIM; kvdim_l_ = kvh_l_ * HEAD_DIM; qkv_l_ = qdim_l_ + 2 * kvdim_l_;
  ffn_l_ = cfg.ffn / tp_size;
  if (cfg.experts > 0) {
    // expert parallel: the experts are spread over the tensor-parallel ranks (whole experts, full ffn width each);
    // attention stays head-parallel.  Tokens are replicated across the ranks (every rank holds xn after the
    // fused exchange), so "dispatch" is a local gather and "combine" is the row-parallel all-reduce.
    if (cfg.experts % tp_size) { fprintf(stderr, "[acp_infer] tp=%d does not divide experts=%d\n", tp_size, cfg.experts); return -1; }
    if (cfg.experts > 16 || lim.max_tokens > 32767) {
      fprintf(stderr, "[acp_infer] mixture of experts: at most 16 experts and max_tokens_per_step <= 32767 (got %d, %d)\n", cfg.experts, lim.max_tokens);
      return -1;
    }
    experts_l_ = cfg.experts / tp_size;
    expert0_ = tp_rank * experts_l_;
    ffn_l_ = cfg.ffn;
  }
  {  // vocab-parallel LM head: whole 128-row tiles per rank
    const int tiles = cfg.vocab / GEMM_BM, per = (tiles + tp_size - 1) / tp_size;
    const int t0 = per * tp_rank < tiles ? per * tp_rank : tiles;
    const int t1 = per * (tp_rank + 1) < tiles ? per * (tp_rank + 1) : tiles;
    lm_row0_ = t0 * GEMM_BM;
    lm_rows_l_ = (t1 - t0) * GEMM_BM;
    lm_rows_per_rank_ = per * GEMM_BM;
    if (lm_rows_l_ <= 0) { fprintf(stderr, "[acp_infer] tp too large for the vocabulary\n"); return -1; }
  }
  const char* env = getenv("ACP_SPLITK_TARGET");
  if (env) lim_.splitk_target_ctas = atoi(env);
  env = getenv("ACP_FUSE_SWIGLU");
  fuse_swiglu_ = env && *env == '1';
  // Prefill: SwiGLU runs in the persistent gate/up GEMM's epilogue (paired-lane exchange; the producer
  // streams the next tile meanwhile).  ACP_FUSE_SWIGLU_PREFILL=0 restores the separate kernel.
  env = getenv("ACP_TP_SYNC_EVERY");
  tp_sync_every_ = (env && tp_size > 1) ? atoi(env) : 0;
  env = getenv("ACP_FUSE_SWIGLU_PREFILL");
  fuse_swiglu_prefill_ = !(env && *env == '0');
  ACP_CUDA_CHECK(cudaSetDevice(device));
  ACP_CUDA_CHECK(cudaStreamCreateWithFlags(&stream_, cudaStreamNonBlocking));
  ACP_TRY(tma_init());
  ACP_TRY(gemm_setup_attributes());
  ACP_TRY(attn_setup_attributes());
  ACP_TRY(alloc_all());
  if (ckpt) ACP_TRY(load_weights(*ckpt));
  else ACP_TRY(gen_weights());
  ACP_TRY(build_rope_tables());
  ACP_CUDA_CHECK(cudaStreamSynchronize(stream_));
  return 0;
}

int Model::alloc_all() {
  const ModelConfig& c = cfg_;
  const size_t H = c.hidden;
  const int T = ((lim_.max_tokens + 255) / 256) * 256;
  const int Bp = ((lim_.max_batch + 255) / 256) * 256;
  layers_.resize(c.layers);
  const size_t kv_elems = (size_t)lim_.num_pages * kvh_l_ * KV_PAGE * HEAD_DIM;
  for (int l = 0; l < c.layers; ++l) {
    Layer& L = layers_[l];
    ACP_TRY(dmalloc_t(allocs_, &L.wqkv, (size_t)qkv_l_ * H));
    ACP_TRY(dmalloc_t(allocs_, &L.wo, H * qdim_l_));
    if (c.experts > 0) {
      ACP_TRY(dmalloc_t(allocs_, &L.router, (size_t)c.experts * H));
      ACP_TRY(dmalloc_t(allocs_, &L.wgu_e, (size_t)experts_l_ * 2 * c.ffn * H));
      ACP_TRY(dmalloc_t(allocs_, &L.wdown_e, (size_t)experts_l_ * H * c.ffn));
      ACP_TRY(tma_make_weight(&L.m_gu_e, L.wgu_e, (uint64_t)experts_l_ * 2 * c.ffn, H));
      ACP_TRY(tma_make_weight(&L.m_down_e, L.wdown_e, (uint64_t)experts_l_ * H, c.ffn));
      L.wgu = L.wdown = nullptr;
    } else {
      ACP_TRY(dmalloc_t(allocs_, &L.wgu, (size_t)2 * ffn_l_ * H));
      ACP_TRY(dmalloc_t(allocs_, &L.wdown, H * ffn_l_));
    }
    ACP_TRY(dmalloc_t(allocs_, &L.attn_norm, H));
    ACP_TRY(dmalloc_t(allocs_, &L.ffn_norm, H));
    ACP_TRY(dmalloc_t(allocs_, &L.k_cache, kv_elems, true));
    ACP_TRY(dmalloc_t(allocs_, &L.v_cache, kv_elems, true));
    ACP_TRY(tma_make_weight(&L.m_qkv, L.wqkv, qkv_l_, H));
    ACP_TRY(tma_make_weight(&L.m_o, L.wo, H, qdim_l_));
    if (c.experts == 0) {
      ACP_TRY(tma_make_weight(&L.m_gu, L.wgu, 2 * ffn_l_, H));
      ACP_TRY(tma_make_weight(&L.m_down, L.wdown, H, ffn_l_));
    }
    ACP_TRY(attn_make_kv_map(&L.tm_k, L.k_cache, lim_.num_pages, kvh_l_));
    ACP_TRY(attn_make_kv_map(&L.tm_v, L.v_cache, lim_.num_pages, kvh_l_));
    ACP_TRY(attn_make_kv_half_map(&L.tm_k32, L.k_cache, lim_.num_pages, kvh_l_));
    ACP_TRY(attn_make_kv_half_map(&L.tm_v32, L.v_cache, lim_.num_pages, kvh_l_));
  }
  ACP_TRY(dmalloc_t(allocs_, &embed_, (size_t)c.vocab * H));
  ACP_TRY(dmalloc_t(allocs_, &lm_head_, (size_t)lm_rows_l_ * H));
  ACP_TRY(dmalloc_t(allocs_, &final_norm_, H));
  ACP_TRY(tma_make_weight(&m_lm_, lm_head_, lm_rows_l_, H));
  ACP_TRY(dmalloc_t(allocs_, &cos_, (size_t)c.max_pos * 64));
  ACP_TRY(dmalloc_t(allocs_, &sin_, (size_t)c.max_pos * 64));
  // activations (rows padded to the largest N tile, zero initialised)
  ACP_TRY(dmalloc_t(allocs_, &x_, (size_t)T * H, true));
  ACP_TRY(dmalloc_t(allocs_, &xn_, (size_t)T * H, true));
  ACP_TRY(dmalloc_t(allocs_, &qbuf_, (size_t)T * qdim_l_, true));
  ACP_TRY(dmalloc_t(allocs_, &attn_, (size_t)T * qdim_l_, true));
  ACP_TRY(dmalloc_t(allocs_, &h_, (size_t)T * (c.experts > 0 ? 8 : ffn_l_), true));
  if (c.experts > 0) {
    const size_t rows = (size_t)2 * T + 256;   // 2 assignments per token, + one N tile of slack for the last group's TMA box
    ACP_TRY(dmalloc_t(allocs_, &xe_, rows * H, true));
    ACP_TRY(dmalloc_t(allocs_, &he_, rows * c.ffn, true));
    ACP_TRY(dmalloc_t(allocs_, &ye_, rows * H, true));
    ACP_TRY(tma_make_act(&m_xe_, xe_, rows, H));
    ACP_TRY(tma_make_act(&m_he_, he_, rows, c.ffn));
    ACP_TRY(dmalloc_t(allocs_, &moe_topk_idx_, (size_t)2 * T));
    ACP_TRY(dmalloc_t(allocs_, &moe_topk_w_, (size_t)2 * T));
    ACP_TRY(dmalloc_t(allocs_, &moe_row_of_, (size_t)2 * T));
    ACP_TRY(dmalloc_t(allocs_, &moe_ranges_, (size_t)moe_ranges_ints(T), true));
  }
  ACP_TRY(dmalloc_t(allocs_, &xs_, (size_t)Bp * H, true));
  int max_m = qkv_l_;
  if (2 * ffn_l_ > max_m) max_m = 2 * ffn_l_;
  if (c.hidden > max_m) max_m = c.hidden;
  ACP_TRY(dmalloc_t(allocs_, &gemm_bf16_, (size_t)T * max_m, true));
  ACP_TRY(attn_make_q_map(&tm_q_, qbuf_, (uint64_t)T, heads_l_, kvh_l_));
  ACP_TRY(tma_make_act(&m_xn_, xn_, T, H));
  ACP_TRY(tma_make_act(&m_attn_, attn_, T, qdim_l_));
  if (c.experts == 0) ACP_TRY(tma_make_act(&m_h_, h_, T, ffn_l_));
  ACP_TRY(tma_make_act(&m_xs_, xs_, Bp, H));
  // split-K workspace: worst case over the four GEMMs of a decode step with max_batch rows
  size_t ws = 0;
  const int shapes[4][2] = {{qkv_l_, c.hidden}, {c.hidden, qdim_l_}, {2 * ffn_l_, c.hidden}, {c.hidden, ffn_l_}};
  for (auto& s : shapes) {
    if (c.experts > 0 && (&s - shapes) >= 2) continue;   // the expert GEMMs are grouped, never split-K
    // the split factor depends on the row count beyond 256 rows: sized over every step height (model_config.cc)
    const size_t b = splitk_workspace_bytes(s[0], s[1], lim_.max_batch, lim_.splitk_target_ctas, lim_.strict_batch_invariance);
    if (b > ws) ws = b;
  }
  if (tp_size_ > 1) {  // row-parallel GEMMs write fp32 (one rounding after the all-reduce), prefill too
    const size_t b = (size_t)T * H * sizeof(float);
    if (b > ws) ws = b;
    ACP_TRY(dmalloc_t(allocs_, &ar_buf_, (size_t)T * H));
    ACP_TRY(dmalloc_t(allocs_, &cand_local_, (size_t)2 * Bp));
    ACP_TRY(dmalloc_t(allocs_, &cand_all_, (size_t)2 * Bp * tp_size_));
    ACP_TRY(dmalloc_t(allocs_, &amax_val_row_, (size_t)Bp));
    ACP_TRY(dmalloc_t(allocs_, &tp_flags_, (size_t)TP_MAX + 8, true));  // [0..7] flags, [8] done counter
  }
  ws_bytes_ = ws;
  ACP_TRY(dmalloc(allocs_, (void**)&ws_, ws_bytes_));
  const int m_tiles_lm = (lm_rows_l_ + GEMM_BM - 1) / GEMM_BM;
  ACP_TRY(dmalloc_t(allocs_, &amax_val_, (size_t)Bp * m_tiles_lm));
  ACP_TRY(dmalloc_t(allocs_, &amax_idx_, (size_t)Bp * m_tiles_lm));
  ACP_TRY(dmalloc_t(allocs_, &logits_, (size_t)lim_.max_batch * lm_rows_per_rank_));
  if (tp_size_ > 1) {
    ACP_TRY(dmalloc_t(allocs_, &logits_gather_, (size_t)tp_size_ * lim_.max_batch * lm_rows_per_rank_));
    ACP_TRY(dmalloc_t(allocs_, &logits_full_, (size_t)lim_.max_batch * cfg_.vocab));
  }
  attn_max_chunks_ = attn_decode_chunks(lim_.max_pages_per_seq * KV_PAGE);
  ACP_TRY(dmalloc_t(allocs_, &attn_ws_, attn_decode_ws_floats(lim_.max_batch, heads_l_, kvh_l_, attn_max_chunks_)));
  // step staging
  ints_cap_ = (size_t)5 * lim_.max_tokens + (size_t)6 * lim_.max_batch +
              (size_t)lim_.max_batch * lim_.max_pages_per_seq + 64;
  ACP_TRY(dmalloc_t(allocs_, &d_ints_, ints_cap_));
  ACP_CUDA_CHECK(cudaMallocHost((void**)&h_ints_, ints_cap_ * sizeof(int)));
  ACP_TRY(dmalloc_t(allocs_, &d_sparams_, (size_t)lim_.max_batch));
  ACP_CUDA_CHECK(cudaMallocHost((void**)&h_sparams_, lim_.max_batch * sizeof(SampleParams)));
  ACP_TRY(dmalloc_t(allocs_, &d_tokens_, (size_t)lim_.max_batch));
  ACP_CUDA_CHECK(cudaMallocHost((void**)&h_tokens_, lim_.max_batch * sizeof(int)));
  ACP_CUDA_CHECK(cudaMallocHost((void**)&h_logits_, (size_t)lim_.max_batch * (tp_rank_ == 0 ? cfg_.vocab : GEMM_BM) * sizeof(float)));
  return 0;
}

int Model::gen_weights() {
  const ModelConfig& c = cfg_;
  const size_t H = c.hidden;
  // tensor ids shared with oracle/synth.py; SynthMap places this shard inside the logical tensors
  const int r = tp_rank_;
  auto tiled = [&](int local_cols, int logical_cols, int col0) {
    SynthMap m;
    m.local_cols = local_cols; m.logical_cols = logical_cols; m.col0 = col0;
    return m;
  };
  ACP_TRY(launch_synth(embed_, (size_t)c.vocab * H, c.seed, 1, c.w_std, 0, stream_));  // replicated, row-major
  {
    SynthMap m = tiled((int)H, (int)H, 0);
    m.nseg = 1; m.seg_rows[0] = lm_rows_l_; m.seg_global[0] = lm_row0_;
    ACP_TRY(launch_synth(lm_head_, (size_t)lm_rows_l_ * H, c.seed, 2, c.w_std, 0, stream_, m));
  }
  ACP_TRY(launch_synth(final_norm_, H, c.seed, 3, 0.1, 1, stream_));
  for (int l = 0; l < c.layers; ++l) {
    Layer& L = layers_[l];
    const uint32_t base = 16 + (uint32_t)l * 16;
    {  // [q heads of this rank | k heads | v heads] rows of the logical [q | k | v] tensor
      SynthMap m = tiled((int)H, (int)H, 0);
      m.nseg = 3;
      m.seg_rows[0] = qdim_l_; m.seg_global[0] = r * qdim_l_;
      m.seg_rows[1] = kvdim_l_; m.seg_global[1] = c.q_dim() + r * kvdim_l_;
      m.seg_rows[2] = kvdim_l_; m.seg_global[2] = c.q_dim() + c.kv_dim() + r * kvdim_l_;
      ACP_TRY(launch_synth(L.wqkv, (size_t)qkv_l_ * H, c.seed, base + 0, c.w_std, 0, stream_, m));
    }
    ACP_TRY(launch_synth(L.wo, H * qdim_l_, c.seed, base + 1, c.w_std, 0, stream_, tiled(qdim_l_, c.q_dim(), r * qdim_l_)));
    if (c.experts > 0) {
      // tensor ids of oracle/synth.py: router = layer_tid(l, 6); expert e: expert_tid(l, e, 0 = [gate; up] | 1 = down)
      ACP_TRY(launch_synth(L.router, (size_t)c.experts * H, c.seed, base + 6, c.w_std, 0, stream_));
      for (int j = 0; j < experts_l_; ++j) {
        const uint32_t etid = (1u << 20) + (uint32_t)l * 256u + (uint32_t)(expert0_ + j) * 2u;
        SynthMap m = tiled((int)H, (int)H, 0);
        m.interleave_half = c.ffn;
        m.seg_global[0] = 0;
        m.seg_global[1] = c.ffn;
        ACP_TRY(launch_synth(L.wgu_e + (size_t)j * 2 * c.ffn * H, (size_t)2 * c.ffn * H, c.seed, etid, c.w_std, 0, stream_, m));
        ACP_TRY(launch_synth(L.wdown_e + (size_t)j * H * c.ffn, H * c.ffn, c.seed, etid + 1, c.w_std, 0, stream_, tiled(c.ffn, c.ffn, 0)));
      }
    } else {
      {  // gate/up rows interleaved (2j = gate_j, 2j+1 = up_j); values = oracle's [gate; up] tensor
        SynthMap m = tiled((int)H, (int)H, 0);
        m.interleave_half = ffn_l_;
        m.seg_global[0] = r * ffn_l_;
        m.seg_global[1] = c.ffn + r * ffn_l_;
        ACP_TRY(launch_synth(L.wgu, (size_t)2 * ffn_l_ * H, c.seed, base + 2, c.w_std, 0, stream_, m));
      }
      ACP_TRY(launch_synth(L.wdown, H * ffn_l_, c.seed, base + 3, c.w_std, 0, stream_, tiled(ffn_l_, c.ffn, r * ffn_l_)));
    }
    ACP_TRY(launch_synth(L.attn_norm, H, c.seed, base + 4, 0.1, 1, stream_));
    ACP_TRY(launch_synth(L.ffn_norm, H, c.seed, base + 5, 0.1, 1, stream_));
  }
  return 0;
}

// RoPE tables: same recipe as oracle/llama_oracle.py rope_tables()
int Model::build_rope_tables() {
  const ModelConfig& c = cfg_;
  std::vector<float> hc((size_t)c.max_pos * 64), hs((size_t)c.max_pos * 64);
  float inv[64];
  rope_inv_freq(c, inv);
  for (int p = 0; p < c.max_pos; ++p)
    for (int i = 0; i < 64; ++i) {
      const float ang = (float)p * inv[i];
      hc[(size_t)p * 64 + i] = (float)cos((double)ang);
      hs[(size_t)p * 64 + i] = (float)sin((double)ang);
    }
  ACP_CUDA_CHECK(cudaMemcpyAsync(cos_, hc.data(), hc.size() * 4, cudaMemcpyHostToDevice, stream_));
  ACP_CUDA_CHECK(cudaMemcpyAsync(sin_, hs.data(), hs.size() * 4, cudaMemcpyHostToDevice, stream_));
  ACP_CUDA_CHECK(cudaStreamSynchronize(stream_));
  return 0;
}

// HuggingFace Llama checkpoint -> this shard's tiled weights.  Every logical tensor ([q;k;v],
// o_proj, [gate;up], down_proj, lm_head rows of this shard) is staged row-major on the device and
// placed by gather_weight_kernel through the SAME SynthMap the synthetic generator uses.
int Model::load_weights(const Checkpoint& ck) {
  const ModelConfig& c = cfg_;

  const size_t H = c.hidden;
  const int r = tp_rank_;
  size_t stage_elems = (size_t)c.qkv_dim() * H;
  if ((size_t)2 * c.ffn * H > stage_elems) stage_elems = (size_t)2 * c.ffn * H;
  if ((size_t)lm_rows_l_ * H > stage_elems) stage_elems = (size_t)lm_rows_l_ * H;
  __nv_bfloat16* stage = nullptr;
  ACP_CUDA_CHECK(cudaMalloc((void**)&stage, stage_elems * sizeof(__nv_bfloat16)));
  std::vector<uint16_t> conv;  // host conversion buffer for F16/F32 checkpoints
  struct Part { std::string name; int64_t rows, cols; int64_t row0, nrows; };
  int rc = 0;
  // copies rows [row0, row0+nrows) of a [rows][cols] tensor to dst (device, bf16)
  auto upload = [&](const Part& p, __nv_bfloat16* dst) -> int {
    const StTensor* t = ck.find(p.name);
    if (!t) { fprintf(stderr, "[acp_infer] checkpoint is missing %s\n", p.name.c_str()); return -1; }
    const bool shape_ok = p.cols == 1 ? (t->shape.size() == 1 && t->shape[0] == p.rows)
                                      : (t->shape.size() == 2 && t->shape[0] == p.rows && t->shape[1] == p.cols);
    if (!shape_ok) { fprintf(stderr, "[acp_infer] %s has an unexpected shape\n", p.name.c_str()); return -1; }
    const size_t e0 = (size_t)p.row0 * (size_t)p.cols, n = (size_t)p.nrows * (size_t)p.cols;
    if (t->dtype == "BF16") {
      ACP_CUDA_CHECK(cudaMemcpyAsync(dst, t->data + e0 * 2, n * 2, cudaMemcpyHostToDevice, stream_));
      ACP_CUDA_CHECK(cudaStreamSynchronize(stream_));
      return 0;
    }
    const size_t chunk = (size_t)16 << 20;
    conv.resize(n < chunk ? n : chunk);
    for (size_t o = 0; o < n; o += chunk) {
      const size_t m = n - o < chunk ? n - o : chunk;
      if (!st_to_bf16(*t, e0 + o, m, conv.data())) {
        fprintf(stderr, "[acp_infer] %s: dtype %s is not supported (BF16, F16, F32)\n", p.name.c_str(), t->dtype.c_str());
        return -1;
      }
      ACP_CUDA_CHECK(cudaMemcpyAsync(dst + o, conv.data(), m * 2, cudaMemcpyHostToDevice, stream_));
      ACP_CUDA_CHECK(cudaStreamSynchronize(stream_));
    }
    return 0;
  };
  auto tiled = [&](int local_cols, int logical_cols, int col0) {
    SynthMap m;
    m.local_cols = local_cols; m.logical_cols = logical_cols; m.col0 = col0;
    return m;
  };
  auto whole = [&](const std::string& name, int64_t rows, int64_t cols) { return Part{name, rows, cols, 0, rows}; };
  do {
    if ((rc = upload(whole("model.embed_tokens.weight", c.vocab, H), embed_)) != 0) break;
    {  // LM head: this shard's rows only (contiguous in the logical tensor)
      const bool tied = c.tied_embeddings || !ck.find("lm_head.weight");
      Part p{tied ? "model.embed_tokens.weight" : "lm_head.weight", c.vocab, (int64_t)H, lm_row0_, lm_rows_l_};
      if ((rc = upload(p, stage)) != 0) break;
      SynthMap m = tiled((int)H, (int)H, 0);
      m.nseg = 1; m.seg_rows[0] = lm_rows_l_; m.seg_global[0] = lm_row0_;
      if ((rc = launch_gather_weight(lm_head_, (size_t)lm_rows_l_ * H, stage, (size_t)lm_row0_ * H, stream_, m)) != 0) break;
      ACP_CUDA_CHECK(cudaStreamSynchronize(stream_));
    }
    if ((rc = upload(whole("model.norm.weight", H, 1), final_norm_)) != 0) break;
    for (int l = 0; l < c.layers && rc == 0; ++l) {
      Layer& L = layers_[l];
      const std::string pre = "model.layers." + std::to_string(l) + ".";
      {  // logical [q; k; v]
        if ((rc = upload(whole(pre + "self_attn.q_proj.weight", c.q_dim(), H), stage)) != 0) break;
        if ((rc = upload(whole(pre + "self_attn.k_proj.weight", c.kv_dim(), H), stage + (size_t)c.q_dim() * H)) != 0) break;
        if ((rc = upload(whole(pre + "self_attn.v_proj.weight", c.kv_dim(), H), stage + (size_t)(c.q_dim() + c.kv_dim()) * H)) != 0) break;
        SynthMap m = tiled((int)H, (int)H, 0);
        m.nseg = 3;
        m.seg_rows[0] = qdim_l_; m.seg_global[0] = r * qdim_l_;
        m.seg_rows[1] = kvdim_l_; m.seg_global[1] = c.q_dim() + r * kvdim_l_;
        m.seg_rows[2] = kvdim_l_; m.seg_global[2] = c.q_dim() + c.kv_dim() + r * kvdim_l_;
        if ((rc = launch_gather_weight(L.wqkv, (size_t)qkv_l_ * H, stage, 0, stream_, m)) != 0) break;
        ACP_CUDA_CHECK(cudaStreamSynchronize(stream_));
      }
      if ((rc = upload(whole(pre + "self_attn.o_proj.weight", H, c.q_dim()), stage)) != 0) break;
      if ((rc = launch_gather_weight(L.wo, H * qdim_l_, stage, 0, stream_, tiled(qdim_l_, c.q_dim(), r * qdim_l_))) != 0) break;
      ACP_CUDA_CHECK(cudaStreamSynchronize(stream_));
      if (c.experts > 0) {
        // Mixtral (hub layout): block_sparse_moe.gate.weight [E][H]; experts.<e>.w1 = gate, w3 = up ([ffn][H]), w2 = down ([H][ffn])
        const std::string moe = pre + "block_sparse_moe.";
        if ((rc = upload(whole(moe + "gate.weight", c.experts, H), L.router)) != 0) break;
        for (int j = 0; j < experts_l_ && rc == 0; ++j) {
          const std::string ex = moe + "experts." + std::to_string(expert0_ + j) + ".";
          if ((rc = upload(whole(ex + "w1.weight", c.ffn, H), stage)) != 0) break;
          if ((rc = upload(whole(ex + "w3.weight", c.ffn, H), stage + (size_t)c.ffn * H)) != 0) break;
          SynthMap m = tiled((int)H, (int)H, 0);
          m.interleave_half = c.ffn;
          m.seg_global[0] = 0;
          m.seg_global[1] = c.ffn;
          if ((rc = launch_gather_weight(L.wgu_e + (size_t)j * 2 * c.ffn * H, (size_t)2 * c.ffn * H, stage, 0, stream_, m)) != 0) break;
          ACP_CUDA_CHECK(cudaStreamSynchronize(stream_));
          if ((rc = upload(whole(ex + "w2.weight", H, c.ffn), stage)) != 0) break;
          if ((rc = launch_gather_weight(L.wdown_e + (size_t)j * H * c.ffn, H * c.ffn, stage, 0, stream_, tiled(c.ffn, c.ffn, 0))) != 0) break;
          ACP_CUDA_CHECK(cudaStreamSynchronize(stream_));
        }
        if (rc != 0) break;
        if ((rc = upload(whole(pre + "input_layernorm.weight", H, 1), L.attn_norm)) != 0) break;
        if ((rc = upload(whole(pre + "post_attention_layernorm.weight", H, 1), L.ffn_norm)) != 0) break;
        continue;
      }
      {  // logical [gate; up], stored interleaved (2j = gate_j, 2j+1 = up_j)
        if ((rc = upload(whole(pre + "mlp.gate_proj.weight", c.ffn, H), stage)) != 0) break;
        if ((rc = upload(whole(pre + "mlp.up_proj.weight", c.ffn, H), stage + (size_t)c.ffn * H)) != 0) break;
        SynthMap m = tiled((int)H, (int)H, 0);
        m.interleave_half = ffn_l_;
        m.seg_global[0] = r * ffn_l_;
        m.seg_global[1] = c.ffn + r * ffn_l_;
        if ((rc = launch_gather_weight(L.wgu, (size_t)2 * ffn_l_ * H, stage, 0, stream_, m)) != 0) break;
        ACP_CUDA_CHECK(cudaStreamSynchronize(stream_));
      }
      if ((rc = upload(whole(pre + "mlp.down_proj.weight", H, c.ffn), stage)) != 0) break;
      if ((rc = launch_gather_weight(L.wdown, H * ffn_l_, stage, 0, stream_, tiled(ffn_l_, c.ffn, r * ffn_l_))) != 0) break;
      ACP_CUDA_CHECK(cudaStreamSynchronize(stream_));
      if ((rc = upload(whole(pre + "input_layernorm.weight", H, 1), L.attn_norm)) != 0) break;
      if ((rc = upload(whole(pre + "post_attention_layernorm.weight", H, 1), L.ffn_norm)) != 0) break;
    }
  } while (false);
  cudaFree(stage);
  return rc;
}

static inline size_t align4(size_t v) { return (v + 3) & ~(size_t)3; }

StepInput& Model::stage_begin(int T, int B, int n_blocks) {
  StepInput& s = stage_;
  s = StepInput();
  s.T = T; s.B = B; s.n_blocks = n_blocks;
  size_t off = 0;
  auto carve = [&](size_t n) { int* p = h_ints_ + off; off += align4(n); return p; };
  s.tok = carve(T); s.pos = carve(T); s.seq_of_row = carve(T);
  s.q_start = carve(B); s.q_len = carve(B); s.ctx_len = carve(B); s.sample_rows = carve(B);
  s.blk_seq = carve(n_blocks); s.blk_tok0 = carve(n_blocks);
  s.page_table = carve((size_t)B * lim_.max_pages_per_seq);
  s.tile_cum = carve((size_t)B + 1);
  ints_used_ = off;
  s.sample_params = h_sparams_;
  return s;
}

int Model::gemm(const TmaMaps& w, const TmaMaps& x, int M, int K, int N, bool decode, GemmOut* out) {
  GemmLaunch g;
  g.tp_shard = tp_size_ > 1;
  g.w = &w.w; g.x = &x; g.M = M; g.N = N; g.K = K;
  const int splits = choose_splits(M, K, N);
  if (decode && splits > 1) {  // a single split writes bf16 directly (same rounding, half the bytes)
    g.epi = EPI_F32; g.splits = splits; g.out = ws_; g.ld = M; g.n_cap = N;
    if ((size_t)splits * N * M * sizeof(float) > ws_bytes_) { fprintf(stderr, "[acp_infer] split-K workspace too small: %d planes x %d x %d\n", splits, N, M); return -4; }
    out->ptr = ws_; out->splits = splits; out->n_cap = N; out->ld = M;
  } else {
    g.epi = EPI_BF16; g.splits = 1; g.out = gemm_bf16_; g.ld = M; g.n_cap = N;
    out->ptr = gemm_bf16_; out->splits = 0; out->n_cap = N; out->ld = M;
  }
  ++launches_;
  return gemm_launch(g, stream_);
}

// Row-parallel GEMM of a tensor-parallel shard (O and down projections): fp32 partial sums, local
// split-K reduce, NCCL all-reduce (sum) across the group over NVLink, consumer rounds to bf16 ONCE.
int Model::gemm_rowpar(const TmaMaps& w, const TmaMaps& x, int M, int K, int N, bool decode, GemmOut* out) {
  GemmLaunch g;
  g.tp_shard = tp_size_ > 1;
  g.w = &w.w; g.x = &x; g.M = M; g.N = N; g.K = K;
  const int splits = decode ? choose_splits(M, K, N) : 1;
  g.epi = EPI_F32; g.splits = splits; g.out = ws_; g.ld = M; g.n_cap = N;
  if ((size_t)splits * N * M * sizeof(float) > ws_bytes_) { fprintf(stderr, "[acp_infer] split-K workspace too small: %d planes x %d x %d\n", splits, N, M); return -4; }
  ++launches_;
  int rc = gemm_launch(g, stream_);
  if (rc != 0) return rc;
  float* ar = ws_;
  if (splits > 1) {
    rc = launch_reduce_planes(ws_, splits, (size_t)N * M, ar_buf_, stream_);
    if (rc != 0) return rc;
    ++launches_;
    ar = ar_buf_;
  }
  const NcclApi& nc = nccl_api();
  rc = nc.AllReduce(ar, ar, (size_t)N * M, kNcclFloat32, kNcclSum, comm_, stream_);
  if (rc != 0) { fprintf(stderr, "[acp_infer] ncclAllReduce: %s\n", nc.GetErrorString(rc)); return -5; }
  ++launches_;
  out->ptr = ar; out->splits = 1; out->n_cap = N; out->ld = M;
  return 0;
}

// Row-parallel GEMM + the fused peer-memory exchange of tp_comm.cu:
//   GEMM (fp32 partial planes) -> local split-K reduce -> barrier -> pull/reduce/residual/RMSNorm/
//   push -> barrier.  x_ and xn_ are updated on EVERY rank by the rank that owns the row.
int Model::rowpar_fused(const TmaMaps& w, const TmaMaps& x, int K, int N, bool decode, const __nv_bfloat16* gain,
                        bool push_x) {
  const int M = cfg_.hidden;
  GemmLaunch g;
  g.tp_shard = tp_size_ > 1;
  g.w = &w.w; g.x = &x; g.M = M; g.N = N; g.K = K;
  const int splits = decode ? choose_splits(M, K, N) : 1;
  g.epi = EPI_F32; g.splits = splits; g.ld = M; g.n_cap = N;
  g.out = splits > 1 ? ws_ : ar_buf_;
  if (splits > 1 && (size_t)splits * N * M * sizeof(float) > ws_bytes_) { fprintf(stderr, "[acp_infer] split-K workspace too small: %d planes x %d x %d\n", splits, N, M); return -4; }
  int rc = gemm_launch(g, stream_);
  if (rc != 0) return rc;
  ++launches_;
  if (splits > 1) {
    rc = launch_reduce_planes(ws_, splits, (size_t)N * M, ar_buf_, stream_);
    if (rc != 0) return rc;
    ++launches_;
  }
  const int epoch = tp_epoch_ + 1;
  tp_epoch_ += 2;
  rc = launch_tp_reduce_norm(peers_, N, M, gain, cfg_.eps, epoch, tp_flags_ + TP_MAX, push_x, stream_);
  ++launches_;  // the kernel itself waits until every rank's rows have landed here
  return rc;
}

// Micro-benchmark of the bare exchange (no GEMM): every shard must call it with the same arguments.
int Model::bench_exchange(int T, int iters, float* avg_us, int diag) {
  if (!have_peers_ || T > lim_.max_tokens) return -1;
  ACP_CUDA_CHECK(cudaSetDevice(device_));
  cudaEvent_t a, b;
  ACP_CUDA_CHECK(cudaEventCreate(&a));
  ACP_CUDA_CHECK(cudaEventCreate(&b));
  ACP_CUDA_CHECK(cudaMemsetAsync(ar_buf_, 0, (size_t)T * cfg_.hidden * sizeof(float), stream_));
  int rc = 0;
  for (int i = 0; i < iters + 10 && rc == 0; ++i) {
    if (i == 10) cudaEventRecord(a, stream_);
    const int epoch = tp_epoch_ + 1;
    tp_epoch_ += 2;
    rc = launch_tp_reduce_norm(peers_, T, cfg_.hidden, layers_[0].ffn_norm, cfg_.eps, epoch, tp_flags_ + TP_MAX, false, stream_, diag);
  }
  cudaEventRecord(b, stream_);
  ACP_CUDA_CHECK(cudaStreamSynchronize(stream_));
  float ms = 0.f;
  cudaEventElapsedTime(&ms, a, b);
  *avg_us = 1e3f * ms / (float)iters;
  cudaEventDestroy(a);
  cudaEventDestroy(b);
  return rc;
}

int Model::forward(const StepInput& in) {
  const ModelConfig& c = cfg_;
  if (in.T <= 0 || in.T > lim_.max_tokens || in.B > lim_.max_batch || in.n_sample > lim_.max_batch) {
    fprintf(stderr, "[acp_infer] step outside the model limits: T=%d (max %d) B=%d n_sample=%d (max_batch %d)\n", in.T, lim_.max_tokens, in.B,
            in.n_sample, lim_.max_batch);
    return -1;
  }
  ACP_CUDA_CHECK(cudaSetDevice(device_));
  // every tensor-parallel shard uploads the SAME pinned step descriptor (the lead shard's staging)
  const int* src_ints = lead_ ? lead_->h_ints_ : h_ints_;
  const size_t used = lead_ ? lead_->ints_used_ : ints_used_;
  ACP_CUDA_CHECK(cudaMemcpyAsync(d_ints_, src_ints, used * sizeof(int), cudaMemcpyHostToDevice, stream_));
  h2d_bytes_ += (long long)(used * sizeof(int));
  auto dev = [&](const int* hp) { return d_ints_ + (hp - src_ints); };
  const int* d_tok = dev(in.tok);
  const int* d_pos = dev(in.pos);
  const int* d_seq = dev(in.seq_of_row);
  const int* d_qstart = dev(in.q_start);
  const int* d_qlen = dev(in.q_len);
  const int* d_ctx = dev(in.ctx_len);
  const int* d_srows = dev(in.sample_rows);
  const int* d_bseq = dev(in.blk_seq);
  const int* d_btok0 = dev(in.blk_tok0);
  const int* d_pt = dev(in.page_table);
  const int T = in.T;
  const float scale = 1.0f / sqrtf((float)HEAD_DIM);

  PROF("embed", launch_embed(d_tok, embed_, x_, T, c.hidden, stream_));
  ++launches_;
  GemmOut none;
  PROF("rmsnorm_first", launch_add_rmsnorm(x_, none, layers_[0].attn_norm, xn_, nullptr, T, c.hidden, c.eps, stream_));
  ++launches_;
  for (int l = 0; l < c.layers; ++l) {
    Layer& L = layers_[l];
    GemmOut qkv, o, dn;
    // investigation knob (ACP_TP_SYNC_EVERY): bound this shard's launch queue
    if (tp_sync_every_ > 0 && l > 0 && l % tp_sync_every_ == 0) ACP_CUDA_CHECK(cudaStreamSynchronize(stream_));
    PROF("gemm_qkv", gemm(L.m_qkv, m_xn_, qkv_l_, c.hidden, T, in.decode, &qkv));
    if (!in.decode) {
      RopeKvArgs ra;
      ra.qkv = qkv; ra.pos = d_pos; ra.seq_of_row = d_seq; ra.page_table = d_pt;
      ra.max_pages = lim_.max_pages_per_seq; ra.cos_tab = cos_; ra.sin_tab = sin_; ra.qbuf = qbuf_;
      ra.k_cache = L.k_cache; ra.v_cache = L.v_cache; ra.T = T; ra.heads = heads_l_; ra.kv_heads = kvh_l_;
      PROF("rope_kv", launch_rope_kv(ra, stream_));
      ++launches_;
    }
    if (in.decode) {
      AttnDecodeArgs aa;
      aa.q = qbuf_; aa.out = attn_; aa.ctx_len = d_ctx; aa.chunk_cum = dev(in.tile_cum); aa.page_table = d_pt;
      aa.max_pages = lim_.max_pages_per_seq; aa.heads = heads_l_; aa.kv_heads = kvh_l_;
      aa.num_seqs = in.B;
      aa.total_chunks = in.tile_cum[in.B];   // host copy of the prefix sum (filled by the engine)
      aa.max_chunks = attn_max_chunks_;
      aa.scale = scale; aa.ws = attn_ws_;
      // decode: RoPE + KV append are fused into the attention kernel (no rope_kv launch)
      aa.qkv_ptr = qkv.ptr; aa.qkv_splits = qkv.splits; aa.qkv_n_cap = qkv.n_cap; aa.qkv_ld = qkv.ld;
      aa.cos_tab = cos_; aa.sin_tab = sin_; aa.k_cache = L.k_cache; aa.v_cache = L.v_cache;
      // every item fits one chunk: one CTA per item writes the output directly (identical
      // arithmetic to chunked + merge for a single chunk, so the choice never changes results)
      aa.per_item = (aa.total_chunks == in.B) ? 1 : 0;
      if (lim_.attn_decode_mode == 1 && aa.total_chunks == in.B) aa.per_item = 1;
      if (lim_.attn_decode_mode == 2) aa.per_item = 0;
      PROF("attn_decode", launch_attn_decode(L.tm_k, L.tm_v, aa, stream_));
      launches_ += aa.per_item ? 1 : 2;
    } else {
      AttnPrefillArgs pa;
      pa.q = qbuf_; pa.out = attn_; pa.blk_seq = d_bseq; pa.blk_tok0 = d_btok0; pa.q_start = d_qstart;
      pa.q_len = d_qlen; pa.ctx_len = d_ctx; pa.page_table = d_pt; pa.max_pages = lim_.max_pages_per_seq;
      pa.heads = heads_l_; pa.kv_heads = kvh_l_; pa.scale = scale;
      if (attn_prefill_tc_enabled()) PROF("attn_prefill", launch_attn_prefill_tc(tm_q_, L.tm_k32, L.tm_v32, pa, in.n_blocks, stream_));
      else PROF("attn_prefill", launch_attn_prefill(L.tm_k, L.tm_v, pa, in.n_blocks, stream_));
      ++launches_;
    }
    if (tp_size_ > 1 && have_peers_) {
      PROF("gemm_o+p2p_allreduce_norm", rowpar_fused(L.m_o, m_attn_, qdim_l_, T, in.decode, L.ffn_norm, false));
    } else {
      if (tp_size_ > 1) PROF("gemm_o_allreduce", gemm_rowpar(L.m_o, m_attn_, c.hidden, qdim_l_, T, in.decode, &o));
      else PROF("gemm_o", gemm(L.m_o, m_attn_, c.hidden, qdim_l_, T, in.decode, &o));
      PROF("add_rmsnorm_o", launch_add_rmsnorm(x_, o, L.ffn_norm, xn_, nullptr, T, c.hidden, c.eps, stream_));
      ++launches_;
    }
    if (c.experts > 0) {
      const __nv_bfloat16* gain = (l + 1 < c.layers) ? layers_[l + 1].attn_norm : final_norm_;
      ACP_TRY(moe_mlp(L, T, gain, l + 1 == c.layers));
      if (l + 1 == c.layers) {
        // moe_mlp left the residual added in x_ on this rank: normalise the sampled rows into xs_
        GemmOut nothing;
        PROF("add_rmsnorm_final", launch_add_rmsnorm(x_, nothing, final_norm_, xs_, d_srows, in.n_sample, c.hidden, c.eps, stream_));
        ++launches_;
      }
      continue;
    }
    if (fuse_swiglu_ || (!in.decode && T > 256 && fuse_swiglu_prefill_)) {
      // SwiGLU in the GEMM epilogue.  Decode (non-persistent kernel, epilogue exposed at the end of
      // every CTA) measured no gain, so it stays a separate kernel there unless ACP_FUSE_SWIGLU=1.
      GemmLaunch g;
      g.tp_shard = tp_size_ > 1;
      g.w = &L.m_gu.w; g.x = &m_xn_; g.M = 2 * ffn_l_; g.N = T; g.K = c.hidden; g.splits = 1;
      g.epi = EPI_SWIGLU; g.out = h_; g.ld = ffn_l_; g.n_cap = T;
      PROF("gemm_gateup_swiglu", gemm_launch(g, stream_));
      ++launches_;
    } else {
      GemmOut gu;
      PROF("gemm_gateup", gemm(L.m_gu, m_xn_, 2 * ffn_l_, c.hidden, T, in.decode, &gu));
      PROF("swiglu", launch_swiglu(gu, h_, T, ffn_l_, stream_));
      ++launches_;
    }
    if (tp_size_ > 1 && have_peers_) {
      // fused exchange writes x_ and xn_ (with the next layer's gain; the last layer's xn_ is unused)
      const __nv_bfloat16* gain = (l + 1 < c.layers) ? layers_[l + 1].attn_norm : final_norm_;
      PROF("gemm_down+p2p_allreduce_norm", rowpar_fused(L.m_down, m_h_, ffn_l_, T, in.decode, gain, l + 1 == c.layers));
      if (l + 1 == c.layers) {
        GemmOut nothing;
        PROF("add_rmsnorm_final", launch_add_rmsnorm(x_, nothing, final_norm_, xs_, d_srows, in.n_sample, c.hidden, c.eps, stream_));
        ++launches_;
      }
      continue;
    }
    if (tp_size_ > 1) PROF("gemm_down_allreduce", gemm_rowpar(L.m_down, m_h_, c.hidden, ffn_l_, T, in.decode, &dn));
    else PROF("gemm_down", gemm(L.m_down, m_h_, c.hidden, ffn_l_, T, in.decode, &dn));
    if (l + 1 < c.layers) {
      PROF("add_rmsnorm_down", launch_add_rmsnorm(x_, dn, layers_[l + 1].attn_norm, xn_, nullptr, T, c.hidden, c.eps, stream_));
    } else {
      // final norm only on the rows that are sampled (residual add folded in, not written back)
      PROF("add_rmsnorm_final", launch_add_rmsnorm(x_, dn, final_norm_, xs_, d_srows, in.n_sample, c.hidden, c.eps, stream_));
    }
    ++launches_;
  }
  if (in.n_sample > 0) {
    const int m_tiles = (lm_rows_l_ + GEMM_BM - 1) / GEMM_BM;
    GemmLaunch g;
    g.tp_shard = tp_size_ > 1;
    g.w = &m_lm_.w; g.x = &m_xs_; g.M = lm_rows_l_; g.N = in.n_sample; g.K = c.hidden; g.splits = 1;
    g.epi = EPI_ARGMAX; g.ld = lm_rows_per_rank_; g.n_cap = in.n_sample;   // == lm_rows_l_ when tp == 1
    const bool logits = in.want_logits || !in.all_greedy;
    g.out = logits ? logits_ : nullptr;
    const float* full_logits = logits_;
    g.amax_val = amax_val_; g.amax_idx = amax_idx_;
    PROF("gemm_lm_head_argmax", gemm_launch(g, stream_));
    ++launches_;
    if (tp_size_ > 1) {
      // vocab-parallel: local arg-max, all-gather the (max, global id) candidates, pick the best
      ACP_TRY(launch_argmax_finish(amax_val_, amax_idx_, m_tiles, in.n_sample, d_tokens_, amax_val_row_, stream_));
      ACP_TRY(launch_pack_candidates(amax_val_row_, d_tokens_, lm_row0_, in.n_sample, cand_local_, stream_));
      const NcclApi& nc = nccl_api();
      int rc = nc.AllGather(cand_local_, cand_all_, (size_t)2 * in.n_sample * sizeof(int), kNcclInt8, comm_, stream_);
      if (rc != 0) { fprintf(stderr, "[acp_infer] ncclAllGather: %s\n", nc.GetErrorString(rc)); return -5; }
      ACP_TRY(launch_argmax_ranks(cand_all_, tp_size_, in.n_sample, d_tokens_, stream_));
      launches_ += 4;
      if (logits) {
        // sampling / return_logits under a vocab-parallel LM head: all-gather the padded logit
        // shards ([n][rows per rank] per rank) and re-pack them as [n][vocab]; every rank then runs
        // the same sampler on the same bits (only rank 0's tokens / logits leave the device)
        rc = nc.AllGather(logits_, logits_gather_, (size_t)in.n_sample * lm_rows_per_rank_ * sizeof(float), kNcclInt8, comm_, stream_);
        if (rc != 0) { fprintf(stderr, "[acp_infer] ncclAllGather(logits): %s\n", nc.GetErrorString(rc)); return -5; }
        ACP_TRY(launch_repack_logits(logits_gather_, tp_size_, in.n_sample, lm_rows_per_rank_, c.vocab, logits_full_, stream_));
        launches_ += 2;
        full_logits = logits_full_;
        if (!in.all_greedy) {
          ACP_CUDA_CHECK(cudaMemcpyAsync(d_sparams_, lead_ ? lead_->h_sparams_ : h_sparams_, in.n_sample * sizeof(SampleParams),
                                         cudaMemcpyHostToDevice, stream_));
          h2d_bytes_ += (long long)(in.n_sample * sizeof(SampleParams));
          ACP_TRY(launch_sample(full_logits, c.vocab, in.n_sample, d_sparams_, d_tokens_, stream_));   // greedy rows: same arg-max, lowest id
        }
      }
    } else if (in.all_greedy) {
      PROF("argmax_finish", launch_argmax_finish(amax_val_, amax_idx_, m_tiles, in.n_sample, d_tokens_, nullptr, stream_));
    } else {
      ACP_CUDA_CHECK(cudaMemcpyAsync(d_sparams_, h_sparams_, in.n_sample * sizeof(SampleParams),
                                     cudaMemcpyHostToDevice, stream_));
      h2d_bytes_ += (long long)(in.n_sample * sizeof(SampleParams));
      ACP_TRY(launch_sample(logits_, c.vocab, in.n_sample, d_sparams_, d_tokens_, stream_));
    }
    ++launches_;
    if (tp_rank_ == 0) {
      ACP_CUDA_CHECK(cudaMemcpyAsync(h_tokens_, d_tokens_, in.n_sample * sizeof(int), cudaMemcpyDeviceToHost, stream_));
      d2h_bytes_ += (long long)(in.n_sample * sizeof(int));
      if (in.want_logits) {
        d2h_bytes_ += (long long)in.n_sample * c.vocab * (long long)sizeof(float);
        ACP_CUDA_CHECK(cudaMemcpyAsync(h_logits_, full_logits, (size_t)in.n_sample * c.vocab * sizeof(float),
                                       cudaMemcpyDeviceToHost, stream_));
      }
    }
  }
  return 0;
}

// Sparse MoE MLP of one layer (Mixtral; oracle/llama_oracle.py _moe): router -> dispatch -> gather ->
// grouped gate/up GEMM with fused SwiGLU -> grouped down GEMM -> weighted combine -> residual + next norm.
// The expert GEMMs never split K (prefill and decode share one arithmetic path).
int Model::moe_mlp(Layer& L, int T, const __nv_bfloat16* gain, bool last_layer) {
  const ModelConfig& c = cfg_;
  PROF("moe_router", launch_moe_router(xn_, L.router, c.hidden, c.experts, T, moe_topk_idx_, moe_topk_w_, stream_));
  // N tile of the expert GEMMs: an expert sees about 2T / E rows (a token picks an expert at most once)
  const int bn = gemm_pick_bn((2 * T + c.experts - 1) / c.experts);
  PROF("moe_dispatch", launch_moe_dispatch(moe_topk_idx_, T, expert0_, experts_l_, bn, moe_ranges_, moe_row_of_, stream_));
  PROF("moe_gather", launch_moe_gather(xn_, moe_row_of_, c.hidden, T, xe_, stream_));
  GemmLaunch g;
  g.tp_shard = tp_size_ > 1;
  g.groups = experts_l_; g.group_ranges = moe_ranges_; g.splits = 1;
  g.bn_override = bn;
  g.N = moe_tile_cap(T, bn, experts_l_) * bn;   // grid.x = capacity of the device-side tile list
  g.w = &L.m_gu_e.w; g.x = &m_xe_; g.M = 2 * c.ffn; g.K = c.hidden; g.epi = EPI_SWIGLU; g.out = he_; g.ld = c.ffn; g.n_cap = T;
  PROF("gemm_experts_gateup_swiglu", gemm_launch(g, stream_));
  g.w = &L.m_down_e.w; g.x = &m_he_; g.M = c.hidden; g.K = c.ffn; g.epi = EPI_BF16; g.out = ye_; g.ld = c.hidden;
  PROF("gemm_experts_down", gemm_launch(g, stream_));
  launches_ += 5;
  if (tp_size_ > 1) {
    // expert parallel: fp32 sum over THIS rank's experts, then the row-parallel exchange sums the ranks,
    // rounds once, adds the residual and normalises (same contract as the dense down projection)
    PROF("moe_combine", launch_moe_combine(ye_, moe_row_of_, moe_topk_w_, c.hidden, T, ar_buf_, true, stream_));
    ++launches_;
    if (have_peers_) {
      const int epoch = tp_epoch_ + 1;
      tp_epoch_ += 2;
      PROF("moe_p2p_allreduce_norm", launch_tp_reduce_norm(peers_, T, c.hidden, gain, c.eps, epoch, tp_flags_ + TP_MAX, last_layer, stream_));
      ++launches_;
    } else {
      const NcclApi& nc = nccl_api();
      int rc = nc.AllReduce(ar_buf_, ar_buf_, (size_t)T * c.hidden, kNcclFloat32, kNcclSum, comm_, stream_);
      if (rc != 0) { fprintf(stderr, "[acp_infer] ncclAllReduce: %s\n", nc.GetErrorString(rc)); return -5; }
      GemmOut o;
      o.ptr = ar_buf_; o.splits = 1; o.n_cap = T; o.ld = c.hidden;
      PROF("add_rmsnorm_moe", launch_add_rmsnorm(x_, o, gain, xn_, nullptr, T, c.hidden, c.eps, stream_));
      launches_ += 2;
    }
    return 0;
  }
  PROF("moe_combine", launch_moe_combine(ye_, moe_row_of_, moe_topk_w_, c.hidden, T, gemm_bf16_, false, stream_));
  GemmOut o;
  o.ptr = gemm_bf16_; o.splits = 0; o.n_cap = T; o.ld = c.hidden;
  PROF("add_rmsnorm_moe", launch_add_rmsnorm(x_, o, gain, xn_, nullptr, T, c.hidden, c.eps, stream_));
  launches_ += 2;
  return 0;
}

int Model::sync() {
  cudaError_t e = cudaStreamSynchronize(stream_);
  if (e != cudaSuccess) {
    fprintf(stderr, "[acp_infer] step failed: %s\n", cudaGetErrorString(e));
    return -5;
  }
  if (profile_enabled()) prof_collect(stage_.decode);
  return 0;
}

}  // namespace acp
