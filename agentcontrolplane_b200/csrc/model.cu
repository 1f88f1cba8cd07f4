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
#include "fp8.h"
#include <math.h>
#include <algorithm>
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
  if (h_grows_) cudaFreeHost(h_grows_);
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
// FP8 GEMMs count k-blocks of 128 e4m3 elements (splitk_factor_fp8).  Still a function of (M, K) alone for one
// N tile, so batch invariance holds under FP8 too.
int Model::choose_splits(int M, int K, int N) const {
  if (cfg_.fp8) return splitk_factor_fp8(M, K, N, lim_.splitk_target_ctas, lim_.strict_batch_invariance);
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
  if (cfg.fp8 && (tp_size > 1 || cfg.experts > 0 || cfg.hidden % 128 || cfg.ffn % 128)) {
    fprintf(stderr, "[acp_infer] fp8 projections need a dense model on one GPU with hidden and ffn multiples of 128\n");
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
  env = getenv("ACP_TP_SYNC_EVERY");
  tp_sync_every_ = (env && tp_size > 1) ? atoi(env) : 0;
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

// Where this shard's weights sit in the logical tensors that oracle/synth.py generates and a checkpoint
// stores: the only place the projection, LM head and expert layouts are written.  The generator and the
// loader both place weights through these maps.
void Model::describe_weights() {
  const ModelConfig& c = cfg_;
  const int H = c.hidden, r = tp_rank_;
  // gate/up rows interleaved (2j = gate_j, 2j+1 = up_j), from row `row0` of each half of the logical [gate; up]
  auto gate_up = [&](int half, int row0) {
    SynthMap m{H, H, 0, half};
    m.seg_global[0] = row0;
    m.seg_global[1] = c.ffn + row0;
    return m;
  };
  SynthMap qkv{H, H, 0};   // [q heads of this rank | k heads | v heads] rows of the logical [q; k; v]
  qkv.nseg = 3;
  qkv.seg_rows[0] = qdim_l_; qkv.seg_global[0] = r * qdim_l_;
  qkv.seg_rows[1] = kvdim_l_; qkv.seg_global[1] = c.q_dim() + r * kvdim_l_;
  qkv.seg_rows[2] = kvdim_l_; qkv.seg_global[2] = c.q_dim() + c.kv_dim() + r * kvdim_l_;
  for (Layer& L : layers_) {
    L.qkv = Proj{qkv_l_, H, qkv, 0, {{"self_attn.q_proj", c.q_dim()}, {"self_attn.k_proj", c.kv_dim()}, {"self_attn.v_proj", c.kv_dim()}}};
    L.o = Proj{H, qdim_l_, SynthMap{qdim_l_, c.q_dim(), r * qdim_l_}, 1, {{"self_attn.o_proj", H}}};
    if (c.experts > 0) continue;
    L.gu = Proj{2 * ffn_l_, H, gate_up(ffn_l_, r * ffn_l_), 2, {{"mlp.gate_proj", c.ffn}, {"mlp.up_proj", c.ffn}}};
    L.down = Proj{H, ffn_l_, SynthMap{ffn_l_, c.ffn, r * ffn_l_}, 3, {{"mlp.down_proj", H}}};
  }
  lm_map_ = SynthMap{H, H, 0};   // this shard's rows, contiguous in the logical tensor
  lm_map_.nseg = 1; lm_map_.seg_rows[0] = lm_rows_l_; lm_map_.seg_global[0] = lm_row0_;
  gu_e_map_ = gate_up(c.ffn, 0);   // whole experts
  down_e_map_ = SynthMap{c.ffn, c.ffn, 0};
}

// Allocates and maps p: bf16 tiles, or e4m3 tiles and row scales under cfg.fp8.  Grows the split-K workspace
// to what p's decode GEMMs need at any step height (the split factor depends on it beyond 256 rows, model_config.cc).
int Model::alloc_proj(Proj& p) {
  const ModelLimits& m = lim_;
  if (cfg_.fp8) {
    ws_bytes_ = std::max(ws_bytes_, splitk_workspace_bytes_fp8(p.M, p.K, m.max_batch, m.splitk_target_ctas, m.strict_batch_invariance));
    ACP_TRY(dmalloc_t(allocs_, &p.codes, (size_t)p.M * p.K));
    ACP_TRY(dmalloc_t(allocs_, &p.scale, (size_t)p.M));
    return tma_make_weight_e4m3(&p.m, p.codes, p.M, p.K);
  }
  ws_bytes_ = std::max(ws_bytes_, splitk_workspace_bytes(p.M, p.K, m.max_batch, m.splitk_target_ctas, m.strict_batch_invariance));
  ACP_TRY(dmalloc_t(allocs_, &p.w, (size_t)p.M * p.K));
  return tma_make_weight(&p.m, p.w, p.M, p.K);
}

// Allocates (zeroed) an activation, and under cfg.fp8 its e4m3 copy and row scales; maps the one GEMMs read
int Model::alloc_act(Act& a, int rows, int cols, const char* quant) {
  a.quant = quant;
  ACP_TRY(dmalloc_t(allocs_, &a.x, (size_t)rows * cols, true));
  if (!cfg_.fp8) return tma_make_act(&a.m, a.x, rows, cols);
  ACP_TRY(dmalloc_t(allocs_, &a.x8, (size_t)rows * cols, true));
  ACP_TRY(dmalloc_t(allocs_, &a.scale, (size_t)rows, true));
  return tma_make_act_e4m3(&a.m, a.x8, rows, cols);
}

int Model::alloc_all() {
  const ModelConfig& c = cfg_;
  const size_t H = c.hidden;
  const int T = ((lim_.max_tokens + 255) / 256) * 256;
  const int Bp = ((lim_.max_batch + 255) / 256) * 256;
  layers_.resize(c.layers);
  describe_weights();
  const size_t kv_elems = (size_t)lim_.num_pages * kvh_l_ * KV_PAGE * HEAD_DIM;
  for (Layer& L : layers_) {
    for (Proj* p : L.projs()) ACP_TRY(alloc_proj(*p));
    if (c.experts > 0) {
      ACP_TRY(dmalloc_t(allocs_, &L.router, (size_t)c.experts * H));
      ACP_TRY(dmalloc_t(allocs_, &L.wgu_e, (size_t)experts_l_ * 2 * c.ffn * H));
      ACP_TRY(dmalloc_t(allocs_, &L.wdown_e, (size_t)experts_l_ * H * c.ffn));
      ACP_TRY(tma_make_weight(&L.m_gu_e, L.wgu_e, (uint64_t)experts_l_ * 2 * c.ffn, H));
      ACP_TRY(tma_make_weight(&L.m_down_e, L.wdown_e, (uint64_t)experts_l_ * H, c.ffn));
    }
    ACP_TRY(dmalloc_t(allocs_, &L.attn_norm, H));
    ACP_TRY(dmalloc_t(allocs_, &L.ffn_norm, H));
    ACP_TRY(dmalloc_t(allocs_, &L.k_cache, kv_elems, true));
    ACP_TRY(dmalloc_t(allocs_, &L.v_cache, kv_elems, true));
    ACP_TRY(attn_make_kv_map(&L.tm_k, L.k_cache, lim_.num_pages, kvh_l_));
    ACP_TRY(attn_make_kv_map(&L.tm_v, L.v_cache, lim_.num_pages, kvh_l_));
    ACP_TRY(attn_make_kv_half_map(&L.tm_k32, L.k_cache, lim_.num_pages, kvh_l_));
    ACP_TRY(attn_make_kv_half_map(&L.tm_v32, L.v_cache, lim_.num_pages, kvh_l_));
  }
  ACP_TRY(dmalloc_t(allocs_, &embed_, (size_t)c.vocab * H));
  ACP_TRY(dmalloc_t(allocs_, &lm_head_, (size_t)lm_rows_l_ * H));
  ACP_TRY(dmalloc_t(allocs_, &final_norm_, H));
  ACP_TRY(tma_make_weight(&m_lm_, lm_head_, lm_rows_l_, H));
  ACP_TRY(dmalloc_t(allocs_, &cos_, (size_t)rope_rows() * 64));
  ACP_TRY(dmalloc_t(allocs_, &sin_, (size_t)rope_rows() * 64));
  // activations (rows padded to the largest N tile, zero initialised)
  ACP_TRY(dmalloc_t(allocs_, &x_, (size_t)T * H, true));
  ACP_TRY(alloc_act(xn_, T, c.hidden, "quant_xn"));
  ACP_TRY(dmalloc_t(allocs_, &qbuf_, (size_t)T * qdim_l_, true));
  ACP_TRY(alloc_act(attn_, T, qdim_l_, "quant_attn"));
  if (c.experts == 0) ACP_TRY(alloc_act(h_, T, ffn_l_, "quant_h"));
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
  size_t max_m = H;   // gemm_bf16_: the output of one dense GEMM or of the expert combine
  for (const Proj* p : layers_[0].projs()) max_m = std::max(max_m, (size_t)p->M);
  ACP_TRY(dmalloc_t(allocs_, &gemm_bf16_, (size_t)T * max_m, true));
  ACP_TRY(attn_make_q_map(&tm_q_, qbuf_, (uint64_t)T, heads_l_, kvh_l_));
  ACP_TRY(tma_make_act(&m_xs_, xs_, Bp, H));
  // split-K workspace: alloc_proj sized it for the dense decode GEMMs (the expert GEMMs are grouped, never split-K)
  if (tp_size_ > 1) {  // row-parallel GEMMs write fp32 (one rounding after the all-reduce), prefill too
    ws_bytes_ = std::max(ws_bytes_, (size_t)T * H * sizeof(float));
    ACP_TRY(dmalloc_t(allocs_, &ar_buf_, (size_t)T * H));
    ACP_TRY(dmalloc_t(allocs_, &cand_local_, (size_t)2 * Bp));
    ACP_TRY(dmalloc_t(allocs_, &cand_all_, (size_t)2 * Bp * tp_size_));
    ACP_TRY(dmalloc_t(allocs_, &amax_val_row_, (size_t)Bp));
    ACP_TRY(dmalloc_t(allocs_, &tp_flags_, (size_t)TP_MAX + 8, true));  // [0..7] flags, [8] done counter
  }
  ACP_TRY(dmalloc(allocs_, (void**)&ws_, ws_bytes_));
  const int m_tiles_lm = (lm_rows_l_ + GEMM_BM - 1) / GEMM_BM;
  ACP_TRY(dmalloc_t(allocs_, &amax_val_, (size_t)Bp * m_tiles_lm));
  ACP_TRY(dmalloc_t(allocs_, &amax_idx_, (size_t)Bp * m_tiles_lm));
  ACP_TRY(dmalloc_t(allocs_, &logits_, (size_t)lim_.max_batch * lm_rows_per_rank_));
  if (tp_size_ > 1) {
    ACP_TRY(dmalloc_t(allocs_, &logits_gather_, (size_t)tp_size_ * lim_.max_batch * lm_rows_per_rank_));
    ACP_TRY(dmalloc_t(allocs_, &logits_full_, (size_t)lim_.max_batch * cfg_.vocab));
  }
  // decode attention partials: every sequence may be at max_pages_per_seq pages in one step (prefix sharing lets
  // many sequences map one long prefix), so the workspace covers max_batch x the longest context (DESIGN.md §2)
  attn_max_chunks_ = attn_decode_chunks(lim_.max_pages_per_seq * KV_PAGE);
  const size_t attn_ws_floats = attn_decode_ws_floats(lim_.max_batch, heads_l_, kvh_l_, attn_max_chunks_);
  {
    size_t free_b = 0, total_b = 0;
    ACP_CUDA_CHECK(cudaMemGetInfo(&free_b, &total_b));
    if (attn_ws_floats * sizeof(float) > free_b) {
      fprintf(stderr,
              "[acp_infer] the decode attention workspace needs %.2f GiB (max_batch %d x %d KV heads x %d chunks of 1024 "
              "tokens at max_pages_per_seq %d) but only %.2f GiB are free beside the weights and the KV pool of %d pages: "
              "lower max_batch, max_pages_per_seq or kv_pages\n",
              attn_ws_floats * 4.0 / (1 << 30), lim_.max_batch, kvh_l_, attn_max_chunks_, lim_.max_pages_per_seq,
              free_b / (double)(1 << 30), lim_.num_pages);
      return -4;
    }
  }
  ACP_TRY(dmalloc_t(allocs_, &attn_ws_, attn_ws_floats));
  // step staging: the arrays of stage_begin, the packed page list forward() uploads, the engine's page table
  ints_cap_ = (size_t)5 * lim_.max_tokens + (size_t)7 * lim_.max_batch +
              (size_t)2 * lim_.max_batch * lim_.max_pages_per_seq + 72;
  ACP_TRY(dmalloc_t(allocs_, &d_ints_, ints_cap_));
  ACP_CUDA_CHECK(cudaMallocHost((void**)&h_ints_, ints_cap_ * sizeof(int)));
  ACP_TRY(dmalloc_t(allocs_, &d_sparams_, (size_t)lim_.max_batch));
  ACP_CUDA_CHECK(cudaMallocHost((void**)&h_sparams_, lim_.max_batch * sizeof(SampleParams)));
  ACP_TRY(dmalloc_t(allocs_, &d_tokens_, (size_t)lim_.max_batch));
  ACP_CUDA_CHECK(cudaMallocHost((void**)&h_tokens_, lim_.max_batch * sizeof(int)));
  ACP_CUDA_CHECK(cudaMallocHost((void**)&h_logits_, (size_t)lim_.max_batch * (tp_rank_ == 0 ? cfg_.vocab : GEMM_BM) * sizeof(float)));
  if (lim_.grammar_vocab && tp_size_ == 1) {   // constrained decoding: vocabulary bytes, name-table slots, row states
    const GrammarVocab& v = *lim_.grammar_vocab;
    if (v.vocab != cfg_.vocab) { fprintf(stderr, "[acp_infer] grammar vocabulary has %d ids, the model %d\n", v.vocab, cfg_.vocab); return -1; }
    int32_t* off = nullptr;
    uint8_t *bytes = nullptr, *stop = nullptr;
    ACP_TRY(dmalloc_t(allocs_, &off, (size_t)v.vocab + 1));
    ACP_TRY(dmalloc_t(allocs_, &bytes, (size_t)v.off[v.vocab]));
    ACP_TRY(dmalloc_t(allocs_, &stop, (size_t)v.vocab));
    ACP_CUDA_CHECK(cudaMemcpy(off, v.off, ((size_t)v.vocab + 1) * sizeof(int32_t), cudaMemcpyHostToDevice));
    ACP_CUDA_CHECK(cudaMemcpy(bytes, v.bytes, (size_t)v.off[v.vocab], cudaMemcpyHostToDevice));
    ACP_CUDA_CHECK(cudaMemcpy(stop, v.stop, (size_t)v.vocab, cudaMemcpyHostToDevice));
    gvocab_.vocab = v.vocab; gvocab_.off = off; gvocab_.bytes = bytes; gvocab_.stop = stop;
    ACP_TRY(dmalloc_t(allocs_, &d_gnames_, (size_t)lim_.max_batch));
    ACP_TRY(dmalloc_t(allocs_, &d_grows_, (size_t)lim_.max_batch));
    ACP_CUDA_CHECK(cudaMallocHost((void**)&h_grows_, lim_.max_batch * sizeof(GrammarRow)));
  }
  return 0;
}

int Model::gen_weights() {
  const ModelConfig& c = cfg_;
  const size_t H = c.hidden;
  // tensor ids shared with oracle/synth.py
  ACP_TRY(launch_synth(embed_, (size_t)c.vocab * H, c.seed, 1, c.w_std, 0, stream_));  // replicated, row-major
  ACP_TRY(launch_synth(lm_head_, (size_t)lm_rows_l_ * H, c.seed, 2, c.w_std, 0, stream_, lm_map_));
  ACP_TRY(launch_synth(final_norm_, H, c.seed, 3, 0.1, 1, stream_));
  // FP8 presets: each projection is generated in bf16 into one staging buffer, quantised row by row into its
  // e4m3 tiles + scales, and the staging buffer is freed at the end
  __nv_bfloat16* stage = nullptr;
  if (c.fp8) {
    size_t n = 0;
    for (const Proj* p : layers_[0].projs()) n = std::max(n, (size_t)p->M * p->K);
    ACP_CUDA_CHECK(cudaMalloc((void**)&stage, n * sizeof(__nv_bfloat16)));
  }
  auto gen_layer = [&](int l) -> int {
    Layer& L = layers_[l];
    const uint32_t base = 16 + (uint32_t)l * 16;
    for (const Proj* p : L.projs()) {
      ACP_TRY(launch_synth(c.fp8 ? stage : p->w, (size_t)p->M * p->K, c.seed, base + p->tid, c.w_std, 0, stream_, p->map));
      if (c.fp8) ACP_TRY(launch_quantize_weight_e4m3(stage, p->M, p->K, p->codes, p->scale, stream_));
    }
    if (c.experts > 0) {
      // tensor ids of oracle/synth.py: router = layer_tid(l, 6); expert e: expert_tid(l, e, 0 = [gate; up] | 1 = down)
      ACP_TRY(launch_synth(L.router, (size_t)c.experts * H, c.seed, base + 6, c.w_std, 0, stream_));
      for (int j = 0; j < experts_l_; ++j) {
        const uint32_t etid = (1u << 20) + (uint32_t)l * 256u + (uint32_t)(expert0_ + j) * 2u;
        ACP_TRY(launch_synth(L.wgu_e + (size_t)j * 2 * c.ffn * H, (size_t)2 * c.ffn * H, c.seed, etid, c.w_std, 0, stream_, gu_e_map_));
        ACP_TRY(launch_synth(L.wdown_e + (size_t)j * H * c.ffn, H * c.ffn, c.seed, etid + 1, c.w_std, 0, stream_, down_e_map_));
      }
    }
    ACP_TRY(launch_synth(L.attn_norm, H, c.seed, base + 4, 0.1, 1, stream_));
    ACP_TRY(launch_synth(L.ffn_norm, H, c.seed, base + 5, 0.1, 1, stream_));
    return 0;
  };
  int rc = 0;
  for (int l = 0; l < c.layers && rc == 0; ++l)
    rc = gen_layer(l);
  if (stage) {
    ACP_CUDA_CHECK(cudaStreamSynchronize(stream_));
    cudaFree(stage);
  }
  return rc;
}

// RoPE tables: same recipe as oracle/llama_oracle.py rope_tables(), one row per position the engine can serve
int Model::build_rope_tables() {
  const ModelConfig& c = cfg_;
  const int rows = rope_rows();
  std::vector<float> hc((size_t)rows * 64), hs((size_t)rows * 64);
  float inv[64];
  rope_inv_freq(c, inv);
  for (int p = 0; p < rows; ++p)
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
  size_t stage_elems = (size_t)lm_rows_l_ * H, scale_rows = 0;
  if (c.experts > 0) stage_elems = std::max(stage_elems, (size_t)2 * c.ffn * H);
  for (const Proj* p : layers_[0].projs()) {
    size_t rows = 0;
    for (const Proj::Part& pt : p->parts) rows += pt.rows;
    stage_elems = std::max(stage_elems, rows * p->map.logical_cols);
    scale_rows = std::max(scale_rows, rows);
  }
  __nv_bfloat16* stage = nullptr;
  float* s_stage = nullptr;   // FP8: the fp32 scale of every logical row
  ACP_CUDA_CHECK(cudaMalloc((void**)&stage, stage_elems * sizeof(__nv_bfloat16)));
  if (c.fp8) ACP_CUDA_CHECK(cudaMalloc((void**)&s_stage, scale_rows * sizeof(float)));
  std::vector<uint16_t> conv;  // host conversion buffer for F16/F32 checkpoints
  std::vector<float> s_host;
  // copies rows [row0, row0+nrows) (default: all) of a [rows][cols] tensor to dst (device, bf16)
  auto upload = [&](const std::string& name, int64_t rows, int64_t cols, __nv_bfloat16* dst, int64_t row0 = 0,
                    int64_t nrows = -1) -> int {
    const StTensor* t = ck.find(name);
    if (!t) { fprintf(stderr, "[acp_infer] checkpoint is missing %s\n", name.c_str()); return -1; }
    const bool shape_ok = cols == 1 ? (t->shape.size() == 1 && t->shape[0] == rows)
                                    : (t->shape.size() == 2 && t->shape[0] == rows && t->shape[1] == cols);
    if (!shape_ok) { fprintf(stderr, "[acp_infer] %s has an unexpected shape\n", name.c_str()); return -1; }
    const size_t e0 = (size_t)row0 * (size_t)cols, n = (size_t)(nrows < 0 ? rows : nrows) * (size_t)cols;
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
        fprintf(stderr, "[acp_infer] %s: dtype %s is not supported (BF16, F16, F32)\n", name.c_str(), t->dtype.c_str());
        return -1;
      }
      ACP_CUDA_CHECK(cudaMemcpyAsync(dst + o, conv.data(), m * 2, cudaMemcpyHostToDevice, stream_));
      ACP_CUDA_CHECK(cudaStreamSynchronize(stream_));
    }
    return 0;
  };
  // FP8 (compressed-tensors float-quantized): the F8_E4M3 codes of `<name>` [rows][cols] to dst (device), used
  // exactly as stored, and its `<name>_scale` (BF16 / F32; [rows, 1] or [rows] per channel, a scalar per tensor,
  // broadcast to every row) widened to fp32 and appended to s_host
  auto upload_e4m3 = [&](const std::string& wn, int64_t rows, int64_t cols, uint8_t* dst) -> int {
    const std::string sn = wn + "_scale";
    const StTensor* t = ck.find(wn);
    const StTensor* ts = ck.find(sn);
    if (!t || !ts) { fprintf(stderr, "[acp_infer] checkpoint is missing %s\n", (!t ? wn : sn).c_str()); return -1; }
    if (t->dtype != "F8_E4M3" || t->shape.size() != 2 || t->shape[0] != rows || t->shape[1] != cols) {
      fprintf(stderr, "[acp_infer] %s: expected F8_E4M3 [%lld, %lld]\n", wn.c_str(), (long long)rows, (long long)cols);
      return -1;
    }
    const int64_t ns = ts->numel();
    const bool per_row = ns == rows && (ts->shape.size() == 1 || (ts->shape.size() == 2 && ts->shape[1] == 1));
    if ((!per_row && ns != 1) || (ts->dtype != "F32" && ts->dtype != "BF16")) {
      fprintf(stderr, "[acp_infer] %s: expected a BF16/F32 scale per output row or per tensor\n", sn.c_str());
      return -1;
    }
    for (int64_t r = 0; r < rows; ++r) {
      const int64_t e = per_row ? r : 0;
      float v;
      if (ts->dtype == "F32") memcpy(&v, ts->data + 4 * e, 4);
      else { uint16_t b; memcpy(&b, ts->data + 2 * e, 2); const uint32_t u = (uint32_t)b << 16; memcpy(&v, &u, 4); }
      s_host.push_back(v);
    }
    ACP_CUDA_CHECK(cudaMemcpyAsync(dst, t->data, t->nbytes, cudaMemcpyHostToDevice, stream_));
    return 0;
  };
  // One projection of the layer with name prefix `pre`: the `<stem>.weight` of every part stacked row-major in
  // `stage` as the logical tensor (bf16, or e4m3 codes + fp32 scales under cfg.fp8), then placed through p.map
  auto load_proj = [&](const Proj& p, const std::string& pre) -> int {
    const int64_t cols = p.map.logical_cols;
    int64_t row0 = 0;
    s_host.clear();
    for (const Proj::Part& pt : p.parts) {
      const std::string wn = pre + pt.stem + ".weight";
      const size_t at = (size_t)row0 * cols;
      ACP_TRY(c.fp8 ? upload_e4m3(wn, pt.rows, cols, (uint8_t*)stage + at) : upload(wn, pt.rows, cols, stage + at));
      row0 += pt.rows;
    }
    if (c.fp8) {
      ACP_CUDA_CHECK(cudaMemcpyAsync(s_stage, s_host.data(), s_host.size() * sizeof(float), cudaMemcpyHostToDevice, stream_));
      ACP_TRY(launch_gather_weight_e4m3(p.codes, (size_t)p.M * p.K, (uint8_t*)stage, p.scale, p.M, s_stage, stream_, p.map));
    } else {
      ACP_TRY(launch_gather_weight(p.w, (size_t)p.M * p.K, stage, 0, stream_, p.map));
    }
    ACP_CUDA_CHECK(cudaStreamSynchronize(stream_));
    return 0;
  };
  auto load_all = [&]() -> int {
    ACP_TRY(upload("model.embed_tokens.weight", c.vocab, H, embed_));
    // LM head: this shard's rows only
    const bool tied = c.tied_embeddings || !ck.find("lm_head.weight");
    ACP_TRY(upload(tied ? "model.embed_tokens.weight" : "lm_head.weight", c.vocab, H, stage, lm_row0_, lm_rows_l_));
    ACP_TRY(launch_gather_weight(lm_head_, (size_t)lm_rows_l_ * H, stage, (size_t)lm_row0_ * H, stream_, lm_map_));
    ACP_CUDA_CHECK(cudaStreamSynchronize(stream_));
    ACP_TRY(upload("model.norm.weight", H, 1, final_norm_));
    for (int l = 0; l < c.layers; ++l) {
      Layer& L = layers_[l];
      const std::string pre = "model.layers." + std::to_string(l) + ".";
      for (const Proj* p : L.projs()) ACP_TRY(load_proj(*p, pre));
      if (c.experts > 0) {
        // Mixtral (hub layout): block_sparse_moe.gate.weight [E][H]; experts.<e>.w1 = gate, w3 = up ([ffn][H]), w2 = down ([H][ffn])
        const std::string moe = pre + "block_sparse_moe.";
        ACP_TRY(upload(moe + "gate.weight", c.experts, H, L.router));
        for (int j = 0; j < experts_l_; ++j) {
          const std::string ex = moe + "experts." + std::to_string(expert0_ + j) + ".";
          ACP_TRY(upload(ex + "w1.weight", c.ffn, H, stage));
          ACP_TRY(upload(ex + "w3.weight", c.ffn, H, stage + (size_t)c.ffn * H));
          ACP_TRY(launch_gather_weight(L.wgu_e + (size_t)j * 2 * c.ffn * H, (size_t)2 * c.ffn * H, stage, 0, stream_, gu_e_map_));
          ACP_CUDA_CHECK(cudaStreamSynchronize(stream_));
          ACP_TRY(upload(ex + "w2.weight", H, c.ffn, stage));
          ACP_TRY(launch_gather_weight(L.wdown_e + (size_t)j * H * c.ffn, H * c.ffn, stage, 0, stream_, down_e_map_));
          ACP_CUDA_CHECK(cudaStreamSynchronize(stream_));
        }
      }
      ACP_TRY(upload(pre + "input_layernorm.weight", H, 1, L.attn_norm));
      ACP_TRY(upload(pre + "post_attention_layernorm.weight", H, 1, L.ffn_norm));
    }
    return 0;
  };
  const int rc = load_all();
  cudaFree(stage);
  if (s_stage) cudaFree(s_stage);
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
  s.tile_cum = carve((size_t)B + 1);
  // forward() packs the pages in use here (page offsets [B+1], then the list) and uploads up to their end;
  // the engine's [B][max_pages_per_seq] table after them stays on the host
  pack_at_ = off;
  off += align4((size_t)B + 1) + align4((size_t)B * lim_.max_pages_per_seq);
  s.page_table = carve((size_t)B * lim_.max_pages_per_seq);
  ints_used_ = off;
  s.sample_params = h_sparams_;
  return s;
}

// One launch of p's GEMM over N rows of a into `out` (leading dimension ld)
int Model::launch_proj(const Proj& p, const Act& a, int N, int epi, int splits, void* out, int ld) {
  GemmLaunch g;
  g.tp_shard = tp_size_ > 1;
  g.w = &p.m.w; g.x = &a.m; g.M = p.M; g.N = N; g.K = p.K;
  g.epi = epi; g.splits = splits; g.out = out; g.ld = ld; g.n_cap = N;
  if (cfg_.fp8) { g.fp8 = true; g.w_scale = p.scale; g.x_scale = a.scale; }
  if (out == ws_ && (size_t)splits * N * p.M * sizeof(float) > ws_bytes_) {
    fprintf(stderr, "[acp_infer] split-K workspace too small: %d planes x %d x %d\n", splits, N, p.M);
    return -4;
  }
  ++launches_;
  return gemm_launch(g, stream_);
}

int Model::gemm(const char* name, const Proj& p, const Act& a, int T, bool decode, GemmOut* out, bool swiglu) {
  if (cfg_.fp8) {   // the activation's columns are p's K
    PROF(a.quant, launch_quantize_rows_e4m3(a.x, T, p.K, a.x8, a.scale, stream_));
    ++launches_;
  }
  if (swiglu) {
    PROF(name, launch_proj(p, a, T, EPI_SWIGLU, 1, h_.x, p.M / 2));
    return 0;
  }
  const int splits = choose_splits(p.M, p.K, T);
  const bool planes = decode && splits > 1;   // a single split writes bf16 directly (same rounding, half the bytes)
  *out = planes ? GemmOut{ws_, splits, T, p.M} : GemmOut{gemm_bf16_, 0, T, p.M};
  PROF(name, launch_proj(p, a, T, planes ? EPI_F32 : EPI_BF16, planes ? splits : 1, (void*)out->ptr, p.M));
  return 0;
}

// Row-parallel GEMM of a tensor-parallel shard (O and down projections): fp32 partial sums, local
// split-K reduce, NCCL all-reduce (sum) across the group over NVLink, consumer rounds to bf16 ONCE.
int Model::gemm_rowpar(const Proj& p, const Act& a, int N, bool decode, GemmOut* out) {
  const int M = p.M;
  const int splits = decode ? choose_splits(M, p.K, N) : 1;
  int rc = launch_proj(p, a, N, EPI_F32, splits, ws_, M);
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
int Model::rowpar_fused(const Proj& p, const Act& a, int N, bool decode, const __nv_bfloat16* gain, bool push_x) {
  const int M = p.M;
  const int splits = decode ? choose_splits(M, p.K, N) : 1;
  int rc = launch_proj(p, a, N, EPI_F32, splits, splits > 1 ? ws_ : ar_buf_, M);
  if (rc != 0) return rc;
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
  // every tensor-parallel shard uploads the SAME step descriptor: the lead shard's staging, copied into the shard's
  // own pinned buffer so that each shard packs its page list without touching another's
  const int* src_ints = lead_ ? lead_->h_ints_ : h_ints_;
  const size_t pack_at = lead_ ? lead_->pack_at_ : pack_at_;
  if (lead_) memcpy(h_ints_, src_ints, pack_at * sizeof(int));
  // page list: the ceil(ctx / 32) pages of each sequence, back to back; uploaded bytes follow the pages in use,
  // not max_batch x max_pages_per_seq
  int* h_off = h_ints_ + pack_at;
  int* h_list = h_off + align4((size_t)in.B + 1);
  h_off[0] = 0;
  for (int b = 0; b < in.B; ++b) {
    const int n = (in.ctx_len[b] + KV_PAGE - 1) / KV_PAGE;
    memcpy(h_list + h_off[b], in.page_table + (size_t)b * lim_.max_pages_per_seq, (size_t)n * sizeof(int));
    h_off[b + 1] = h_off[b] + n;
  }
  const size_t used = (size_t)(h_list - h_ints_) + (size_t)h_off[in.B];
  ACP_CUDA_CHECK(cudaMemcpyAsync(d_ints_, h_ints_, used * sizeof(int), cudaMemcpyHostToDevice, stream_));
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
  const int* d_poff = d_ints_ + (h_off - h_ints_);
  const int* d_pt = d_ints_ + (h_list - h_ints_);
  const int T = in.T;
  const float scale = 1.0f / sqrtf((float)HEAD_DIM);

  PROF("embed", launch_embed(d_tok, embed_, x_, T, c.hidden, stream_));
  ++launches_;
  GemmOut none;
  PROF("rmsnorm_first", launch_add_rmsnorm(x_, none, layers_[0].attn_norm, xn_.x, nullptr, T, c.hidden, c.eps, stream_));
  ++launches_;
  for (int l = 0; l < c.layers; ++l) {
    Layer& L = layers_[l];
    GemmOut qkv, o, dn;
    // investigation knob (ACP_TP_SYNC_EVERY): bound this shard's launch queue
    if (tp_sync_every_ > 0 && l > 0 && l % tp_sync_every_ == 0) ACP_CUDA_CHECK(cudaStreamSynchronize(stream_));
    ACP_TRY(gemm("gemm_qkv", L.qkv, xn_, T, in.decode, &qkv));
    if (!in.decode) {
      RopeKvArgs ra;
      ra.qkv = qkv; ra.pos = d_pos; ra.seq_of_row = d_seq; ra.page_table = d_pt;
      ra.page_off = d_poff; ra.cos_tab = cos_; ra.sin_tab = sin_; ra.qbuf = qbuf_;
      ra.k_cache = L.k_cache; ra.v_cache = L.v_cache; ra.T = T; ra.heads = heads_l_; ra.kv_heads = kvh_l_;
      PROF("rope_kv", launch_rope_kv(ra, stream_));
      ++launches_;
    }
    if (in.decode) {
      AttnDecodeArgs aa;
      aa.q = qbuf_; aa.out = attn_.x; aa.ctx_len = d_ctx; aa.chunk_cum = dev(in.tile_cum); aa.page_table = d_pt;
      aa.page_off = d_poff; aa.heads = heads_l_; aa.kv_heads = kvh_l_;
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
      if (!aa.per_item) PROF("attn_merge", launch_attn_merge(aa, stream_));
      launches_ += aa.per_item ? 1 : 2;
    } else {
      AttnPrefillArgs pa;
      pa.q = qbuf_; pa.out = attn_.x; pa.blk_seq = d_bseq; pa.blk_tok0 = d_btok0; pa.q_start = d_qstart;
      pa.q_len = d_qlen; pa.ctx_len = d_ctx; pa.page_table = d_pt; pa.page_off = d_poff;
      pa.heads = heads_l_; pa.kv_heads = kvh_l_; pa.scale = scale;
      if (attn_prefill_tc_enabled()) PROF("attn_prefill", launch_attn_prefill_tc(tm_q_, L.tm_k32, L.tm_v32, pa, in.n_blocks, stream_));
      else PROF("attn_prefill", launch_attn_prefill(L.tm_k, L.tm_v, pa, in.n_blocks, stream_));
      ++launches_;
    }
    if (tp_size_ > 1 && have_peers_) {
      PROF("gemm_o+p2p_allreduce_norm", rowpar_fused(L.o, attn_, T, in.decode, L.ffn_norm, false));
    } else {
      if (tp_size_ > 1) PROF("gemm_o_allreduce", gemm_rowpar(L.o, attn_, T, in.decode, &o));
      else ACP_TRY(gemm("gemm_o", L.o, attn_, T, in.decode, &o));
      PROF("add_rmsnorm_o", launch_add_rmsnorm(x_, o, L.ffn_norm, xn_.x, nullptr, T, c.hidden, c.eps, stream_));
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
    if (!in.decode && T > 256) {
      // prefill: SwiGLU in the persistent gate/up GEMM's epilogue, overlapped with the next tile.  Decode
      // (non-persistent kernel, epilogue exposed at the end of every CTA) measured no gain from fusing.
      ACP_TRY(gemm("gemm_gateup_swiglu", L.gu, xn_, T, in.decode, nullptr, true));
    } else {
      GemmOut gu;
      ACP_TRY(gemm("gemm_gateup", L.gu, xn_, T, in.decode, &gu));
      PROF("swiglu", launch_swiglu(gu, h_.x, T, ffn_l_, stream_));
      ++launches_;
    }
    if (tp_size_ > 1 && have_peers_) {
      // fused exchange writes x_ and xn_ (with the next layer's gain; the last layer's xn_ is unused)
      const __nv_bfloat16* gain = (l + 1 < c.layers) ? layers_[l + 1].attn_norm : final_norm_;
      PROF("gemm_down+p2p_allreduce_norm", rowpar_fused(L.down, h_, T, in.decode, gain, l + 1 == c.layers));
      if (l + 1 == c.layers) {
        GemmOut nothing;
        PROF("add_rmsnorm_final", launch_add_rmsnorm(x_, nothing, final_norm_, xs_, d_srows, in.n_sample, c.hidden, c.eps, stream_));
        ++launches_;
      }
      continue;
    }
    if (tp_size_ > 1) PROF("gemm_down_allreduce", gemm_rowpar(L.down, h_, T, in.decode, &dn));
    else ACP_TRY(gemm("gemm_down", L.down, h_, T, in.decode, &dn));
    if (l + 1 < c.layers) {
      PROF("add_rmsnorm_down", launch_add_rmsnorm(x_, dn, layers_[l + 1].attn_norm, xn_.x, nullptr, T, c.hidden, c.eps, stream_));
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
    const bool constrained = in.n_constrained > 0;
    if (constrained && (!d_grows_ || tp_size_ > 1 || in.n_constrained > in.n_sample)) {
      fprintf(stderr, "[acp_infer] constrained rows on an engine that does not serve them\n");
      return -1;
    }
    const bool logits = in.want_logits || !in.all_greedy || constrained;
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
    } else if (in.all_greedy && !constrained) {
      PROF("argmax_finish", launch_argmax_finish(amax_val_, amax_idx_, m_tiles, in.n_sample, d_tokens_, nullptr, stream_));
    } else {
      if (constrained) {
        // a sequence's name table goes up once, in its first constrained step; then only the row states
        for (int i = 0; i < in.n_name_uploads; ++i) {
          ACP_CUDA_CHECK(cudaMemcpyAsync(d_gnames_ + in.g_upload_slot[i], in.g_upload_names[i], sizeof(GrammarNames),
                                         cudaMemcpyHostToDevice, stream_));
          h2d_bytes_ += (long long)sizeof(GrammarNames);
        }
        memcpy(h_grows_, in.g_rows, (size_t)in.n_constrained * sizeof(GrammarRow));
        ACP_CUDA_CHECK(cudaMemcpyAsync(d_grows_, h_grows_, (size_t)in.n_constrained * sizeof(GrammarRow),
                                       cudaMemcpyHostToDevice, stream_));
        h2d_bytes_ += (long long)(in.n_constrained * sizeof(GrammarRow));
        PROF("grammar_mask", launch_grammar_mask(logits_, lm_rows_per_rank_, gvocab_, d_grows_, in.n_constrained, d_gnames_, stream_));
        ++launches_;
      }
      // greedy rows of this path pick the arg-max path's token (lowest id among the maxima)
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
  PROF("moe_router", launch_moe_router(xn_.x, L.router, c.hidden, c.experts, T, moe_topk_idx_, moe_topk_w_, stream_));
  // N tile of the expert GEMMs: an expert sees about 2T / E rows (a token picks an expert at most once)
  const int bn = gemm_pick_bn((2 * T + c.experts - 1) / c.experts);
  PROF("moe_dispatch", launch_moe_dispatch(moe_topk_idx_, T, expert0_, experts_l_, bn, moe_ranges_, moe_row_of_, stream_));
  PROF("moe_gather", launch_moe_gather(xn_.x, moe_row_of_, c.hidden, T, xe_, stream_));
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
      PROF("add_rmsnorm_moe", launch_add_rmsnorm(x_, o, gain, xn_.x, nullptr, T, c.hidden, c.eps, stream_));
      launches_ += 2;
    }
    return 0;
  }
  PROF("moe_combine", launch_moe_combine(ye_, moe_row_of_, moe_topk_w_, c.hidden, T, gemm_bf16_, false, stream_));
  GemmOut o;
  o.ptr = gemm_bf16_; o.splits = 0; o.n_cap = T; o.ld = c.hidden;
  PROF("add_rmsnorm_moe", launch_add_rmsnorm(x_, o, gain, xn_.x, nullptr, T, c.hidden, c.eps, stream_));
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
