// model.h — Llama-architecture weights, HBM layout and the per-step forward pass of the local
// provider's decode engine.  One Model per GPU (request-level data parallelism = one engine
// replica per GPU, no collective; see DESIGN.md §6).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <algorithm>
#include <string>
#include <vector>
#include "attention.h"
#include "gemm.h"
#include "json.h"
#include "model_config.h"
#include "kernels.cuh"
#include "moe.h"
#include "nccl_dyn.h"
#include "tp_comm.h"

namespace acp {

struct ModelLimits {
  int max_batch = 256;       // sequences per decode step / sampled rows per step
  int max_tokens = 8192;     // token rows per step (prefill chunk budget)
  int num_pages = 2048;      // KV pages (32 tokens each) in the pool, page 0 is reserved
  int max_pages_per_seq = 256;
  int splitk_target_ctas = 222;
  bool strict_batch_invariance = false;   // true: decode steps of > 256 rows keep the one-tile split-K factors
  int attn_decode_mode = 0;  // 0 = auto, 1 = one CTA per (sequence, kv head) when possible, 2 = always chunked + merge
  // constrained tool-call decoding (grammar.h): every id's bytes, read once at init into a device table; null =
  // the engine serves no constrained requests
  const GrammarVocab* grammar_vocab = nullptr;
};

// Host-side description of one engine step (all arrays in pinned host memory, sized by limits).
struct StepInput {
  int T = 0;            // token rows
  int B = 0;            // sequences taking part in this step
  int n_sample = 0;     // rows whose next token is sampled
  int n_blocks = 0;     // prefill query blocks (0 for a pure decode step)
  bool decode = false;  // every sequence has exactly one new token
  bool want_logits = false;
  bool all_greedy = true;
  int max_ctx = 0;
  // packed int32 region, uploaded with one copy:
  int* tok;         // [T]
  int* pos;         // [T]
  int* seq_of_row;  // [T]
  int* q_start;     // [B]
  int* q_len;       // [B]
  int* ctx_len;     // [B]
  int* sample_rows; // [n_sample]
  int* blk_seq;     // [n_blocks]
  int* blk_tok0;    // [n_blocks]
  int* page_table;  // [B][max_pages_per_seq]; entries past a sequence's ceil(ctx_len / 32) pages are not read
  int* tile_cum;    // [B+1] prefix sum of attn_decode_chunks(ctx_len) (decode attention schedule)
  SampleParams* sample_params;  // [n_sample] (pinned, separate upload when !all_greedy)
  // constrained rows (host memory of the caller): their logits are masked by the grammar before sampling
  int n_constrained = 0;
  const GrammarRow* g_rows = nullptr;               // [n_constrained]
  int n_name_uploads = 0;                           // name tables to place before the mask reads them
  const int* g_upload_slot = nullptr;               // [n_name_uploads]
  const GrammarNames* const* g_upload_names = nullptr;
};

class Model {
 public:
  Model() = default;
  ~Model();
  // tp_size > 1: this Model is shard `tp_rank` of a tensor-parallel group (Megatron layout: QKV and
  // gate/up column-parallel, O and down row-parallel + NCCL all-reduce, LM head vocab-parallel);
  // `lead` is shard 0, whose pinned step staging every shard uploads from.
  int init(const ModelConfig& cfg, const ModelLimits& lim, int device, int tp_rank = 0, int tp_size = 1,
           NcclComm comm = nullptr, Model* lead = nullptr, const Checkpoint* ckpt = nullptr);
  // Runs one step on `stream()`: tokens for the n_sample rows land in host_tokens() after sync().
  int forward(const StepInput& in);
  int sync();
  int bench_exchange(int T, int iters, float* avg_us, int diag = 0);  // dev: bare peer-memory exchange, all shards together
  // Carves the pinned staging buffer for a step of T rows, B sequences, n_blocks prefill query
  // blocks; the engine fills the returned arrays, then calls forward(staging()).
  StepInput& stage_begin(int T, int B, int n_blocks);
  StepInput& staging() { return stage_; }
  const int* host_tokens() const { return h_tokens_; }
  const float* host_logits() const { return h_logits_; }  // [n_sample][vocab] when want_logits
  cudaStream_t stream() const { return stream_; }
  const ModelConfig& config() const { return cfg_; }
  const ModelLimits& limits() const { return lim_; }
  int device() const { return device_; }
  long long launches() const { return launches_; }
  long long h2d_bytes() const { return h2d_bytes_; }
  long long d2h_bytes() const { return d2h_bytes_; }
  // ACP_PROFILE=1: CUDA events around every launch of decode steps (breaks PDL overlap; warm caches)
  std::string profile_json();
  // peer-memory exchange (set by the engine once every shard is initialised)
  void set_peers(const TpPeers& p) { peers_ = p; have_peers_ = true; }
  float* ar_buffer() const { return ar_buf_; }
  __nv_bfloat16* x_buffer() const { return x_; }
  __nv_bfloat16* xn_buffer() const { return xn_.x; }
  int* tp_flags() const { return tp_flags_; }

 private:
  int alloc_all();
  int gen_weights();
  int load_weights(const Checkpoint& ck);   // HuggingFace Llama safetensors -> tiled/sharded HBM layout
  int build_rope_tables();
  // positions a sequence can reach: the model's window, or less when max_pages_per_seq caps the context
  int rope_rows() const { return std::min(cfg_.max_pos, lim_.max_pages_per_seq * KV_PAGE); }
  int choose_splits(int M, int K, int N) const;

  ModelConfig cfg_;
  ModelLimits lim_;
  int device_ = 0;
  cudaStream_t stream_ = nullptr;
  long long launches_ = 0, h2d_bytes_ = 0, d2h_bytes_ = 0;
  int tp_sync_every_ = 0;   // ACP_TP_SYNC_EVERY=n (tensor-parallel engines only): stream synchronize every n layers
  // tensor parallel
  int tp_rank_ = 0, tp_size_ = 1;
  NcclComm comm_ = nullptr;
  Model* lead_ = nullptr;
  int heads_l_ = 0, kvh_l_ = 0, qdim_l_ = 0, kvdim_l_ = 0, qkv_l_ = 0, ffn_l_ = 0;
  int lm_rows_l_ = 0, lm_row0_ = 0;
  int lm_rows_per_rank_ = 0;       // rows of the widest vocabulary shard (logits rows are padded to it)
  float* logits_gather_ = nullptr; // [P][max_batch][lm_rows_per_rank_] all-gathered logits (sampling / return_logits under TP)
  float* logits_full_ = nullptr;   // [max_batch][vocab] re-packed on every rank (rank 0 samples / copies out)
  float* ar_buf_ = nullptr;      // [T][hidden] fp32 all-reduce buffer
  int* cand_local_ = nullptr;    // [2][B] packed (max, id)
  int* cand_all_ = nullptr;      // [P][2][B]
  float* amax_val_row_ = nullptr;
  TpPeers peers_;
  bool have_peers_ = false;
  int* tp_flags_ = nullptr;
  int tp_epoch_ = 0;
  // One dense projection of a layer (QKV, O, gate/up, down): this shard's M x K weight, where it sits in the
  // logical tensor that oracle/synth.py generates and a checkpoint stores, and its storage.
  struct Proj {
    struct Part { const char* stem; int rows; };   // checkpoint tensor `<stem>.weight` of the layer
    int M = 0, K = 0;
    SynthMap map;
    uint32_t tid = 0;               // synthetic tensor id: the layer's base + tid
    std::vector<Part> parts;        // stacked row-wise into the logical tensor, e.g. [q; k; v]
    __nv_bfloat16* w = nullptr;     // bf16 tiles
    uint8_t* codes = nullptr;       // cfg.fp8 instead: e4m3 tiles and one fp32 scale per row
    float* scale = nullptr;
    TmaMaps m;
  };
  // An activation a projection reads, [rows][cols] row-major; under cfg.fp8 also its e4m3 copy and per-token scales
  struct Act {
    __nv_bfloat16* x = nullptr;
    uint8_t* x8 = nullptr;
    float* scale = nullptr;
    TmaMaps m;                      // what the GEMM reads: over x, or over x8 under cfg.fp8
    const char* quant = nullptr;    // profile name of its quantiser
  };
  void describe_weights();   // the layout of every projection, the LM head and the experts
  int alloc_proj(Proj& p);
  int alloc_act(Act& a, int rows, int cols, const char* quant);
  int launch_proj(const Proj& p, const Act& a, int N, int epi, int splits, void* out, int ld);
  // `name`: the GEMM's profile segment.  Quantises `a` first under cfg.fp8; swiglu: gate/up into h_
  int gemm(const char* name, const Proj& p, const Act& a, int T, bool decode, GemmOut* out, bool swiglu = false);
  int gemm_rowpar(const Proj& p, const Act& a, int N, bool decode, GemmOut* out);
  int rowpar_fused(const Proj& p, const Act& a, int N, bool decode, const __nv_bfloat16* gain, bool push_x);

  struct Layer {
    Proj qkv, o, gu, down;          // gu, down: dense layers only (M == 0 otherwise)
    std::vector<Proj*> projs() { return gu.M ? std::vector<Proj*>{&qkv, &o, &gu, &down} : std::vector<Proj*>{&qkv, &o}; }
    __nv_bfloat16 *attn_norm, *ffn_norm;
    // mixture of experts (cfg.experts > 0): router [E][hidden] row-major; this rank's experts concatenated,
    // each tiled like the dense matrices: wgu_e [E_l][2 ffn][hidden] (gate/up rows interleaved), wdown_e [E_l][hidden][ffn]
    __nv_bfloat16 *router = nullptr, *wgu_e = nullptr, *wdown_e = nullptr;
    TmaMaps m_gu_e, m_down_e;
    __nv_bfloat16 *k_cache, *v_cache;
    CUtensorMap tm_k, tm_v;       // box = one (page, kv head) block, both dim halves (decode kernels)
    CUtensorMap tm_k32, tm_v32;   // box = one dim half of a page (wgmma prefill kernel)
  };
  std::vector<Layer> layers_;
  __nv_bfloat16 *embed_ = nullptr, *lm_head_ = nullptr, *final_norm_ = nullptr;
  TmaMaps m_lm_;
  SynthMap lm_map_, gu_e_map_, down_e_map_;   // LM head rows of this shard; one expert's [gate; up] and down
  float *cos_ = nullptr, *sin_ = nullptr;
  // activations
  __nv_bfloat16 *x_ = nullptr, *qbuf_ = nullptr, *xs_ = nullptr, *gemm_bf16_ = nullptr;
  Act xn_, attn_, h_;   // h_: dense layers only
  TmaMaps m_xs_;
  CUtensorMap tm_q_;   // qbuf_ as {128 dims, heads, rows} for the prefill attention's Q tiles
  float* ws_ = nullptr;  // split-K partial planes
  size_t ws_bytes_ = 0;
  float *amax_val_ = nullptr, *logits_ = nullptr;
  int* amax_idx_ = nullptr;
  // mixture-of-experts scratch: expert-sorted activations and the routing tables of the current layer
  int experts_l_ = 0, expert0_ = 0;   // experts on this rank (expert parallel = one slice per tensor-parallel rank)
  __nv_bfloat16 *xe_ = nullptr, *he_ = nullptr, *ye_ = nullptr;   // [T][hidden], [T][ffn], [T][hidden] x 2 assignments
  TmaMaps m_xe_, m_he_;
  int *moe_topk_idx_ = nullptr, *moe_row_of_ = nullptr, *moe_ranges_ = nullptr;
  float* moe_topk_w_ = nullptr;
  int moe_mlp(Layer& L, int T, const __nv_bfloat16* gain, bool last_layer);
  float* attn_ws_ = nullptr;
  int attn_max_chunks_ = 1;
  int* d_ints_ = nullptr;     // packed step ints
  size_t ints_cap_ = 0, ints_used_ = 0;   // ints_used_: carved by stage_begin
  size_t pack_at_ = 0;        // where forward() packs the step's page offsets and page list
  int* h_ints_ = nullptr;     // pinned mirror
  SampleParams *d_sparams_ = nullptr, *h_sparams_ = nullptr;
  int *d_tokens_ = nullptr, *h_tokens_ = nullptr;
  float* h_logits_ = nullptr;
  GrammarVocab gvocab_;                 // device copy of lim_.grammar_vocab
  GrammarNames* d_gnames_ = nullptr;    // [max_batch] name tables, indexed by the engine's slot
  GrammarRow *d_grows_ = nullptr, *h_grows_ = nullptr;   // [max_batch] the step's constrained rows
  StepInput stage_;
  std::vector<void*> allocs_;
  // per-kernel profile (ACP_PROFILE=1)
  struct ProfSeg { const char* name; cudaEvent_t a, b; };
  std::vector<ProfSeg> prof_segs_;
  std::vector<cudaEvent_t> prof_pool_;
  size_t prof_used_ = 0;
  struct ProfAcc { long long n = 0; double ms = 0; };
  std::vector<std::pair<std::string, ProfAcc>> prof_acc_[2];  // [0] prefill steps, [1] decode steps
  bool prof_begin(const char* name);
  void prof_end();
  void prof_collect(bool decode);
};

}  // namespace acp
