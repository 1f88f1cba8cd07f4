// model_config.h — the architecture description of the served model (pure C++, no CUDA): shared by
// the engine (libacp_infer.so) and by the host-side mirror of the reference (libacp_host.so), which
// only needs it to inspect checkpoints.
#pragma once
#include <stdint.h>
#include <string>
#include "json.h"

namespace acp {

constexpr int KV_PAGE = 32;   // tokens per KV page
constexpr int HEAD_DIM = 128;

struct ModelConfig {
  std::string name = "tiny";
  int hidden = 512, layers = 2, heads = 4, kv_heads = 1, ffn = 1024, vocab = 128256;
  double rope_theta = 500000.0;
  float eps = 1e-5f;
  double w_std = 0.02;
  int max_pos = 8192;
  uint64_t seed = 0xACB200ull;
  int experts = 0;                // Mixtral-style sparse MoE: experts per layer (top-2 routing); 0 = dense MLP
  bool tied_embeddings = false;   // checkpoint without lm_head.weight: LM head = embedding matrix
  // Llama-3.1 "llama3" RoPE frequency scaling (config.json rope_scaling); factor 0 = none
  double rope_factor = 0.0, rope_low_freq = 1.0, rope_high_freq = 4.0;
  int rope_orig_max_pos = 8192;
  // FP8 (e4m3) QKV / O / gate-up / down projections with per-row weight and per-token activation scales
  // (DESIGN.md §5): the `-fp8` presets; dense, single-GPU models only
  bool fp8 = false;
  int q_dim() const { return heads * HEAD_DIM; }
  int kv_dim() const { return kv_heads * HEAD_DIM; }
  int qkv_dim() const { return q_dim() + 2 * kv_dim(); }
  // bytes of weights streamed by one decode step (SURVEY.md §8d "W")
  // (a mixture-of-experts step streams every expert that has a token; with >= 32 sequences and 8 experts
  // that is all of them, so all experts are counted)
  double weight_bytes() const {
    const double mlp = 3.0 * ffn * hidden * (experts > 0 ? experts : 1) + (experts > 0 ? (double)experts * hidden : 0.0);
    double per_layer = (double)qkv_dim() * hidden + (double)hidden * q_dim() + mlp + 2.0 * hidden;
    if (!fp8) return 2.0 * (per_layer * layers + (double)vocab * hidden + hidden);
    // FP8: the four projections at one byte per weight plus one fp32 scale per output row; the rest stays bf16
    const double proj = (double)qkv_dim() * hidden + (double)hidden * q_dim() + 3.0 * ffn * hidden;
    const double rows = (double)qkv_dim() + hidden + 2.0 * ffn + hidden;
    return 2.0 * ((per_layer - proj) * layers + (double)vocab * hidden + hidden) + (proj + 4.0 * rows) * layers;
  }
  double kv_bytes_per_token() const { return 2.0 * kv_dim() * 2.0 * layers; }
  // algorithmic FLOPs of one step (SURVEY.md §8d): 2 per weight per token row for the layer matrices,
  // 2 per LM-head weight per SAMPLED row, and QK^T + PV = 4 * head_dim per (query head, visible key)
  double layer_params() const {   // weights a token row is multiplied with (top-2 of the experts + the router)
    const double mlp = experts > 0 ? 2.0 * 3.0 * ffn * hidden + (double)experts * hidden : 3.0 * ffn * hidden;
    return ((double)qkv_dim() * hidden + (double)hidden * q_dim() + mlp) * layers;
  }
  double step_flops(double token_rows, double sampled_rows, double query_key_pairs) const {
    return 2.0 * layer_params() * token_rows + 2.0 * (double)vocab * hidden * sampled_rows +
           4.0 * q_dim() * query_key_pairs * layers;
  }
};
bool model_preset(const std::string& name, ModelConfig* out);
class Checkpoint;
// ModelConfig from a HuggingFace Llama config.json; false + *err when the architecture is not one
// this engine runs (head_dim must be 128, vocab a multiple of 128, ...).
bool model_config_from_hf(const Json& hf, ModelConfig* out, std::string* err);
// inverse RoPE frequencies [64] as the engine and oracle/llama_oracle.py rope_tables() build them
void rope_inv_freq(const ModelConfig& c, float* inv64);

// Split-K factor of a decode GEMM out[N][M] = X[N][K] W[M][K]^T (pure host logic; the rule and its reasons are
// written out at Model::choose_splits in model.cu).  target_ctas = ModelLimits::splitk_target_ctas.
int splitk_factor(int M, int K, int N, int target_ctas, bool strict_batch_invariance);
// fp32 split-K workspace that holds the planes of ANY decode step of up to max_batch rows of a [M][K] GEMM
size_t splitk_workspace_bytes(int M, int K, int max_batch, int target_ctas, bool strict_batch_invariance);
// The same rule and workspace for the FP8 GEMMs, whose k-blocks hold 128 e4m3 codes (K in elements)
int splitk_factor_fp8(int M, int K, int N, int target_ctas, bool strict_batch_invariance);
size_t splitk_workspace_bytes_fp8(int M, int K, int max_batch, int target_ctas, bool strict_batch_invariance);

}  // namespace acp
