// model_config.cc — see model_config.h.
#include "model_config.h"
#include <math.h>

namespace acp {

bool model_preset(const std::string& name, ModelConfig* c) {
  // "<dense preset>-fp8": the same shapes and seeded weights, projections quantised to e4m3 at init
  const std::string sfx = "-fp8";
  if (name.size() > sfx.size() && name.compare(name.size() - sfx.size(), sfx.size(), sfx) == 0) {
    ModelConfig m;
    if (!model_preset(name.substr(0, name.size() - sfx.size()), &m) || m.fp8 || m.experts > 0 || m.name == "sim" ||
        m.name == "llama-3-70b")
      return false;
    m.name = name;
    m.fp8 = true;
    *c = m;
    return true;
  }
  ModelConfig m;
  m.name = name;
  if (name == "tiny") { m.hidden = 512; m.layers = 2; m.heads = 4; m.kv_heads = 1; m.ffn = 1024; }
  else if (name == "sim") { m.hidden = 512; m.layers = 2; m.heads = 4; m.kv_heads = 1; m.ffn = 1024; }   // scheduler simulations (tests/sanitizers)
  else if (name == "tiny-g2") { m.hidden = 512; m.layers = 3; m.heads = 4; m.kv_heads = 2; m.ffn = 1536; }
  // the head grouping of one Llama-3-70B tensor-parallel shard at TP=8: 8 query heads on 1 KV head
  else if (name == "tiny-g8") { m.hidden = 1024; m.layers = 2; m.heads = 8; m.kv_heads = 1; m.ffn = 2048; }
  else if (name == "llama-3-8b-l2") { m.hidden = 4096; m.layers = 2; m.heads = 32; m.kv_heads = 8; m.ffn = 14336; }
  else if (name == "llama-3-8b") { m.hidden = 4096; m.layers = 32; m.heads = 32; m.kv_heads = 8; m.ffn = 14336; }
  // Mixtral-8x7B architecture (BASELINE config 4).  Synthetic presets keep the 128256-entry vocabulary of
  // the synthetic tokenizer; a real checkpoint brings its own 32000 entries + tokenizer.json.
  else if (name == "tiny-moe") { m.hidden = 512; m.layers = 2; m.heads = 4; m.kv_heads = 2; m.ffn = 768; m.experts = 8; m.rope_theta = 1000000.0; }
  else if (name == "mixtral-8x7b-l2") { m.hidden = 4096; m.layers = 2; m.heads = 32; m.kv_heads = 8; m.ffn = 14336; m.experts = 8; m.rope_theta = 1000000.0; }
  else if (name == "mixtral-8x7b") { m.hidden = 4096; m.layers = 32; m.heads = 32; m.kv_heads = 8; m.ffn = 14336; m.experts = 8; m.rope_theta = 1000000.0; }
  else if (name == "llama-3-70b") { m.hidden = 8192; m.layers = 80; m.heads = 64; m.kv_heads = 8; m.ffn = 28672; }
  // Llama-3.1: the shapes and seeded weights of the Llama-3 preset without the ".1", with the "llama3" RoPE scaling
  // of the published checkpoints and their 131072-token window
  else if (name == "tiny-3.1" || name == "llama-3.1-8b-l2" || name == "llama-3.1-8b") {
    const std::string base = name == "tiny-3.1" ? "tiny" : "llama-3" + name.substr(9);
    if (!model_preset(base, &m)) return false;
    m.name = name;
    m.rope_factor = 8.0; m.rope_low_freq = 1.0; m.rope_high_freq = 4.0; m.rope_orig_max_pos = 8192;
    m.max_pos = 131072;
  }
  else return false;
  *c = m;
  return true;
}

void rope_inv_freq(const ModelConfig& c, float* inv64) {
  const double kTwoPi = 6.283185307179586476925286766559;
  for (int i = 0; i < 64; ++i) {
    double f = pow(c.rope_theta, -(2.0 * i) / (double)HEAD_DIM);
    if (c.rope_factor > 0.0) {  // Llama-3.1 "llama3" scaling: long wavelengths slowed by `factor`
      const double wavelen = kTwoPi / f;
      const double low_wl = (double)c.rope_orig_max_pos / c.rope_low_freq;
      const double high_wl = (double)c.rope_orig_max_pos / c.rope_high_freq;
      if (wavelen > low_wl) {
        f = f / c.rope_factor;
      } else if (!(wavelen < high_wl)) {
        const double smooth = ((double)c.rope_orig_max_pos / wavelen - c.rope_low_freq) / (c.rope_high_freq - c.rope_low_freq);
        f = (1.0 - smooth) * f / c.rope_factor + smooth * f;
      }
    }
    inv64[i] = (float)f;
  }
}

// The one quantization_config this engine serves: compressed-tensors FP8_DYNAMIC (e4m3 weights with a per-channel
// or per-tensor scale, activations quantised per token at run time, lm_head left in bf16).  Anything else is refused
// with the offending field named.
static bool parse_fp8_quantization(const Json& q, std::string* err) {
  auto bad = [&](const std::string& field, const std::string& why) {
    *err = "config.json: quantization_config." + field + " " + why;
    return false;
  };
  const std::string method = q.get("quant_method").as_string();
  if (method != "compressed-tensors") return bad("quant_method", "\"" + method + "\" is not supported (compressed-tensors)");
  if (q.get("format").as_string() != "float-quantized")
    return bad("format", "\"" + q.get("format").as_string() + "\" is not supported (float-quantized)");
  if (!q.get("kv_cache_scheme").is_null()) return bad("kv_cache_scheme", "is not supported (the KV cache stays bf16)");
  const Json& groups = q.get("config_groups");
  if (!groups.is_object() || groups.size() != 1) return bad("config_groups", "must hold exactly one group");
  const std::string gname = groups.members()[0].first;
  const Json& g = groups.members()[0].second;
  const std::string pre = "config_groups." + gname + ".";
  const Json& tg = g.get("targets");
  if (!tg.is_array() || tg.size() != 1 || tg.items()[0].as_string() != "Linear") return bad(pre + "targets", "must be [\"Linear\"]");
  if (!g.get("output_activations").is_null()) return bad(pre + "output_activations", "is not supported");
  auto check = [&](const char* which, const char* strategy, bool dynamic) {
    const Json& a = g.get(which);
    const std::string p = pre + which;
    if (!a.is_object()) return bad(p, "is missing");
    if (a.get("type").as_string() != "float") return bad(p + ".type", "\"" + a.get("type").as_string() + "\" is not supported (float)");
    if (a.get("num_bits").as_int(0) != 8) return bad(p + ".num_bits", "must be 8");
    const std::string st = a.get("strategy").as_string();
    const bool st_ok = std::string(strategy) == "channel" ? (st == "channel" || st == "tensor") : st == strategy;
    if (!st_ok) return bad(p + ".strategy", "\"" + st + "\" is not supported (" + (std::string(strategy) == "channel" ? "channel, tensor" : strategy) + ")");
    if (a.get("dynamic").as_bool(!dynamic) != dynamic) return bad(p + ".dynamic", dynamic ? "must be true" : "must be false");
    if (!a.get("group_size").is_null()) return bad(p + ".group_size", "is not supported");
    if (!a.get("block_structure").is_null()) return bad(p + ".block_structure", "is not supported");
    return true;
  };
  if (!check("weights", "channel", false) || !check("input_activations", "token", true)) return false;
  bool lm_head = false;
  for (const Json& i : q.get("ignore").items()) lm_head |= i.as_string() == "lm_head";
  if (!lm_head) return bad("ignore", "must list lm_head (the LM head stays bf16)");
  return true;
}

bool model_config_from_hf(const Json& hf, ModelConfig* out, std::string* err) {
  ModelConfig m;
  auto need = [&](const char* key, int* v) {
    const Json* j = hf.find(key);
    if (!j || !j->is_number()) { *err = std::string("config.json: missing ") + key; return false; }
    *v = (int)j->as_int();
    return true;
  };
  const std::string mt = hf.get("model_type").as_string();
  if (!mt.empty() && mt != "llama" && mt != "mixtral") { *err = "config.json: model_type \"" + mt + "\" is not supported (llama, mixtral)"; return false; }
  if (mt == "mixtral") {
    m.experts = (int)hf.get("num_local_experts").as_int(8);
    if (hf.get("num_experts_per_tok").as_int(2) != 2 || m.experts < 2 || m.experts > 16) { *err = "config.json: mixtral needs top-2 routing over 2..16 experts"; return false; }
    if (!hf.get("sliding_window").is_null() && hf.get("sliding_window").as_int(0) > 0) { *err = "config.json: sliding-window attention is not supported"; return false; }
  }
  if (!need("hidden_size", &m.hidden) || !need("num_hidden_layers", &m.layers) ||
      !need("num_attention_heads", &m.heads) || !need("intermediate_size", &m.ffn) || !need("vocab_size", &m.vocab))
    return false;
  m.kv_heads = (int)hf.get("num_key_value_heads").as_int(m.heads);
  const int head_dim = (int)hf.get("head_dim").as_int(m.heads > 0 ? m.hidden / m.heads : 0);
  if (head_dim != HEAD_DIM) { *err = "config.json: head_dim " + std::to_string(head_dim) + " (this engine is built for 128)"; return false; }
  if (m.kv_heads <= 0 || m.heads % m.kv_heads || m.heads / m.kv_heads > 16 || 16 % (m.heads / m.kv_heads)) {
    *err = "config.json: unsupported attention head grouping";
    return false;
  }
  if (m.hidden % 128 || m.ffn % 64 || m.vocab % 128) { *err = "config.json: hidden/ffn/vocab must be multiples of 128/64/128"; return false; }
  if (hf.get("attention_bias").as_bool(false) || hf.get("mlp_bias").as_bool(false)) { *err = "config.json: biased projections are not supported"; return false; }
  const std::string act = hf.get("hidden_act").as_string();
  if (!act.empty() && act != "silu") { *err = "config.json: hidden_act must be silu"; return false; }
  m.rope_theta = hf.get("rope_theta").as_double(10000.0);
  m.eps = (float)hf.get("rms_norm_eps").as_double(1e-5);
  m.tied_embeddings = hf.get("tie_word_embeddings").as_bool(false);
  m.max_pos = (int)hf.get("max_position_embeddings").as_int(8192);
  const Json& rs = hf.get("rope_scaling");
  if (rs.is_object()) {
    std::string type = rs.get("rope_type").as_string();
    if (type.empty()) type = rs.get("type").as_string();
    if (type == "llama3") {
      m.rope_factor = rs.get("factor").as_double(8.0);
      m.rope_low_freq = rs.get("low_freq_factor").as_double(1.0);
      m.rope_high_freq = rs.get("high_freq_factor").as_double(4.0);
      m.rope_orig_max_pos = (int)rs.get("original_max_position_embeddings").as_int(8192);
    } else if (!type.empty() && type != "default") {
      *err = "config.json: rope_scaling type \"" + type + "\" is not supported";
      return false;
    }
  }
  const Json& qc = hf.get("quantization_config");
  if (!qc.is_null()) {
    if (!parse_fp8_quantization(qc, err)) return false;
    if (m.experts > 0) { *err = "config.json: quantization_config: FP8 is not supported for mixture-of-experts models"; return false; }
    if (m.hidden % 128 || m.ffn % 128) { *err = "config.json: quantization_config: FP8 needs hidden and intermediate_size multiples of 128"; return false; }
    m.fp8 = true;
  }
  m.name = "checkpoint";
  *out = m;
  return true;
}

int splitk_factor_fp8(int M, int K, int N, int target_ctas, bool strict) {
  // an FP8 k-block holds 128 e4m3 codes in the same 128-byte row as 64 bf16: the rule sees K / 2 columns
  return splitk_factor(M, K / 2, N, target_ctas, strict);
}
size_t splitk_workspace_bytes_fp8(int M, int K, int max_batch, int target_ctas, bool strict) {
  return splitk_workspace_bytes(M, K / 2, max_batch, target_ctas, strict);
}

int splitk_factor(int M, int K, int N, int target_ctas, bool strict) {
  const int m_tiles = (M + 127) / 128;
  const int nkb = (K + 63) / 64;
  const int max_s = nkb / 4 > 0 ? nkb / 4 : 1;  // at least 4 k-blocks per split
  int s;
  if (N > 256 && !strict) {
    // co-resident CTAs share an SM's tensor pipe, so the GEMM's time follows the busiest SM: minimise
    // ceil(tiles * S / SMS) / S (waves of one CTA per SM, each doing 1/S of K); ties -> fewer planes
    constexpr int SMS = 132;   // H100 SXM
    const int tiles = m_tiles * ((N + 255) / 256);
    s = 1;
    // (>= one tile per SM already: no split — the persistent kernel balances those itself, bf16 epilogue)
    if (tiles < SMS) {
      const int cap = max_s < 8 ? max_s : 8;
      double best = 1e30;
      for (int cand = 1; cand <= cap; ++cand) {
        const double cost = (double)((tiles * cand + SMS - 1) / SMS) / cand;
        if (cost < best) best = cost;
      }
      // every extra plane is N x M fp32 written and re-read: take the FEWEST planes within 15 % of the best
      // wave count (128 tiles: 1 plane at cost 1.0, not 8 planes at 0.875; 64 tiles: 2; 96 tiles: 4)
      for (int cand = 1; cand <= cap; ++cand) {
        const double cost = (double)((tiles * cand + SMS - 1) / SMS) / cand;
        if (cost <= best * 1.15 + 1e-9) { s = cand; break; }
      }
    }
  } else {
    s = (target_ctas + m_tiles / 2) / m_tiles;
  }
  if (s < 1) s = 1;
  if (s > max_s) s = max_s;
  if (s > 16) s = 16;
  return s;
}

size_t splitk_workspace_bytes(int M, int K, int max_batch, int target_ctas, bool strict) {
  // the factor depends on the row count beyond 256 rows, and only through ceil(rows / 256): the largest plane set
  // of every 256-row band is at its top
  size_t ws = 0;
  for (int n = 256; n < max_batch + 256; n += 256) {
    const int rows = n < max_batch ? n : max_batch;
    const size_t b = (size_t)splitk_factor(M, K, rows, target_ctas, strict) * rows * M * sizeof(float);
    if (b > ws) ws = b;
  }
  return ws;
}

}  // namespace acp
