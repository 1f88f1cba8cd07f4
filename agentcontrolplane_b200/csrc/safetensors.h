// safetensors.h — read-only view of a HuggingFace Llama checkpoint directory: `config.json`,
// `model.safetensors` or `model.safetensors.index.json` + shards (files are mmap'ed; tensors are
// borrowed views).  This is the "real weights" data format on the far side of the hot path: the
// reference delegates the model to a hosted provider (acp/internal/llmclient/langchaingo_client.go:102),
// the local provider has to bring the weights itself (`"weights": "<dir>"` in acp_infer_init).
//
// safetensors file = u64 little-endian header length N, N bytes of JSON
// {"tensor": {"dtype": "BF16", "shape": [r, c], "data_offsets": [begin, end]}, "__metadata__": {...}},
// then the byte buffer the offsets index.
#pragma once
#include <stdint.h>
#include <map>
#include <memory>
#include <string>
#include <vector>
#include "json.h"

namespace acp {

struct StTensor {
  std::string dtype;            // "BF16" | "F16" | "F32" | "F8_E4M3"
  std::vector<int64_t> shape;
  const uint8_t* data = nullptr;
  size_t nbytes = 0;
  int64_t numel() const {
    int64_t n = 1;
    for (int64_t d : shape) n *= d;
    return n;
  }
};

class Checkpoint {
 public:
  Checkpoint() = default;
  ~Checkpoint();
  Checkpoint(const Checkpoint&) = delete;
  Checkpoint& operator=(const Checkpoint&) = delete;

  // `path` = checkpoint directory, or one .safetensors file (config.json is then looked up beside it)
  bool open(const std::string& path, std::string* err);
  const StTensor* find(const std::string& name) const;
  bool has_config() const { return has_config_; }
  const Json& config() const { return config_; }
  const std::string& dir() const { return dir_; }
  size_t tensor_count() const { return tensors_.size(); }
  // {"dir":…, "config":{…}, "tensors":{"name":{"dtype":…,"shape":[…],"nbytes":…}}} (tests, diagnostics)
  std::string index_json() const;

 private:
  struct Mapping { void* base = nullptr; size_t len = 0; };
  bool map_file(const std::string& file, std::string* err);
  std::vector<Mapping> maps_;
  std::map<std::string, StTensor> tensors_;
  Json config_;
  bool has_config_ = false;
  std::string dir_;
};

// Copies `n` elements of a BF16/F16/F32 tensor into bf16 bits (round to nearest even).
bool st_to_bf16(const StTensor& t, size_t elem0, size_t n, uint16_t* out);

}  // namespace acp
