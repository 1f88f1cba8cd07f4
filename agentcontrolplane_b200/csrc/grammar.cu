// grammar.cu — the token mask of constrained tool-call decoding (grammar.h, DESIGN.md §3.3), and its test hooks.
#include <math.h>
#include <string.h>
#include <string>
#include <vector>
#include "acp_infer.h"
#include "acp_infer_kernels.h"
#include "chat.h"
#include "common.cuh"
#include "grammar.h"
#include "kernels.cuh"

namespace acp {

// One thread per vocabulary id, one grid row per constrained logits row: the id's bytes run from the row's
// state through the grammar, and a rejected id's logit becomes -inf.  Rows without a constraint get no CTAs.
__global__ void __launch_bounds__(256)
grammar_mask_kernel(float* __restrict__ logits, int ld, GrammarVocab v, const GrammarRow* __restrict__ rows,
                    const GrammarNames* __restrict__ tables) {
  pdl_launch_dependents();
  pdl_wait();
  const int id = blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= v.vocab) return;
  const GrammarRow r = rows[blockIdx.y];
  if (!grammar_token_allowed(r.state, v, id, tables[r.slot])) logits[(size_t)r.row * ld + id] = -INFINITY;
}

int launch_grammar_mask(float* logits, int ld, const GrammarVocab& v, const GrammarRow* rows_dev, int n_rows,
                        const GrammarNames* tables_dev, cudaStream_t s) {
  if (n_rows <= 0) return 0;
  const dim3 grid((unsigned)((v.vocab + 255) / 256), (unsigned)n_rows);
  cudaError_t e = acp_launch(grammar_mask_kernel, grid, dim3(256), 0, s, logits, ld, v, rows_dev, tables_dev);
  if (e != cudaSuccess) {
    fprintf(stderr, "[acp_infer] launch grammar_mask failed: %s\n", cudaGetErrorString(e));
    return -5;
  }
  return 0;
}

}  // namespace acp

namespace {
bool names_from_json(const char* names_json, acp::GrammarNames* out) {
  acp::Json arr;
  std::string err;
  if (!names_json || !acp::Json::parse(names_json, strlen(names_json), &arr, &err) || !arr.is_array() || arr.size() == 0) return false;
  std::vector<std::string> names;
  for (const acp::Json& n : arr.items()) {
    if (!n.is_string()) return false;
    names.push_back(n.as_string());
  }
  return acp::build_grammar_names(names, out, &err);
}
}  // namespace

extern "C" {

int acp_kernel_grammar_accepts(const char* names_json, int parallel, const uint8_t* text, size_t len, size_t* consumed,
                               int* complete) {
  if (!consumed || !complete || (len && !text)) return ACP_ERR_INVALID;
  try {
    std::unique_ptr<acp::GrammarNames> names(new acp::GrammarNames());
    if (!names_from_json(names_json, names.get())) return ACP_ERR_INVALID;
    acp::GrammarState s;
    acp::grammar_init(&s, names->n, parallel != 0);
    size_t i = 0;
    while (i < len && acp::grammar_step(s, text[i], *names)) ++i;
    *consumed = i;
    *complete = i == len && acp::grammar_accepting(s);
    return ACP_OK;
  } catch (...) { return ACP_ERR_NOMEM; }
}

int acp_kernel_grammar_mask(const char* names_json, int parallel, const uint8_t* prefix, size_t prefix_len,
                            const int32_t* vocab_off, const uint8_t* vocab_bytes, const uint8_t* vocab_stop, int vocab,
                            uint8_t* allowed_bits) {
  if (!vocab_off || !vocab_stop || !allowed_bits || vocab <= 0 || (prefix_len && !prefix)) return ACP_ERR_INVALID;
  std::unique_ptr<acp::GrammarNames> names(new acp::GrammarNames());
  if (!names_from_json(names_json, names.get())) return ACP_ERR_INVALID;
  acp::GrammarRow row;
  row.row = 0;
  row.slot = 0;
  acp::grammar_init(&row.state, names->n, parallel != 0);
  for (size_t i = 0; i < prefix_len; ++i)
    if (!acp::grammar_step(row.state, prefix[i], *names)) return ACP_ERR_INVALID;
  const size_t nbytes = (size_t)vocab_off[vocab];
  int32_t* d_off = nullptr;
  uint8_t *d_bytes = nullptr, *d_stop = nullptr;
  acp::GrammarNames* d_names = nullptr;
  acp::GrammarRow* d_row = nullptr;
  float* d_logits = nullptr;
  int rc = ACP_OK;
  cudaStream_t st = nullptr;
  std::vector<float> logits((size_t)vocab);
  auto ok = [&](cudaError_t e) {
    if (e != cudaSuccess && rc == ACP_OK) { fprintf(stderr, "[acp_infer] grammar_mask hook: %s\n", cudaGetErrorString(e)); rc = ACP_ERR_CUDA; }
    return rc == ACP_OK;
  };
  if (ok(cudaStreamCreate(&st)) && ok(cudaMalloc(&d_off, ((size_t)vocab + 1) * sizeof(int32_t))) &&
      ok(cudaMalloc(&d_bytes, nbytes ? nbytes : 1)) && ok(cudaMalloc(&d_stop, (size_t)vocab)) &&
      ok(cudaMalloc(&d_names, sizeof(acp::GrammarNames))) && ok(cudaMalloc(&d_row, sizeof row)) &&
      ok(cudaMalloc(&d_logits, (size_t)vocab * sizeof(float))) &&
      ok(cudaMemcpy(d_off, vocab_off, ((size_t)vocab + 1) * sizeof(int32_t), cudaMemcpyHostToDevice)) &&
      ok(nbytes ? cudaMemcpy(d_bytes, vocab_bytes, nbytes, cudaMemcpyHostToDevice) : cudaSuccess) &&
      ok(cudaMemcpy(d_stop, vocab_stop, (size_t)vocab, cudaMemcpyHostToDevice)) &&
      ok(cudaMemcpy(d_names, names.get(), sizeof(acp::GrammarNames), cudaMemcpyHostToDevice)) &&
      ok(cudaMemcpy(d_row, &row, sizeof row, cudaMemcpyHostToDevice)) &&
      ok(cudaMemset(d_logits, 0, (size_t)vocab * sizeof(float)))) {
    acp::GrammarVocab v;
    v.vocab = vocab; v.off = d_off; v.bytes = d_bytes; v.stop = d_stop;
    if (acp::launch_grammar_mask(d_logits, vocab, v, d_row, 1, d_names, st) != 0) rc = ACP_ERR_CUDA;
    if (ok(cudaStreamSynchronize(st)) &&
        ok(cudaMemcpy(logits.data(), d_logits, (size_t)vocab * sizeof(float), cudaMemcpyDeviceToHost))) {
      memset(allowed_bits, 0, ((size_t)vocab + 7) / 8);
      for (int i = 0; i < vocab; ++i)
        if (logits[(size_t)i] == 0.f) allowed_bits[i >> 3] |= (uint8_t)(1u << (i & 7));
    }
  }
  cudaFree(d_off); cudaFree(d_bytes); cudaFree(d_stop); cudaFree(d_names); cudaFree(d_row); cudaFree(d_logits);
  if (st) cudaStreamDestroy(st);
  return rc;
}

}  // extern "C"
