// kernels.cuh — host launchers of the HBM-bound (non-GEMM) kernels of the decode engine.
// Every kernel that consumes a GEMM result accepts it either as bf16 [T][M] (prefill, split-K off)
// or as `splits` fp32 partial planes [splits][n_cap][M] which it sums in index order before the
// bf16 rounding — the deterministic split-K reduction (see gemm_wgmma.cuh).
#pragma once
#include "grammar.h"
#include "model_config.h"
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>

namespace acp {

// A GEMM result as seen by its consumer.
struct GemmOut {
  const void* ptr = nullptr;  // bf16* when splits == 0, else float* partial planes
  int splits = 0;             // 0 => bf16 [T][ld]; >=1 => fp32 [splits][n_cap][ld]
  int n_cap = 0;
  int ld = 0;
};

// x[t][:] = E[tok[t]][:]
int launch_embed(const int* tok, const __nv_bfloat16* E, __nv_bfloat16* x, int T, int hidden,
                 cudaStream_t s);

// (optional) x = bf16(x + bf16(gemm_out)); xn[i] = bf16(g * bf16(x[row] * rstd)).
// row_map == nullptr: row i <- i for i < T, residual x is updated in place.
// row_map != nullptr: output row i is computed from source row row_map[i] (i < T outputs); the
//                     residual is NOT written back (used for the final norm on sampled rows).
int launch_add_rmsnorm(__nv_bfloat16* x, const GemmOut& add, const __nv_bfloat16* gain,
                       __nv_bfloat16* xn, const int* row_map, int T, int hidden, float eps,
                       cudaStream_t s);

// RoPE (rotate-half, table driven) on q and k, then scatter k,v into the paged KV cache and q
// into qbuf.  qkv row layout: [q_dim | kv_dim (k) | kv_dim (v)].
struct RopeKvArgs {
  GemmOut qkv;
  const int* pos;        // [T] absolute position of each row
  const int* seq_of_row; // [T] sequence of each row
  const int* page_table; // packed: pages of sequence b are page_table[page_off[b] .. page_off[b+1])
  const int* page_off;   // [num_seqs+1]
  const float* cos_tab;  // [max_pos][64]
  const float* sin_tab;
  __nv_bfloat16* qbuf;   // [T][q_dim]
  __nv_bfloat16* k_cache;  // layer base: [num_pages][kv_heads][2 dim-halves][KV_PAGE][64]
  __nv_bfloat16* v_cache;
  int T, heads, kv_heads;
};
int launch_rope_kv(const RopeKvArgs& a, cudaStream_t s);

// h[t][j] = bf16( bf16(silu(g)) * u ), g = gu[t][2j], u = gu[t][2j+1]  (interleaved gate/up columns)
int launch_swiglu(const GemmOut& gu, __nv_bfloat16* h, int T, int ffn, cudaStream_t s);

// token[n] = argmax over m-tiles of the fused GEMM arg-max epilogue (lowest index on ties)
int launch_argmax_finish(const float* tile_val, const int* tile_idx, int m_tiles, int N,
                         int* token_out, float* val_out, cudaStream_t s);

// Non-greedy sampling on fp32 logits [N][V]: temperature, top-k, top-p, deterministic counter RNG.
struct SampleParams {  // per row
  float temperature;   // <= 0 => greedy
  int top_k;           // <= 0 => off
  float top_p;         // >= 1 => off
  uint64_t seed;       // request seed
  uint32_t step;       // decode step index (RNG counter)
};
int launch_sample(const float* logits, int V, int N, const SampleParams* params_dev,
                  int* token_out, cudaStream_t s);

// Constrained decoding (grammar.cu): logits[rows[r].row][id] = -inf for every id the grammar rejects from
// rows[r].state, name tables indexed by rows[r].slot; one grid row per constrained row (ld = row stride).
int launch_grammar_mask(float* logits, int ld, const GrammarVocab& v, const GrammarRow* rows_dev, int n_rows,
                        const GrammarNames* tables_dev, cudaStream_t s);

// Seeded synthetic tensor (values bit-identical to oracle/synth.py).  SynthMap says where the
// LOCAL tensor (a tensor-parallel shard, stored as contiguous 128x64 tiles, optionally with
// gate/up rows interleaved) sits inside the LOGICAL row-major tensor of the oracle.
struct SynthMap {
  int local_cols = 1;       // K of the local tensor; 1 = flat vector (no tiling)
  int logical_cols = 1;     // row length of the logical tensor
  int col0 = 0;             // first logical column held by this shard
  int interleave_half = 0;  // > 0: local row 2j -> seg_global[0] + j, 2j+1 -> seg_global[1] + j
  int nseg = 1;             // otherwise: consecutive local row ranges
  int seg_rows[3] = {0x7fffffff, 0, 0};
  int seg_global[3] = {0, 0, 0};
};
int launch_synth(__nv_bfloat16* out, size_t n, uint64_t seed, uint32_t tid, double std,
                 int plus_one, cudaStream_t s, const SynthMap& map = SynthMap());

// out[i] = src[logical_index(i) - src_elem0]: places a row-major checkpoint tensor (staged on the
// device) into the tiled / interleaved / sharded weight layout described by `map`
int launch_gather_weight(__nv_bfloat16* out, size_t n, const __nv_bfloat16* src, size_t src_elem0,
                         cudaStream_t s, const SynthMap& map);

// FP8 checkpoints: row-major e4m3 codes `src` ([logical rows][logical_cols], the whole logical tensor) into the
// 128 x 128-code tiles of `map`, and the fp32 scale of each of the `rows` local rows from s_src[logical row]
int launch_gather_weight_e4m3(uint8_t* out, size_t n, const uint8_t* src, float* s_out, int rows, const float* s_src,
                              cudaStream_t s, const SynthMap& map);

// out[i] = sum_s planes[s][i] (index order), fp32 -> fp32: local split-K reduction in front of a
// tensor-parallel all-reduce
int launch_reduce_planes(const float* planes, int splits, size_t plane_elems, float* out, cudaStream_t s);

// Tensor-parallel arg-max: gathered[P][2][B] (per rank: B fp32 maxima then B int32 global ids)
// -> token[B], lowest id wins ties.
int launch_repack_logits(const float* gathered, int P, int n, int rows_per_rank, int vocab, float* out, cudaStream_t s);
int launch_argmax_ranks(const int* gathered, int P, int B, int* token_out, cudaStream_t s);
// packs (val[B], idx[B] + idx_offset) into out[2][B] words
int launch_pack_candidates(const float* val, const int* idx, int idx_offset, int B, int* out, cudaStream_t s);


}  // namespace acp
