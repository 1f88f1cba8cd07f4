// attention.h — host interface of the paged-KV attention kernels (attention.cu).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include "kernels.cuh"

namespace acp {

// Decode attention.  per_item = 1: one CTA per (sequence, kv head).  Otherwise chunked: one CTA
// per (sequence, kv head, chunk of ATTN_CHUNK_TILES x 64 tokens), then launch_attn_merge.
constexpr int ATTN_CHUNK_TILES = 16;  // 1024 tokens
struct AttnDecodeArgs {
  const __nv_bfloat16* q;   // [B][heads*128] (row b = sequence b)
  __nv_bfloat16* out;       // [B][heads*128]
  const int* ctx_len;       // [B] keys visible to the query of sequence b (incl. its own token)
  const int* chunk_cum;     // [B+1] prefix sum of the per-sequence chunk counts
  const int* page_table;    // packed: pages of sequence b are page_table[page_off[b] .. page_off[b+1])
  const int* page_off;      // [B+1]
  int heads, kv_heads;
  int num_seqs;
  int total_chunks;         // chunk_cum[B]
  int max_chunks;           // workspace stride (chunks per item)
  int per_item;             // 1: whole item per CTA, no workspace / merge
  float scale;              // 1/sqrt(128)
  float* ws;                // partials [(item*max_chunks + chunk)*4 + warp][G rows][130] fp32
  // Fused RoPE + KV append (decode): q/k/v of the NEW token come straight from the QKV GEMM result
  // (split-K planes reduced here), are rotated in the kernel, K/V are appended to the cache by the
  // CTA that owns the sequence's last chunk, and the new token is folded into the softmax from
  // registers.  Replaces the rope_kv kernel on decode steps.
  const void* qkv_ptr;      // GemmOut of the QKV projection: row b = [q heads | k heads | v heads]
  int qkv_splits, qkv_n_cap, qkv_ld;
  const float* cos_tab;     // [max_pos][64]
  const float* sin_tab;
  __nv_bfloat16* k_cache;   // this layer's caches (written)
  __nv_bfloat16* v_cache;
};

struct AttnPrefillArgs {
  const __nv_bfloat16* q;
  __nv_bfloat16* out;
  const int* blk_seq;       // [num_blocks] sequence of each query block
  const int* blk_tok0;      // [num_blocks] first new-token index of the block
  const int* q_start;       // [B] first row of the sequence's new tokens
  const int* q_len;         // [B] number of new tokens
  const int* ctx_len;       // [B] total tokens after this step (cached + new)
  const int* page_table;    // packed, as in AttnDecodeArgs
  const int* page_off;      // [B+1]
  int heads, kv_heads;
  float scale;
};

int attn_setup_attributes();
int attn_make_kv_map(CUtensorMap* out, const void* base, uint64_t num_pages, int kv_heads);
int attn_decode_chunks(int ctx_len);  // chunks of one sequence
size_t attn_decode_ws_floats(int max_batch, int heads, int kv_heads, int max_chunks);
int launch_attn_decode(const CUtensorMap& tm_k, const CUtensorMap& tm_v, const AttnDecodeArgs& a,
                       cudaStream_t s);
// chunked decode only (no-op when per_item): combines the partials launch_attn_decode left in ws
int launch_attn_merge(const AttnDecodeArgs& a, cudaStream_t s);
int attn_prefill_block_tokens(int heads, int kv_heads);
// wgmma prefill attention (attention_prefill_tc.cu): 128 query rows = 128/G tokens x G heads per CTA
int attn_prefill_tc_setup();
int attn_prefill_tc_block_tokens(int heads, int kv_heads);
int attn_make_kv_half_map(CUtensorMap* out, const void* base, uint64_t num_pages, int kv_heads);
int attn_make_q_map(CUtensorMap* out, const void* qbuf, uint64_t rows, int heads, int kv_heads);
int launch_attn_prefill_tc(const CUtensorMap& tm_q, const CUtensorMap& tm_k, const CUtensorMap& tm_v,
                           const AttnPrefillArgs& a, int num_blocks, cudaStream_t s);
bool attn_prefill_tc_enabled();   // ACP_ATTN_PREFILL_TC=0 selects round 1's mma.sync kernel (A/B only)
int launch_attn_prefill(const CUtensorMap& tm_k, const CUtensorMap& tm_v, const AttnPrefillArgs& a,
                        int num_blocks, cudaStream_t s);

}  // namespace acp
