/* acp_infer_kernels.h — per-kernel test entry points of libacp_infer.so.
 *
 * These are NOT part of the drop-in boundary (that is include/acp_infer.h).  They exist so the
 * parity tests in tests/ can drive each sm_90a kernel in isolation with HOST buffers (plain
 * pointers and sizes; the library does the cudaMalloc / cudaMemcpy) and compare against the
 * oracle in oracle/.  Every function returns 0 on success or a negative ACP_ERR_* code, never
 * throws, and fails loudly (ACP_ERR_CUDA) when no CUDA device is usable — there is no CPU
 * fallback anywhere in the library.
 */
#ifndef ACP_INFER_KERNELS_H
#define ACP_INFER_KERNELS_H
#include <stddef.h>
#include <stdint.h>
/* a kernel stored past the end of a hook's output, or into a K/V cache slot it does not own */
#define ACP_ERR_GUARD (-8)

#ifdef __cplusplus
extern "C" {
#endif

/* out[n][m] = sum_k w[m][k] * x[n][k]; w,x are bf16 bit patterns.
 * epi 0: out = bf16 [N][M]; epi 1: out = fp32 [splits][N][M] (split-K partial planes);
 * epi 2: amax_val/amax_idx = per-row arg-max over M (lowest index wins ties), out = optional
 * fp32 logits [N][M] (may be NULL); epi 3: rows of w interleaved (gate_j, up_j), out = bf16
 * [N][M/2] = bf16(bf16(silu(g)) * u).  bn = 0 picks the N tile from N; otherwise 16..256;
 * bn = -1 (N > 256, epi 0, 1 or 3) forces the persistent prefill kernel.
 * The output buffer is followed by a guard region; a store past its end returns ACP_ERR_GUARD.
 * iters > 0 additionally times `iters` launches with CUDA events (L2 flushed between
 * launches) and stores the mean milliseconds in *elapsed_ms; iters < 0 is a stress mode: -iters launches back
 * to back (no flush, one synchronize at the end), mean milliseconds in *elapsed_ms. */
/* Which kernel the dispatcher picks for this problem (host logic only, no GPU needed): 0 = tiled
 * gemm_wx_kernel, 1 = persistent kernel.  `splits`, `epi` and `bn` as below. */
int acp_kernel_gemm_path(int M, int N, int K, int splits, int epi, int bn);
/* 2-CTA clusters the persistent prefill GEMM launches (bf16 or FP8 flavour, epilogue epi): what
   cudaOccupancyMaxActiveClusters reports for it on the current device; < 0 on error. */
int acp_kernel_gemm_persistent_clusters(int fp8, int epi);

int acp_kernel_gemm(const uint16_t* w, const uint16_t* x, int M, int N, int K, int splits,
                    int epi, int bn, void* out, float* amax_val, int* amax_idx, int iters,
                    float* elapsed_ms);

/* FP8 (e4m3) GEMM of the `-fp8` presets: w = e4m3 codes [M][K] with fp32 scales w_scale[M], x = e4m3
 * codes [N][K] with fp32 scales x_scale[N]; out[n][m] = fp32(fp32(acc * w_scale[m]) * x_scale[n]) with
 * acc = sum_k w[m][k] * x[n][k] (DESIGN.md §5), then stored as for acp_kernel_gemm: epi 0 bf16 [N][M],
 * epi 1 fp32 [splits][N][M] (each split scaled), epi 3 SwiGLU bf16 [N][M/2] (gate and up rows scaled by
 * their own w_scale before the bf16 rounding).  No arg-max epilogue.  bn = 0 picks the N tile from N;
 * otherwise 16..128; bn = -1 (N > 256, epi 0, 1 or 3) forces the persistent prefill kernel.  iters > 0
 * also stores the mean milliseconds of `iters` launches (L2 flushed between launches) in *elapsed_ms. */
int acp_kernel_gemm_fp8(const uint8_t* w, const float* w_scale, const uint8_t* x, const float* x_scale, int M, int N,
                        int K, int splits, int epi, int bn, void* out, int iters, float* elapsed_ms);

/* The FP8 row quantiser on the device: x = bf16 bit patterns [rows][cols] (cols % 8 == 0) ->
 * codes = e4m3 [rows][cols], scales = fp32 [rows]; amax = max|x|, s = fp32(amax / 448) (1 for a zero
 * row), code = e4m3_rne(clamp(fp32(x / s), -448, 448)). */
int acp_kernel_quantize_fp8(const uint16_t* x, int rows, int cols, uint8_t* codes, float* scales);

/* Causal paged-KV GQA attention of ONE sequence's prefill chunk.  q: bf16 [q_len][heads][128] (already
 * rotated), k, v: bf16 [ctx][kv_heads][128] — the whole context, the last q_len keys belong to the
 * query tokens (query i sits at absolute position ctx - q_len + i and sees keys 0..that position).
 * The hook scatters k/v into a paged cache with a shuffled page table, runs the kernel and returns
 * out: bf16 [q_len][heads][128].  impl 1 = wgmma kernel (attention_prefill_tc.cu), 0 = round 1's
 * mma.sync kernel.  iters > 0 also times the launch (mean ms, L2 flushed between launches). */
int acp_kernel_attn_prefill(const uint16_t* q, const uint16_t* k, const uint16_t* v, int heads, int kv_heads,
                            int q_len, int ctx, int impl, uint16_t* out, int iters, float* elapsed_ms);

/* The paged K/V cache of the attention hooks below: the pages of all sequences are a shuffled permutation of
 * physical pages 1..n (two spare), page 0 is reserved and zero, and every slot no sequence owns (the tail of a
 * sequence's last page, the spare pages) holds the bf16 bit pattern `stale`, as a recycled page keeps its previous
 * owner's bytes.  A kernel that changes any cache byte it does not own makes the hook return ACP_ERR_GUARD, as does
 * a store past the end of an output buffer. */

/* acp_kernel_attn_prefill for one prefill step of B sequences packed as the engine packs them: q = bf16
 * [sum q_len][heads][128] (sequence after sequence; rows past the step hold `stale`), k, v = bf16
 * [sum ctx_len][kv_heads][128] (each sequence's whole context), out = bf16 [sum q_len][heads][128]; query blocks per
 * sequence as the engine builds them. */
int acp_kernel_attn_prefill_batch(const uint16_t* q, const uint16_t* k, const uint16_t* v, int heads, int kv_heads,
                                  int B, const int* q_len, const int* ctx_len, uint16_t stale, int impl, uint16_t* out,
                                  int iters, float* elapsed_ms);

/* One decode step of B sequences (attn_decode_item_kernel, or attn_decode_kernel + attn_merge_kernel), with the
 * fused RoPE + K/V append of the new token.  k, v = bf16 [sum (ctx_len[b] - 1)][kv_heads][128]: positions
 * 0..ctx_len[b]-2 of each sequence, sequence after sequence.  qkv = the QKV projection rows of the new tokens
 * ([q heads | k heads | v heads], ld = (heads + 2 kv_heads) * 128): bf16 [B][ld] when splits = 0, else fp32 split-K
 * planes [splits][B][ld]; the hook stores them in [n_cap] rows (n_cap >= B) whose rows B.. are NaN.  cos_tab,
 * sin_tab = fp32 [max_pos][64].  mode 0 picks the kernel as the model does, 1 = per-item kernel (ACP_ERR_INVALID
 * when a context needs more than one 1024-token chunk), 2 = chunked + merge.  out = bf16 [B][heads][128];
 * k_new, v_new = bf16 [B][kv_heads][128], the cache slots of position ctx_len[b] - 1 after the step. */
int acp_kernel_attn_decode(const uint16_t* k, const uint16_t* v, const void* qkv, int splits, int n_cap,
                           const float* cos_tab, const float* sin_tab, int max_pos, int B, const int* ctx_len, int heads,
                           int kv_heads, int mode, uint16_t stale, uint16_t* out, uint16_t* k_new, uint16_t* v_new);

/* rope_kv_kernel over T rows of a prefill step: row t is position pos[t] of sequence seq_of_row[t] (B sequences;
 * no (sequence, position) twice).  qkv, splits, n_cap, cos_tab, sin_tab, max_pos as for acp_kernel_attn_decode
 * with T rows.  q_out = the rotated q rows bf16 [T][heads][128]; k_out, v_out = bf16 [T][kv_heads][128], the cache
 * slots the rows were written to. */
int acp_kernel_rope_kv(const void* qkv, int splits, int n_cap, int T, const int* seq_of_row, const int* pos, int B,
                       const float* cos_tab, const float* sin_tab, int max_pos, int heads, int kv_heads, uint16_t stale,
                       uint16_t* q_out, uint16_t* k_out, uint16_t* v_out);

/* The Mixtral mixture-of-experts block of one layer, as Model::moe_mlp launches it: moe_router_kernel ->
 * moe_dispatch_kernel -> moe_gather_kernel -> grouped gate/up GEMM with fused SwiGLU -> grouped down GEMM ->
 * moe_combine_kernel (csrc/moe.cu, the grouped mode of csrc/gemm_wgmma.cuh).
 *   xn = bf16 [T][hidden]; wr = bf16 [E][hidden], the router of all E experts (may be NULL with topk_in);
 *   wgu = bf16 [e_local][2 ffn][hidden] (gate rows, then up rows) and wdown = bf16 [e_local][hidden][ffn]: the
 *   weights of experts e_first .. e_first + e_local - 1 only, as an expert-parallel rank holds them.
 *   bn = 0 picks the N tile of the expert GEMMs as the model does; 16, 32, 64, 128 or 256 forces one.
 *   t_cap >= T: the max_tokens_per_step the expert buffers are sized for.
 *   topk_in, topk_w_in = [T][2] expert ids and weights (both or neither): they replace the router's output.
 * Outputs: topk_idx, topk_w = [T][2]; row_of = [T][2] (-1: expert not local); ranges = [e_local][2] {first row,
 * rows}; tiles = [2 T + e_local][2], the tile list {expert, first row inside the expert}; info = {bn, tiles,
 * n_local = local assignments, tile capacity}; he = bf16 [2 T][ffn] and ye = bf16 [2 T][hidden], of which rows
 * 0..n_local-1 are written; out = bf16 [T][hidden], or with partial_f32 the fp32 sum over the local experts.
 * The hook fills the expert buffers with NaN first and returns ACP_ERR_GUARD when a row past n_local of them was
 * written, an int of the dispatch array past its tile list changed, the tile count exceeds its capacity or a store
 * went past an output.  ACP_ERR_INVALID: hidden % 128, ffn % 64, E outside 2..16, 2 t_cap > 65535. */
int acp_kernel_moe(const uint16_t* xn, const uint16_t* wr, const uint16_t* wgu, const uint16_t* wdown, int T, int hidden,
                   int ffn, int E, int e_first, int e_local, int bn, int t_cap, int partial_f32, const int32_t* topk_in,
                   const float* topk_w_in, int32_t* topk_idx, float* topk_w, int32_t* row_of, int32_t* ranges,
                   int32_t* tiles, int32_t* info, uint16_t* he, uint16_t* ye, void* out);

/* The tool-call grammar of tool_choice "required" / named functions (DESIGN.md §3.3) on the host, no GPU:
 * names_json = JSON array of the allowed tool names (raw, as in `tools`), parallel = parallel_tool_calls.
 * Runs `text` from the start state; *consumed = bytes accepted before the first rejected byte (len when none
 * is), *complete = 1 when all of `text` was accepted and a stop token may follow. */
int acp_kernel_grammar_accepts(const char* names_json, int parallel, const uint8_t* text, size_t len, size_t* consumed,
                               int* complete);

/* grammar_mask_kernel on the device for one row: the state `prefix` reaches (ACP_ERR_INVALID when the grammar
 * rejects it) against a vocabulary given as byte strings — id i is vocab_bytes[vocab_off[i], vocab_off[i+1]),
 * vocab_stop[i] != 0 marks a stop id.  allowed_bits[(vocab + 7) / 8]: bit i (LSB first) = id i allowed. */
int acp_kernel_grammar_mask(const char* names_json, int parallel, const uint8_t* prefix, size_t prefix_len,
                            const int32_t* vocab_off, const uint8_t* vocab_bytes, const uint8_t* vocab_stop, int vocab,
                            uint8_t* allowed_bits);

/* Number of visible CUDA devices (0 when none / no driver). */
int acp_kernel_device_count(void);

#ifdef __cplusplus
}
#endif
#endif
