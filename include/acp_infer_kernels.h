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
/* acp_kernel_gemm / acp_kernel_gemm_fp8: a kernel stored past the end of the output */
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
