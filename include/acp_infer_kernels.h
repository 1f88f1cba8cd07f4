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
#ifdef __cplusplus
extern "C" {
#endif

/* out[n][m] = sum_k w[m][k] * x[n][k]; w,x are bf16 bit patterns.
 * epi 0: out = bf16 [N][M]; epi 1: out = fp32 [splits][N][M] (split-K partial planes);
 * epi 2: amax_val/amax_idx = per-row arg-max over M (lowest index wins ties), out = optional
 * fp32 logits [N][M] (may be NULL); epi 3: rows of w interleaved (gate_j, up_j), out = bf16
 * [N][M/2] = bf16(bf16(silu(g)) * u).  bn = 0 picks the N tile from N; otherwise 16..256;
 * bn = -1 (N > 256, epi 0, 1 or 3) forces the persistent prefill kernel.
 * iters > 0 additionally times `iters` launches with CUDA events (L2 flushed between
 * launches) and stores the mean milliseconds in *elapsed_ms; iters < 0 is a stress mode: -iters launches back
 * to back (no flush, one synchronize at the end), mean milliseconds in *elapsed_ms. */
/* Which kernel the dispatcher picks for this problem (host logic only, no GPU needed): 0 = tiled
 * gemm_wx_kernel, 1 = persistent kernel.  `splits`, `epi` and `bn` as below. */
int acp_kernel_gemm_path(int M, int N, int K, int splits, int epi, int bn);

int acp_kernel_gemm(const uint16_t* w, const uint16_t* x, int M, int N, int K, int splits,
                    int epi, int bn, void* out, float* amax_val, int* amax_idx, int iters,
                    float* elapsed_ms);

/* Causal paged-KV GQA attention of ONE sequence's prefill chunk.  q: bf16 [q_len][heads][128] (already
 * rotated), k, v: bf16 [ctx][kv_heads][128] — the whole context, the last q_len keys belong to the
 * query tokens (query i sits at absolute position ctx - q_len + i and sees keys 0..that position).
 * The hook scatters k/v into a paged cache with a shuffled page table, runs the kernel and returns
 * out: bf16 [q_len][heads][128].  impl 1 = wgmma kernel (attention_prefill_tc.cu), 0 = round 1's
 * mma.sync kernel.  iters > 0 also times the launch (mean ms, L2 flushed between launches). */
int acp_kernel_attn_prefill(const uint16_t* q, const uint16_t* k, const uint16_t* v, int heads, int kv_heads,
                            int q_len, int ctx, int impl, uint16_t* out, int iters, float* elapsed_ms);

/* Number of visible CUDA devices (0 when none / no driver). */
int acp_kernel_device_count(void);

#ifdef __cplusplus
}
#endif
#endif
