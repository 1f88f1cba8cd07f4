// fp8.cu — device row quantiser (fp8.h): one CTA per row, two passes over the row (max, then codes).
#include "fp8.h"
#include "common.cuh"
#include <cuda_fp8.h>

namespace acp {

namespace {
constexpr int QT = 256;

// element offset of (row, k) for a chunk of 8 consecutive k: row-major, or the GEMM's tiled layout
// (tiles of 128 rows x `bk` columns, ordered [row tile][k block])
template <bool TILED>
__device__ __forceinline__ size_t q_off(int row, int k, int cols, int bk) {
  if constexpr (TILED)
    return ((size_t)(row / 128) * (cols / bk) + k / bk) * (128 * bk) + (size_t)(row % 128) * bk + (k % bk);
  else
    return (size_t)row * cols + k;
}

template <bool TILED>
__global__ void __launch_bounds__(QT) quantize_rows_e4m3_kernel(const __nv_bfloat16* __restrict__ x, int cols,
                                                                uint8_t* __restrict__ codes, float* __restrict__ scales) {
  __shared__ float red[QT / 32];
  pdl_launch_dependents();
  pdl_wait();
  const int row = blockIdx.x;
  float amax = 0.f;
  for (int k = threadIdx.x * 8; k < cols; k += QT * 8) {
    const uint4 v = *(const uint4*)(x + q_off<TILED>(row, k, cols, 64));
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) amax = fmaxf(amax, fmaxf(fabsf(bf16_lo(w[j])), fabsf(bf16_hi(w[j]))));
  }
  amax = warp_max(amax);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = amax;
  __syncthreads();
  amax = red[0];
#pragma unroll
  for (int i = 1; i < QT / 32; ++i) amax = fmaxf(amax, red[i]);
  const float s = amax == 0.f ? 1.0f : __fdiv_rn(amax, 448.0f);
  if (threadIdx.x == 0) scales[row] = s;
  for (int k = threadIdx.x * 8; k < cols; k += QT * 8) {
    const uint4 v = *(const uint4*)(x + q_off<TILED>(row, k, cols, 64));
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    uint32_t out[2];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float2 q;
      q.x = fminf(fmaxf(__fdiv_rn(bf16_lo(w[j]), s), -448.0f), 448.0f);
      q.y = fminf(fmaxf(__fdiv_rn(bf16_hi(w[j]), s), -448.0f), 448.0f);
      const uint32_t pair = (uint32_t)__nv_cvt_float2_to_fp8x2(q, __NV_SATFINITE, __NV_E4M3);   // RNE
      if (j & 1) out[j >> 1] |= pair << 16;
      else out[j >> 1] = pair;
    }
    *(uint2*)(codes + q_off<TILED>(row, k, cols, 128)) = make_uint2(out[0], out[1]);
  }
}
}  // namespace

int launch_quantize_rows_e4m3(const __nv_bfloat16* x, int rows, int cols, uint8_t* codes, float* scales,
                              cudaStream_t stream) {
  if (rows <= 0) return 0;
  if (cols % 8) return -1;
  cudaError_t e = acp_launch(quantize_rows_e4m3_kernel<false>, dim3(rows), dim3(QT), 0, stream, x, cols, codes, scales);
  return e == cudaSuccess ? 0 : -5;
}

int launch_quantize_weight_e4m3(const __nv_bfloat16* w_tiled, int M, int K, uint8_t* codes_tiled, float* scales,
                                cudaStream_t stream) {
  if (M % 128 || K % 128) return -1;
  cudaError_t e = acp_launch(quantize_rows_e4m3_kernel<true>, dim3(M), dim3(QT), 0, stream, w_tiled, K, codes_tiled, scales);
  return e == cudaSuccess ? 0 : -5;
}

}  // namespace acp
