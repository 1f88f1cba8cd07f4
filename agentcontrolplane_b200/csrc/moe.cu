// moe.cu — sparse mixture-of-experts MLP (Mixtral): router, token dispatch, weighted combine.
//
// Per layer (T token rows, E experts, top-2; the expert GEMMs are the grouped mode of gemm_wgmma.cuh):
//   moe_router_kernel    r[t][e] = xn[t] . Wr[e] in a FIXED fp32 summation order (the oracle's
//                        router_logits() restates it, so expert selection is bit-identical), top-2 by
//                        logit (lowest index wins ties), w0 = 1/(1+exp(r1-r0)), w1 = exp(r1-r0)/(1+exp(r1-r0))
//   moe_dispatch_kernel  counting sort of the 2T (token, expert) assignments by expert, token order kept
//                        inside an expert: ranges[e] = {first row, rows}, row_of[t][k] = row of assignment k
//                        of token t in the expert-sorted buffers (-1: expert not on this rank)
//   moe_gather_kernel    xe[row_of[t][k]] = xn[t]
//   (grouped GEMMs)      he = swiglu(xe @ Wgu[e]^T), ye = bf16(he @ Wd[e]^T)      per expert row range
//   moe_combine_kernel   out[t] = bf16(w0 * ye[row_of[t][0]] + w1 * ye[row_of[t][1]])   (bf16, one
//                        rounding) — or the fp32 partial sum over this rank's experts (expert parallel:
//                        the tensor-parallel exchange then sums the ranks, rounds once, adds the residual)
//
// Reference boundary: part of the arithmetic behind langchaingo_client.go:102 for BASELINE config 4
// (Mixtral-8x7B); architecture = transformers MixtralSparseMoeBlock (oracle/llama_oracle.py _moe).
#include "moe.h"
#include "common.cuh"
#include "gemm_wgmma.cuh"

namespace acp {

namespace {

constexpr int MOE_MAX_E = GEMM_GROUP_MAX;   // experts per rank

__global__ void __launch_bounds__(128)
moe_router_kernel(const __nv_bfloat16* __restrict__ xn, const __nv_bfloat16* __restrict__ wr, int hidden, int E, int T,
                  int* __restrict__ topk_idx, float* __restrict__ topk_w) {
  pdl_launch_dependents();
  pdl_wait();
  const int t = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (t >= T) return;
  float acc[MOE_MAX_E];
#pragma unroll
  for (int e = 0; e < MOE_MAX_E; ++e) acc[e] = 0.f;
  const __nv_bfloat16* xr = xn + (size_t)t * hidden;
  // lane j owns elements j, j+32, j+64, ... and adds their products in that order (separately
  // rounded multiply and add: no FMA contraction, so numpy reproduces every bit)
  for (int k = lane; k < hidden; k += 32) {
    const float x = __bfloat162float(xr[k]);
#pragma unroll
    for (int e = 0; e < MOE_MAX_E; ++e)
      if (e < E) acc[e] = __fadd_rn(acc[e], __fmul_rn(x, __bfloat162float(wr[(size_t)e * hidden + k])));
  }
  // fold the lanes 16, 8, 4, 2, 1 (lane j < half adds lane j + half): lane 0 ends with the total
#pragma unroll
  for (int half = 16; half >= 1; half >>= 1)
#pragma unroll
    for (int e = 0; e < MOE_MAX_E; ++e)
      if (e < E) acc[e] = __fadd_rn(acc[e], __shfl_down_sync(0xffffffffu, acc[e], half));
  if (lane == 0) {
    int e0 = 0;
    for (int e = 1; e < E; ++e) if (acc[e] > acc[e0]) e0 = e;
    int e1 = e0 == 0 ? 1 : 0;
    for (int e = 0; e < E; ++e) if (e != e0 && acc[e] > acc[e1]) e1 = e;
    // ties: the strict > keeps the lowest index, like numpy's argmax
    const float ex = expf(acc[e1] - acc[e0]);
    topk_idx[2 * t] = e0;
    topk_idx[2 * t + 1] = e1;
    topk_w[2 * t] = 1.0f / (1.0f + ex);
    topk_w[2 * t + 1] = ex / (1.0f + ex);
  }
}

// One CTA of 1024 threads; thread i owns tokens [i*per, (i+1)*per).  Experts e_first .. e_first+e_local-1
// live on this rank (expert parallel); assignments to other experts get row -1.
__global__ void __launch_bounds__(1024)
moe_dispatch_kernel(const int* __restrict__ topk_idx, int T, int e_first, int e_local, int bn, int* __restrict__ ranges,
                    int* __restrict__ row_of) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ unsigned short s_cnt[MOE_MAX_E][1024 + 2];   // per-thread counts, then exclusive prefix per expert (2T <= 65535)
  __shared__ int s_off[MOE_MAX_E + 1];
  const int tid = threadIdx.x;
  const int per = (T + 1023) / 1024;
  const int t0 = tid * per, t1 = min(T, t0 + per);
  int cnt[MOE_MAX_E];
#pragma unroll
  for (int e = 0; e < MOE_MAX_E; ++e) cnt[e] = 0;
  for (int t = t0; t < t1; ++t)
    for (int k = 0; k < 2; ++k) {
      const int e = topk_idx[2 * t + k] - e_first;
      if (e >= 0 && e < e_local) {
#pragma unroll
        for (int q = 0; q < MOE_MAX_E; ++q) if (q == e) ++cnt[q];
      }
    }
#pragma unroll
  for (int e = 0; e < MOE_MAX_E; ++e) if (e < e_local) s_cnt[e][tid] = (unsigned short)cnt[e];
  __syncthreads();
  // exclusive scan over the 1024 per-thread counts of each expert: warp w scans expert w, w+32, ...
  const int warp = tid >> 5, lane = tid & 31;
  for (int e = warp; e < e_local; e += 32) {
    int carry = 0;
    for (int base = 0; base < 1024; base += 32) {
      const int v = s_cnt[e][base + lane];
      int inc = v;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int n = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += n;
      }
      s_cnt[e][base + lane] = (unsigned short)(carry + inc - v);
      carry += __shfl_sync(0xffffffffu, inc, 31);
    }
    if (lane == 0) s_cnt[e][1024] = (unsigned short)carry;   // total rows of expert e
  }
  __syncthreads();
  if (tid == 0) {
    int off = 0;
    for (int e = 0; e < e_local; ++e) {
      s_off[e] = off;
      ranges[2 * e] = off;
      ranges[2 * e + 1] = s_cnt[e][1024];
      off += s_cnt[e][1024];
    }
    s_off[e_local] = off;
    // flat work list of the grouped GEMMs (layout: GEMM_GROUP_TILES in gemm_wgmma.cuh): one entry
    // {expert, first row inside the expert} per BN-row tile
    int n = 0;
    int* tiles = ranges + GEMM_GROUP_TILES + 2;
    for (int e = 0; e < e_local; ++e)
      for (int n0 = 0; n0 < (int)s_cnt[e][1024]; n0 += bn) { tiles[2 * n] = e; tiles[2 * n + 1] = n0; ++n; }
    ranges[GEMM_GROUP_TILES] = n;
  }
  __syncthreads();
  int pos[MOE_MAX_E];
#pragma unroll
  for (int e = 0; e < MOE_MAX_E; ++e) pos[e] = (e < e_local) ? s_off[e] + s_cnt[e][tid] : 0;
  for (int t = t0; t < t1; ++t)
    for (int k = 0; k < 2; ++k) {
      const int e = topk_idx[2 * t + k] - e_first;
      int r = -1;
      if (e >= 0 && e < e_local) {
#pragma unroll
        for (int q = 0; q < MOE_MAX_E; ++q) if (q == e) r = pos[q]++;
      }
      row_of[2 * t + k] = r;
    }
}

__global__ void __launch_bounds__(128)
moe_gather_kernel(const __nv_bfloat16* __restrict__ xn, const int* __restrict__ row_of, int hidden,
                  __nv_bfloat16* __restrict__ xe) {
  pdl_launch_dependents();
  pdl_wait();
  const int t = blockIdx.x;
  const uint4* src = reinterpret_cast<const uint4*>(xn + (size_t)t * hidden);
  for (int k = 0; k < 2; ++k) {
    const int r = row_of[2 * t + k];
    if (r < 0) continue;
    uint4* dst = reinterpret_cast<uint4*>(xe + (size_t)r * hidden);
    for (int i = threadIdx.x; i < hidden / 8; i += blockDim.x) dst[i] = src[i];
  }
}

template <bool PARTIAL_F32>
__global__ void __launch_bounds__(128)
moe_combine_kernel(const __nv_bfloat16* __restrict__ ye, const int* __restrict__ row_of, const float* __restrict__ topk_w,
                   int hidden, void* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  const int t = blockIdx.x;
  const int r0 = row_of[2 * t], r1 = row_of[2 * t + 1];
  const float w0 = topk_w[2 * t], w1 = topk_w[2 * t + 1];
  for (int i = threadIdx.x * 4; i < hidden; i += blockDim.x * 4) {
    float a[4] = {0.f, 0.f, 0.f, 0.f}, b[4] = {0.f, 0.f, 0.f, 0.f};
    if (r0 >= 0) {
      const uint2 raw = *reinterpret_cast<const uint2*>(ye + (size_t)r0 * hidden + i);
      a[0] = bf16_lo(raw.x); a[1] = bf16_hi(raw.x); a[2] = bf16_lo(raw.y); a[3] = bf16_hi(raw.y);
    }
    if (r1 >= 0) {
      const uint2 raw = *reinterpret_cast<const uint2*>(ye + (size_t)r1 * hidden + i);
      b[0] = bf16_lo(raw.x); b[1] = bf16_hi(raw.x); b[2] = bf16_lo(raw.y); b[3] = bf16_hi(raw.y);
    }
    float o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) o[j] = __fadd_rn(__fmul_rn(w0, a[j]), __fmul_rn(w1, b[j]));
    if constexpr (PARTIAL_F32) {
      *reinterpret_cast<float4*>((float*)out + (size_t)t * hidden + i) = make_float4(o[0], o[1], o[2], o[3]);
    } else {
      uint2 packed;
      packed.x = pack_bf16x2(o[0], o[1]);
      packed.y = pack_bf16x2(o[2], o[3]);
      *reinterpret_cast<uint2*>((__nv_bfloat16*)out + (size_t)t * hidden + i) = packed;
    }
  }
}

}  // namespace

#define MOE_LAUNCH(name, call)                                                              \
  do {                                                                                      \
    cudaError_t _e = (call);                                                                \
    if (_e != cudaSuccess) {                                                                \
      fprintf(stderr, "[acp_infer] launch %s failed: %s\n", name, cudaGetErrorString(_e));  \
      return -5;                                                                            \
    }                                                                                       \
  } while (0)

int launch_moe_router(const __nv_bfloat16* xn, const __nv_bfloat16* wr, int hidden, int E, int T, int* topk_idx,
                      float* topk_w, cudaStream_t s) {
  if (T <= 0) return 0;
  if (E < 2 || E > MOE_MAX_E || hidden % 32) return -1;
  MOE_LAUNCH("moe_router", acp_launch(moe_router_kernel, dim3((T + 3) / 4), dim3(128), 0, s, xn, wr, hidden, E, T, topk_idx, topk_w));
  return 0;
}
int launch_moe_dispatch(const int* topk_idx, int T, int e_first, int e_local, int bn, int* ranges, int* row_of, cudaStream_t s) {
  if (T <= 0) return 0;
  if (e_local < 1 || e_local > MOE_MAX_E || 2 * T > 65535 || bn < 16) return -1;
  MOE_LAUNCH("moe_dispatch", acp_launch(moe_dispatch_kernel, dim3(1), dim3(1024), 0, s, topk_idx, T, e_first, e_local, bn, ranges, row_of));
  return 0;
}
int moe_ranges_ints(int T) { return GEMM_GROUP_TILES + 2 + 2 * (2 * T / 16 + MOE_MAX_E + 1); }
int moe_tile_cap(int T, int bn, int e_local) { return (2 * T + bn - 1) / bn + e_local; }
int launch_moe_gather(const __nv_bfloat16* xn, const int* row_of, int hidden, int T, __nv_bfloat16* xe, cudaStream_t s) {
  if (T <= 0) return 0;
  MOE_LAUNCH("moe_gather", acp_launch(moe_gather_kernel, dim3(T), dim3(128), 0, s, xn, row_of, hidden, xe));
  return 0;
}
int launch_moe_combine(const __nv_bfloat16* ye, const int* row_of, const float* topk_w, int hidden, int T, void* out,
                       bool partial_f32, cudaStream_t s) {
  if (T <= 0) return 0;
  if (partial_f32) MOE_LAUNCH("moe_combine_f32", acp_launch(moe_combine_kernel<true>, dim3(T), dim3(128), 0, s, ye, row_of, topk_w, hidden, out));
  else MOE_LAUNCH("moe_combine", acp_launch(moe_combine_kernel<false>, dim3(T), dim3(128), 0, s, ye, row_of, topk_w, hidden, out));
  return 0;
}

}  // namespace acp
