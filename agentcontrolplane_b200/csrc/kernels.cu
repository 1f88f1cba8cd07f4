// kernels.cu — HBM-bound kernels: embedding gather, (residual add +) RMSNorm, RoPE + paged-KV
// scatter, SwiGLU, arg-max finish, sampling, synthetic weight generation.
// All vectorised (8/16-byte accesses), warp-shuffle reductions, bf16 round-to-nearest-even at
// exactly the points listed in oracle/llama_oracle.py.
#include "kernels.cuh"
#include "common.cuh"
#include "gemm_out.cuh"

namespace acp {

#define ACP_LAUNCH(name, call)                                                         \
  do {                                                                                 \
    cudaError_t _e = (call);                                                           \
    if (_e != cudaSuccess) {                                                           \
      fprintf(stderr, "[acp_infer] launch %s failed: %s\n", name, cudaGetErrorString(_e)); \
      return -5;                                                                       \
    }                                                                                  \
  } while (0)
#define ACP_LAUNCH_CHECK(name)                                                         \
  do {                                                                                 \
    cudaError_t _e = cudaGetLastError();                                               \
    if (_e != cudaSuccess) {                                                           \
      fprintf(stderr, "[acp_infer] launch %s failed: %s\n", name, cudaGetErrorString(_e)); \
      return -5;                                                                       \
    }                                                                                  \
  } while (0)

// ---------------------------------------------------------------------------------
// embedding gather
// ---------------------------------------------------------------------------------
__global__ void embed_kernel(const int* __restrict__ tok, const __nv_bfloat16* __restrict__ E,
                             __nv_bfloat16* __restrict__ x, int hidden) {
  pdl_launch_dependents();
  pdl_wait();
  const int t = blockIdx.x;
  const uint4* src = reinterpret_cast<const uint4*>(E + (size_t)tok[t] * hidden);
  uint4* dst = reinterpret_cast<uint4*>(x + (size_t)t * hidden);
  for (int i = threadIdx.x; i < hidden / 8; i += blockDim.x) dst[i] = src[i];
}
int launch_embed(const int* tok, const __nv_bfloat16* E, __nv_bfloat16* x, int T, int hidden,
                 cudaStream_t s) {
  if (T <= 0) return 0;
  ACP_LAUNCH("embed", acp_launch(embed_kernel, dim3(T), dim3(128), 0, s, tok, E, x, hidden));
  return 0;
}

// ---------------------------------------------------------------------------------
// (residual add +) RMSNorm.  One CTA per output row, row staged in shared memory as fp32.
// ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024)
add_rmsnorm_kernel(__nv_bfloat16* __restrict__ x, GemmOutDev add, const __nv_bfloat16* __restrict__ gain,
                   __nv_bfloat16* __restrict__ xn, const int* __restrict__ row_map, int hidden,
                   float eps) {
  pdl_launch_dependents();
  pdl_wait();
  extern __shared__ float row[];
  __shared__ float red[32];
  const int out_row = blockIdx.x;
  const int src_row = row_map ? row_map[out_row] : out_row;
  __nv_bfloat16* xr = x + (size_t)src_row * hidden;
  float ss = 0.f;
  for (int i = threadIdx.x * 4; i < hidden; i += blockDim.x * 4) {
    const uint2 raw = *reinterpret_cast<const uint2*>(xr + i);
    float v[4] = {bf16_lo(raw.x), bf16_hi(raw.x), bf16_lo(raw.y), bf16_hi(raw.y)};
    if (add.ptr != nullptr) {
      float a[4];
      gemm_out_load4(add, src_row, i, a);
#pragma unroll
      for (int j = 0; j < 4; ++j) v[j] = bf16_round(v[j] + a[j]);
      if (row_map == nullptr) {
        uint2 packed;
        packed.x = pack_bf16x2(v[0], v[1]);
        packed.y = pack_bf16x2(v[2], v[3]);
        *reinterpret_cast<uint2*>(xr + i) = packed;
      }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) { row[i + j] = v[j]; ss += v[j] * v[j]; }
  }
  ss = warp_sum(ss);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
  __syncthreads();
  float tot = 0.f;
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) tot += red[w];
  const float rstd = 1.0f / sqrtf(tot / (float)hidden + eps);
  __nv_bfloat16* o = xn + (size_t)out_row * hidden;
  for (int i = threadIdx.x * 4; i < hidden; i += blockDim.x * 4) {
    const uint2 graw = *reinterpret_cast<const uint2*>(gain + i);
    const float g[4] = {bf16_lo(graw.x), bf16_hi(graw.x), bf16_lo(graw.y), bf16_hi(graw.y)};
    float y[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) y[j] = g[j] * bf16_round(row[i + j] * rstd);
    uint2 packed;
    packed.x = pack_bf16x2(y[0], y[1]);
    packed.y = pack_bf16x2(y[2], y[3]);
    *reinterpret_cast<uint2*>(o + i) = packed;
  }
}
// Prefill variant (bf16 GEMM output, rows updated in place): 128 threads per row, each thread keeps
// its <= 64 elements in registers, every 16-byte load of the row is issued before the first use.
ACP_DEVINL void unpack8(const uint4& r, float (&v)[8]) {
  v[0] = bf16_lo(r.x); v[1] = bf16_hi(r.x); v[2] = bf16_lo(r.y); v[3] = bf16_hi(r.y);
  v[4] = bf16_lo(r.z); v[5] = bf16_hi(r.z); v[6] = bf16_lo(r.w); v[7] = bf16_hi(r.w);
}
ACP_DEVINL uint4 pack8(const float (&v)[8]) {
  uint4 r;
  r.x = pack_bf16x2(v[0], v[1]); r.y = pack_bf16x2(v[2], v[3]);
  r.z = pack_bf16x2(v[4], v[5]); r.w = pack_bf16x2(v[6], v[7]);
  return r;
}
__global__ void __launch_bounds__(128)
add_rmsnorm_bf16_kernel(__nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ add, int add_ld,
                        const __nv_bfloat16* __restrict__ gain, __nv_bfloat16* __restrict__ xn, int hidden,
                        float eps) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float red[4];
  const int t = blockIdx.x;
  const int nv = hidden / 8;  // 16-byte chunks per row (<= 1024)
  uint4* xr = reinterpret_cast<uint4*>(x + (size_t)t * hidden);
  const uint4* ar = reinterpret_cast<const uint4*>(add + (size_t)t * add_ld);
  uint4 xraw[8], araw[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const int ch = threadIdx.x + c * 128;
    if (ch < nv) { xraw[c] = xr[ch]; araw[c] = ar[ch]; }
  }
  float v[8][8];
  float ss = 0.f;
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const int ch = threadIdx.x + c * 128;
    if (ch < nv) {
      float a[8];
      unpack8(xraw[c], v[c]);
      unpack8(araw[c], a);
#pragma unroll
      for (int j = 0; j < 8; ++j) { v[c][j] = bf16_round(v[c][j] + a[j]); ss += v[c][j] * v[c][j]; }
      xr[ch] = pack8(v[c]);
    }
  }
  ss = warp_sum(ss);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
  __syncthreads();
  const float tot = red[0] + red[1] + red[2] + red[3];
  const float rstd = 1.0f / sqrtf(tot / (float)hidden + eps);
  uint4* o = reinterpret_cast<uint4*>(xn + (size_t)t * hidden);
  const uint4* gr = reinterpret_cast<const uint4*>(gain);
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const int ch = threadIdx.x + c * 128;
    if (ch < nv) {
      float g[8], y[8];
      unpack8(gr[ch], g);
#pragma unroll
      for (int j = 0; j < 8; ++j) y[j] = g[j] * bf16_round(v[c][j] * rstd);
      o[ch] = pack8(y);
    }
  }
}

int launch_add_rmsnorm(__nv_bfloat16* x, const GemmOut& add, const __nv_bfloat16* gain,
                       __nv_bfloat16* xn, const int* row_map, int T, int hidden, float eps,
                       cudaStream_t s) {
  if (T <= 0) return 0;
  if (add.ptr != nullptr && add.splits == 0 && row_map == nullptr && hidden % 8 == 0 && hidden <= 8192) {
    ACP_LAUNCH("add_rmsnorm_bf16", acp_launch(add_rmsnorm_bf16_kernel, dim3(T), dim3(128), 0, s, x,
                                            (const __nv_bfloat16*)add.ptr, add.ld, gain, xn, hidden, eps));
    return 0;
  }
  // one thread per 4 elements (single trip through the loads => one L2 round trip per phase)
  int threads = ((hidden / 4 + 31) / 32) * 32;
  if (threads > 1024) threads = 1024;
  ACP_LAUNCH("add_rmsnorm", acp_launch(add_rmsnorm_kernel, dim3(T), dim3(threads), hidden * sizeof(float), s, x,
                                       to_dev(add), gain, xn, row_map, hidden, eps));
  return 0;
}

// ---------------------------------------------------------------------------------
// RoPE + paged-KV scatter.  One CTA per token row; each thread handles 4 consecutive "i"
// (frequency indices) of one head: elements (i, i+64) of the 128-wide head vector.
// ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024)
rope_kv_kernel(GemmOutDev qkv, const int* __restrict__ pos, const int* __restrict__ seq_of_row,
               const int* __restrict__ page_table, int max_pages, const float* __restrict__ cos_tab,
               const float* __restrict__ sin_tab, __nv_bfloat16* __restrict__ qbuf,
               __nv_bfloat16* __restrict__ k_cache, __nv_bfloat16* __restrict__ v_cache, int heads,
               int kv_heads) {
  pdl_launch_dependents();
  pdl_wait();
  const int t = blockIdx.x;
  const int p = pos[t];
  const int seq = seq_of_row[t];
  const int page = page_table[(size_t)seq * max_pages + p / KV_PAGE];
  const int q_dim = heads * HEAD_DIM, kv_dim = kv_heads * HEAD_DIM;
  const float* ct = cos_tab + (size_t)p * (HEAD_DIM / 2);
  const float* st = sin_tab + (size_t)p * (HEAD_DIM / 2);
  // rotated heads: q heads then k heads; 16 threads per head (4 i's each)
  const int n_rot = heads + kv_heads;
  for (int w = threadIdx.x; w < n_rot * 16; w += blockDim.x) {
    const int head = w >> 4, i0 = (w & 15) * 4;
    const int col = head * HEAD_DIM;  // q heads and k heads are contiguous in the qkv row
    float a[4], b[4];
    gemm_out_load4(qkv, t, col + i0, a);
    gemm_out_load4(qkv, t, col + 64 + i0, b);
    const float4 c = *reinterpret_cast<const float4*>(ct + i0);
    const float4 s = *reinterpret_cast<const float4*>(st + i0);
    const float cc[4] = {c.x, c.y, c.z, c.w}, sn[4] = {s.x, s.y, s.z, s.w};
    float lo[4], hi[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      // explicit rn ops: no FMA contraction, so the oracle's numpy expression matches bit for bit
      lo[j] = __fsub_rn(__fmul_rn(a[j], cc[j]), __fmul_rn(b[j], sn[j]));
      hi[j] = __fadd_rn(__fmul_rn(b[j], cc[j]), __fmul_rn(a[j], sn[j]));
    }
    uint2 plo, phi;
    plo.x = pack_bf16x2(lo[0], lo[1]); plo.y = pack_bf16x2(lo[2], lo[3]);
    phi.x = pack_bf16x2(hi[0], hi[1]); phi.y = pack_bf16x2(hi[2], hi[3]);
    __nv_bfloat16* dst;
    if (head < heads) {
      dst = qbuf + (size_t)t * q_dim + head * HEAD_DIM;
    } else {
      // K/V block of a (page, kv head): [2 dim-halves][32 tokens][64 dims] = 8 KiB contiguous
      const int kh = head - heads;
      dst = k_cache + ((size_t)page * kv_heads + kh) * (KV_PAGE * HEAD_DIM) + (p % KV_PAGE) * 64;
      *reinterpret_cast<uint2*>(dst + i0) = plo;
      *reinterpret_cast<uint2*>(dst + KV_PAGE * 64 + i0) = phi;
      continue;
    }
    *reinterpret_cast<uint2*>(dst + i0) = plo;
    *reinterpret_cast<uint2*>(dst + 64 + i0) = phi;
  }
  // v: plain copy, 4 elements per thread
  for (int w = threadIdx.x; w < kv_dim / 4; w += blockDim.x) {
    const int e = w * 4;
    float v[4];
    gemm_out_load4(qkv, t, q_dim + kv_dim + e, v);
    const int kh = e / HEAD_DIM, d = e % HEAD_DIM;
    uint2 pv;
    pv.x = pack_bf16x2(v[0], v[1]); pv.y = pack_bf16x2(v[2], v[3]);
    *reinterpret_cast<uint2*>(v_cache + ((size_t)page * kv_heads + kh) * (KV_PAGE * HEAD_DIM) +
                              (d >> 6) * (KV_PAGE * 64) + (p % KV_PAGE) * 64 + (d & 63)) = pv;
  }
}
int launch_rope_kv(const RopeKvArgs& a, cudaStream_t s) {
  if (a.T <= 0) return 0;
  int threads = (a.heads + a.kv_heads) * 16;   // one thread per 4 rotated pairs
  threads = ((threads + 31) / 32) * 32;
  if (threads > 1024) threads = 1024;
  ACP_LAUNCH("rope_kv", acp_launch(rope_kv_kernel, dim3(a.T), dim3(threads), 0, s, to_dev(a.qkv), a.pos,
                                   a.seq_of_row, a.page_table, a.max_pages, a.cos_tab, a.sin_tab, a.qbuf,
                                   a.k_cache, a.v_cache, a.heads, a.kv_heads));
  return 0;
}

// ---------------------------------------------------------------------------------
// SwiGLU
// ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
swiglu_kernel(GemmOutDev gu, __nv_bfloat16* __restrict__ h, int ffn) {
  pdl_launch_dependents();
  pdl_wait();
  // gate/up columns are interleaved: column 2j = gate_j, 2j+1 = up_j.  4 outputs per thread.
  const int t = blockIdx.y;
  const int j = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (j >= ffn) return;
  float a[4], b[4], o[4];
  gemm_out_load4(gu, t, 2 * j, a);       // g0 u0 g1 u1
  gemm_out_load4(gu, t, 2 * j + 4, b);   // g2 u2 g3 u3
  const float g[4] = {a[0], a[2], b[0], b[2]}, u[4] = {a[1], a[3], b[1], b[3]};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float act = bf16_round(g[k] / (1.0f + expf(-g[k])));
    o[k] = act * u[k];
  }
  uint2 packed;
  packed.x = pack_bf16x2(o[0], o[1]);
  packed.y = pack_bf16x2(o[2], o[3]);
  *reinterpret_cast<uint2*>(h + (size_t)t * ffn + j) = packed;
}
int launch_swiglu(const GemmOut& gu, __nv_bfloat16* h, int T, int ffn, cudaStream_t s) {
  if (T <= 0) return 0;
  dim3 grid((ffn / 4 + 255) / 256, T);
  ACP_LAUNCH("swiglu", acp_launch(swiglu_kernel, grid, dim3(256), 0, s, to_dev(gu), h, ffn));
  return 0;
}

// ---------------------------------------------------------------------------------
// arg-max finish: reduce the per-m-tile candidates of the fused LM-head epilogue
// ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
argmax_finish_kernel(const float* __restrict__ tile_val, const int* __restrict__ tile_idx,
                     int m_tiles, int* __restrict__ token_out, float* __restrict__ val_out) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float sv[4];
  __shared__ int si[4];
  const int n = blockIdx.x;
  float v = -INFINITY;
  int idx = 0x7fffffff;
  for (int t = threadIdx.x; t < m_tiles; t += blockDim.x) {
    const float ov = tile_val[(size_t)n * m_tiles + t];
    const int oi = tile_idx[(size_t)n * m_tiles + t];
    if (ov > v || (ov == v && oi < idx)) { v = ov; idx = oi; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, v, o);
    const int oi = __shfl_xor_sync(0xffffffffu, idx, o);
    if (ov > v || (ov == v && oi < idx)) { v = ov; idx = oi; }
  }
  if ((threadIdx.x & 31) == 0) { sv[threadIdx.x >> 5] = v; si[threadIdx.x >> 5] = idx; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < 4; ++w)
      if (sv[w] > v || (sv[w] == v && si[w] < idx)) { v = sv[w]; idx = si[w]; }
    token_out[n] = idx;
    if (val_out) val_out[n] = v;
  }
}
int launch_argmax_finish(const float* tile_val, const int* tile_idx, int m_tiles, int N,
                         int* token_out, float* val_out, cudaStream_t s) {
  if (N <= 0) return 0;
  ACP_LAUNCH("argmax_finish", acp_launch(argmax_finish_kernel, dim3(N), dim3(128), 0, s, tile_val, tile_idx,
                                         m_tiles, token_out, val_out));
  return 0;
}

// ---------------------------------------------------------------------------------
// Sampling: temperature / top-k / top-p on fp32 logits, one CTA per row.
//   1. m = max logit; weights w_i = exp((l_i - m)/T)
//   2. top-k: threshold = k-th largest logit, found by bisection on the value range
//   3. top-p: smallest threshold tau such that sum_{w_i >= tau} w_i >= top_p * Z (bisection)
//   4. inverse-CDF walk in index order over the kept set with a counter-based uniform.
// Everything is a deterministic function of (logits, params): reductions are fixed-shape.
// ---------------------------------------------------------------------------------
ACP_DEVINL float block_sum(float v, float* red) {
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.f;
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += red[w];
  return t;
}
ACP_DEVINL float block_max(float v, float* red) {
  v = warp_max(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = -INFINITY;
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t = fmaxf(t, red[w]);
  return t;
}
ACP_DEVINL uint64_t splitmix64(uint64_t z) {
  z ^= z >> 30; z *= 0xBF58476D1CE4E5B9ull;
  z ^= z >> 27; z *= 0x94D049BB133111EBull;
  z ^= z >> 31;
  return z;
}

__global__ void __launch_bounds__(1024)
sample_kernel(const float* __restrict__ logits, int V, const SampleParams* __restrict__ params,
              int* __restrict__ token_out) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float red[32];
  __shared__ float s_prefix[1024];
  const int n = blockIdx.x;
  const SampleParams sp = params[n];
  const float* l = logits + (size_t)n * V;
  float lmax = -INFINITY;
  for (int i = threadIdx.x; i < V; i += blockDim.x) lmax = fmaxf(lmax, l[i]);
  lmax = block_max(lmax, red);
  if (sp.temperature <= 0.f) {  // greedy: lowest index among maxima
    int best = 0x7fffffff;
    for (int i = threadIdx.x; i < V; i += blockDim.x)
      if (l[i] == lmax) best = min(best, i);
    best = -(int)block_max((float)(-best), red);  // V < 2^24 so exact in fp32
    if (threadIdx.x == 0) token_out[n] = best;
    return;
  }
  const float invT = 1.0f / sp.temperature;
  float lo_thr = -INFINITY;  // keep logits >= lo_thr
  if (sp.top_k > 0 && sp.top_k < V) {
    float lo = lmax - 80.f * sp.temperature - 1.f, hi = lmax;
    // smallest interval [lo, hi] with count(l >= hi) <= k: 40 bisection steps
    for (int it = 0; it < 40; ++it) {
      const float mid = 0.5f * (lo + hi);
      float c = 0.f;
      for (int i = threadIdx.x; i < V; i += blockDim.x) c += (l[i] >= mid) ? 1.f : 0.f;
      c = block_sum(c, red);
      if (c > (float)sp.top_k) lo = mid; else hi = mid;
    }
    lo_thr = hi;
  }
  float z = 0.f;
  for (int i = threadIdx.x; i < V; i += blockDim.x)
    if (l[i] >= lo_thr) z += expf((l[i] - lmax) * invT);
  z = block_sum(z, red);
  if (sp.top_p < 1.0f) {
    float lo = fmaxf(lo_thr, lmax - 80.f * sp.temperature - 1.f), hi = lmax;
    for (int it = 0; it < 40; ++it) {
      const float mid = 0.5f * (lo + hi);
      float m = 0.f;
      for (int i = threadIdx.x; i < V; i += blockDim.x)
        if (l[i] >= mid && l[i] >= lo_thr) m += expf((l[i] - lmax) * invT);
      m = block_sum(m, red);
      if (m >= sp.top_p * z) lo = mid; else hi = mid;
    }
    lo_thr = fmaxf(lo_thr, lo);
    z = 0.f;
    for (int i = threadIdx.x; i < V; i += blockDim.x)
      if (l[i] >= lo_thr) z += expf((l[i] - lmax) * invT);
    z = block_sum(z, red);
  }
  // uniform in [0,1) from (seed, step)
  const uint64_t r = splitmix64(sp.seed * 0x9E3779B97F4A7C15ull + (uint64_t)sp.step + 1ull);
  const float u = (float)(r >> 40) * (1.0f / 16777216.0f);
  const float target = u * z;
  // contiguous chunk per thread so the CDF walk is in index order
  const int chunk = (V + blockDim.x - 1) / blockDim.x;
  const int b = threadIdx.x * chunk, e = min(V, b + chunk);
  float mine = 0.f;
  for (int i = b; i < e; ++i)
    if (l[i] >= lo_thr) mine += expf((l[i] - lmax) * invT);
  s_prefix[threadIdx.x] = mine;
  __syncthreads();
  if (threadIdx.x == 0) {
    float acc = 0.f;
    int chosen_thread = -1;
    float base = 0.f;
    for (int t = 0; t < (int)blockDim.x; ++t) {
      if (acc + s_prefix[t] > target && s_prefix[t] > 0.f) { chosen_thread = t; base = acc; break; }
      acc += s_prefix[t];
    }
    int tok = -1;
    if (chosen_thread >= 0) {
      const int bb = chosen_thread * chunk, ee = min(V, bb + chunk);
      float a2 = base;
      for (int i = bb; i < ee; ++i) {
        if (l[i] >= lo_thr) {
          a2 += expf((l[i] - lmax) * invT);
          tok = i;  // last kept index seen; stop once the CDF passes the target
          if (a2 > target) break;
        }
      }
    }
    if (tok < 0) {  // numerical corner (target == z): fall back to the arg-max
      for (int i = 0; i < V; ++i) if (l[i] == lmax) { tok = i; break; }
    }
    token_out[n] = tok;
  }
}
int launch_sample(const float* logits, int V, int N, const SampleParams* params_dev,
                  int* token_out, cudaStream_t s) {
  if (N <= 0) return 0;
  ACP_LAUNCH("sample", acp_launch(sample_kernel, dim3(N), dim3(1024), 0, s, logits, V, params_dev, token_out));
  return 0;
}

// ---------------------------------------------------------------------------------
// synthetic weights (bit-identical to oracle/synth.py)
// ---------------------------------------------------------------------------------
// Local element i of a (possibly tiled / interleaved / sharded) tensor -> index in the logical
// row-major tensor whose values oracle/synth.py defines.
__device__ __forceinline__ size_t synth_logical_index(size_t i, const SynthMap& mp) {
  if (mp.local_cols <= 1) return i;
  // storage is tiled: [m_tile][kb][128 rows][64 cols]  ->  local (row, col) of element i
  const size_t nkb = (size_t)mp.local_cols / 64;
  const size_t tile = i / 8192, in_tile = i % 8192;
  const size_t r = (tile / nkb) * 128 + in_tile / 64, c = (tile % nkb) * 64 + in_tile % 64;
  size_t lr;
  if (mp.interleave_half > 0) {
    lr = (size_t)mp.seg_global[r & 1] + (r >> 1);
  } else {
    size_t rr = r;
    int sg = 0;
    while (sg + 1 < mp.nseg && rr >= (size_t)mp.seg_rows[sg]) { rr -= (size_t)mp.seg_rows[sg]; ++sg; }
    lr = (size_t)mp.seg_global[sg] + rr;
  }
  return lr * (size_t)mp.logical_cols + (size_t)mp.col0 + c;
}

__global__ void synth_weight_kernel(__nv_bfloat16* __restrict__ out, size_t n, uint64_t base,
                                    float scale, int plus_one, SynthMap mp) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) {
    const size_t li = synth_logical_index(i, mp);
    const uint64_t z = splitmix64(base + (uint64_t)li * 0xD1B54A32D192ED03ull);
    const int s = (int)(z & 0xffff) + (int)((z >> 16) & 0xffff) + (int)((z >> 32) & 0xffff) +
                  (int)(z >> 48) - 131070;
    float w = __fmul_rn((float)s, scale);
    if (plus_one) w = __fadd_rn(w, 1.0f);
    out[i] = __float2bfloat16_rn(w);
  }
}

// Checkpoint weights: `src` holds the logical row-major tensor (or the part of it that starts at
// logical element `src_elem0`); every local element fetches its value through the same map the
// synthetic generator uses, so tiling / interleaving / sharding are defined in ONE place.
__global__ void gather_weight_kernel(__nv_bfloat16* __restrict__ out, size_t n,
                                     const __nv_bfloat16* __restrict__ src, size_t src_elem0, SynthMap mp) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) out[i] = src[synth_logical_index(i, mp) - src_elem0];
}
int launch_gather_weight(__nv_bfloat16* out, size_t n, const __nv_bfloat16* src, size_t src_elem0,
                         cudaStream_t s, const SynthMap& map) {
  if (n == 0) return 0;
  gather_weight_kernel<<<132 * 8, 256, 0, s>>>(out, n, src, src_elem0, map);
  ACP_LAUNCH_CHECK("gather_weight");
  return 0;
}

int launch_synth(__nv_bfloat16* out, size_t n, uint64_t seed, uint32_t tid, double std,
                 int plus_one, cudaStream_t s, const SynthMap& map) {
  if (n == 0) return 0;
  const uint64_t base = seed + (uint64_t)tid * 0x9E3779B97F4A7C15ull;
  const float scale = (float)(std / 37837.22671196048);
  synth_weight_kernel<<<132 * 8, 256, 0, s>>>(out, n, base, scale, plus_one, map);
  ACP_LAUNCH_CHECK("synth");
  return 0;
}

// ---------------------------------------------------------------------------------
// tensor-parallel helpers
// ---------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
reduce_planes_kernel(const float* __restrict__ planes, int splits, size_t plane_elems, float* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t i = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (i >= plane_elems) return;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int s0 = 0; s0 < splits; s0 += 8) {
    float4 q[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int sj = (s0 + j < splits) ? s0 + j : splits - 1;
      q[j] = ld_nc_f4(planes + (size_t)sj * plane_elems + i);
    }
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (s0 + j < splits) { acc.x += q[j].x; acc.y += q[j].y; acc.z += q[j].z; acc.w += q[j].w; }
  }
  *reinterpret_cast<float4*>(out + i) = acc;
}
int launch_reduce_planes(const float* planes, int splits, size_t plane_elems, float* out, cudaStream_t s) {
  if (plane_elems == 0) return 0;
  const unsigned blocks = (unsigned)((plane_elems / 4 + 255) / 256);
  ACP_LAUNCH("reduce_planes", acp_launch(reduce_planes_kernel, dim3(blocks), dim3(256), 0, s, planes, splits, plane_elems, out));
  return 0;
}

__global__ void pack_candidates_kernel(const float* __restrict__ val, const int* __restrict__ idx,
                                       int idx_offset, int B, int* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b < B) { out[b] = __float_as_int(val[b]); out[B + b] = idx[b] + idx_offset; }
}
int launch_pack_candidates(const float* val, const int* idx, int idx_offset, int B, int* out, cudaStream_t s) {
  if (B <= 0) return 0;
  ACP_LAUNCH("pack_candidates", acp_launch(pack_candidates_kernel, dim3((B + 127) / 128), dim3(128), 0, s, val, idx, idx_offset, B, out));
  return 0;
}
__global__ void argmax_ranks_kernel(const int* __restrict__ gathered, int P, int B, int* __restrict__ token_out) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  float v = -INFINITY;
  int idx = 0x7fffffff;
  for (int r = 0; r < P; ++r) {  // fixed order; lowest id wins ties
    const float ov = __int_as_float(gathered[(size_t)r * 2 * B + b]);
    const int oi = gathered[(size_t)r * 2 * B + B + b];
    if (ov > v || (ov == v && oi < idx)) { v = ov; idx = oi; }
  }
  token_out[b] = idx;
}
int launch_argmax_ranks(const int* gathered, int P, int B, int* token_out, cudaStream_t s) {
  if (B <= 0) return 0;
  argmax_ranks_kernel<<<(B + 127) / 128, 128, 0, s>>>(gathered, P, B, token_out);
  ACP_LAUNCH_CHECK("argmax_ranks");
  return 0;
}

// [P][n][rows_per_rank] padded logit shards (rank r holds vocabulary rows r*rows_per_rank ...) -> [n][vocab]
__global__ void __launch_bounds__(256)
repack_logits_kernel(const float* __restrict__ gathered, int n, int rows_per_rank, int vocab, float* __restrict__ out) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)n * vocab) return;
  const int row = (int)(i / vocab), v = (int)(i % vocab);
  const int r = v / rows_per_rank, c = v % rows_per_rank;
  out[i] = gathered[((size_t)r * n + row) * rows_per_rank + c];
}
int launch_repack_logits(const float* gathered, int P, int n, int rows_per_rank, int vocab, float* out, cudaStream_t s) {
  (void)P;
  if (n <= 0) return 0;
  const size_t total = (size_t)n * vocab;
  ACP_LAUNCH("repack_logits", acp_launch(repack_logits_kernel, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, s,
                                         gathered, n, rows_per_rank, vocab, out));
  return 0;
}

}  // namespace acp
