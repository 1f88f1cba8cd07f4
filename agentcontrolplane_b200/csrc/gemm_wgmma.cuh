// gemm_wgmma.cuh — the one dense-contraction kernel family of the decode engine.
//
//   out[n][m] = sum_k W[m][k] * X[n][k]          (W: [M][K] bf16 stored as contiguous 128x64 tiles,
//                                                 X: [N][K] bf16 row-major; both K-major operands)
//
// "Swap-AB" orientation: the WEIGHT matrix is the wgmma A operand (128 output features per tile,
// 64 per consumer warpgroup) and the ACTIVATIONS are the B operand (N = sequences/tokens, 16..256
// per tile).  Decode batches (N = 16..256 live sequences) therefore keep the M=64 MMAs full while
// streaming every weight byte exactly once from HBM; prefill uses 256-token N tiles.
//
// Pipeline (warp-specialised, three warpgroups):
//   warpgroup 0   TMA producer (one thread): cp.async.bulk.tensor.2d W-tile {64 x 128} + X-tile
//                 {64 x BN}, 128-byte swizzle, into a STAGES-deep shared-memory ring (full/empty mbarriers)
//   warpgroups 1, 2  consumers: wgmma m64nBNk16 over weight rows 0..63 / 64..127 of the tile, fp32
//                 accumulators in registers, then the epilogue straight from those registers:
//                 bf16 / fp32-partial / fused SwiGLU / fused arg-max store
//
// Split-K: grid.z splits the k-block range; partials are written as fp32 [split][N][M] and are
// summed IN FIXED ORDER by the consumer kernel (rope / add+rmsnorm / swiglu), which keeps the
// result bit-reproducible run to run (no atomics).
//
// Persistent flavour (prefill, N > 256): one CTA per SM walks (m-tile, 256-token n-tile) tiles; the
// producer streams the next tile's stages while the consumers run the previous tile's epilogue.
// Both flavours accumulate K in the same order, so they agree bit for bit.
//
// Reference boundary: this replaces the remote model behind
// acp/internal/llmclient/langchaingo_client.go:102 (GenerateContent); see DESIGN.md.
#pragma once
#include "common.cuh"
#include <cuda.h>

namespace acp {

constexpr int GEMM_BM = 128;  // weight rows per tile (two m64 warpgroup MMAs)
constexpr int GEMM_BK = 64;   // bf16 elements per k-block (= one 128-byte swizzle row)
constexpr int GEMM_THREADS = 384;
constexpr int GEMM_SMS = 132;  // H100 SXM: one persistent CTA per SM
// grouped mode: layout of the device-side `group_ranges` array (written by moe_dispatch_kernel):
//   [2g], [2g+1]                    first row and row count of group g            (g < GEMM_GROUP_MAX)
//   [GEMM_GROUP_TILES]              number of entries of the flat tile list
//   [GEMM_GROUP_TILES + 2 + 2i ..]  tile i = {group, first row inside the group}
constexpr int GEMM_GROUP_MAX = 16;
constexpr int GEMM_GROUP_TILES = 2 * GEMM_GROUP_MAX;

enum GemmEpi : int {
  EPI_BF16 = 0,     // out_bf16[n*ld + m]
  EPI_F32 = 1,      // out_f32[(split*n_cap + n)*ld + m]      (split-K partials, logits)
  EPI_ARGMAX = 2,   // per (n, m-tile): max value + lowest index; optional fp32 logits
  EPI_SWIGLU = 3,   // rows interleaved (gate_j, up_j): out_bf16[n*ld + m/2] = bf16(bf16(silu(g))*u)
};

struct GemmArgs {
  int M;         // rows of W (output features)
  int N;         // valid activation rows
  int K;
  int splits;    // == gridDim.z
  int ld;        // output leading dimension (elements)
  int n_cap;     // row capacity of one split-K partial plane
  void* out;     // bf16* or float* (may be null for EPI_ARGMAX)
  float* amax_val;   // EPI_ARGMAX: [N][m_tiles]
  int* amax_idx;     // EPI_ARGMAX: [N][m_tiles]
  const int* n_dev;  // optional device scalar overriding N (CUDA-graph replay with varying batch)
  // GROUPED mode (mixture of experts): group g's weights are m-tiles [g*gridDim.y, (g+1)*gridDim.y) of the
  // (concatenated) weight tensor, its activation / output rows are [ranges[2g], ranges[2g] + ranges[2g+1]).
  // blockIdx.x indexes a flat tile list {group, first row inside the group} (layout: GEMM_GROUP_TILES above)
  // — all written on the device by moe_dispatch_kernel, so row counts never visit the host and
  // no CTA is launched for rows that do not exist (beyond the <= E slack of the grid bound).  splits must be 1.
  const int* group_ranges;
};

template <int BN>
struct GemmCfg {
  // decode tiles (BN <= 64) keep two CTAs per SM (2 x <= 97 KiB); wide tiles fill one SM's 227 KiB
  static constexpr int kStages = (BN <= 64) ? 4 : (BN == 128 ? 6 : 4);
  static constexpr int kMinBlocks = (BN <= 64) ? 2 : 1;
  static constexpr int kABytes = GEMM_BM * GEMM_BK * 2;  // 16 KiB
  static constexpr int kBBytes = BN * GEMM_BK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kSmemBytes = kStages * kStageBytes + 1024 /*align*/ + 256 /*barriers*/;
};
constexpr int PGEMM_BN = 256;
using PGemmCfg = GemmCfg<PGEMM_BN>;

// ---------------------------------------------------------------------------------
// producer: the k-blocks [kb_begin, kb_end) of one tile into the ring (one thread)
// ---------------------------------------------------------------------------------
template <int BN, int STAGES>
__device__ __forceinline__ void gemm_produce(uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar, int& s, uint32_t& ph,
                                             const CUtensorMap* tmap_w, const CUtensorMap* tmap_x, int w_row0, int kb_begin,
                                             int nkb, int x_row, uint64_t w_hint) {
  using Cfg = GemmCfg<BN>;
  for (int kb = 0; kb < nkb; ++kb) {
    mbar_wait_mma(&empty_bar[s], ph ^ 1);
    uint8_t* a_dst = smem + s * Cfg::kStageBytes;
    mbar_arrive_expect_tx(&full_bar[s], Cfg::kStageBytes);
    tma_load_2d(a_dst, tmap_w, &full_bar[s], 0, w_row0 + (kb_begin + kb) * GEMM_BM, w_hint);
    tma_load_2d(a_dst + Cfg::kABytes, tmap_x, &full_bar[s], (kb_begin + kb) * GEMM_BK, x_row, kEvictLast);
    if (++s == STAGES) { s = 0; ph ^= 1; }
  }
}

// ---------------------------------------------------------------------------------
// consumer warpgroup `wg` (0/1): d = W[rows 64*wg ..][k-blocks] x X^T over nkb ring stages.
// Every warp releases a stage once its own MMAs have read it (empty barriers count 8 warps).
// ---------------------------------------------------------------------------------
template <int BN, int STAGES>
__device__ __forceinline__ void gemm_consume(float (&d)[BN / 2], uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar,
                                             int& s, uint32_t& ph, int nkb, int wg, int lane) {
  using Cfg = GemmCfg<BN>;
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) d[i] = 0.f;
  int prev = -1;
  for (int kb = 0; kb < nkb; ++kb) {
    mbar_wait_mma(&full_bar[s], ph);
    const uint32_t a_addr = smem_u32(smem + s * Cfg::kStageBytes) + (uint32_t)wg * (64 * 128);
    const uint64_t a_desc = gmma_desc_k_sw128(a_addr);
    const uint64_t b_desc = gmma_desc_k_sw128(smem_u32(smem + s * Cfg::kStageBytes + Cfg::kABytes));
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < GEMM_BK / 16; ++k)
      // advancing 16 bf16 (32 bytes) along K inside the swizzle atom = +2 in the (addr >> 4) field
      wgmma_bf16_ss<BN>(d, a_desc + (uint64_t)(k * 2), b_desc + (uint64_t)(k * 2), (kb > 0 || k > 0) ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<1>();   // the MMAs of the previous stage are done: release it
    if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
    prev = s;
    if (++s == STAGES) { s = 0; ph ^= 1; }
  }
  wgmma_wait<0>();
  wgmma_fence_regs(d);
  if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
}

// ---------------------------------------------------------------------------------
// epilogue from the accumulator registers (layout: common.cuh, above wgmma_bf16_ss).
//   row m = m_base + l/4 + 8h (m_base = m0 + 64*wg + 16*warp), column n = n0 + 8j + 2(l%4) + e,
//   value d[4j + 2h + e].
// ---------------------------------------------------------------------------------
template <int BN, int EPI>
__device__ __forceinline__ void gemm_store(const float (&d)[BN / 2], const GemmArgs& args, int m_base, int n0, int row_off,
                                           int n_valid, int split, int lane) {
  const int mr = m_base + (lane >> 2);
  const int nc = n0 + 2 * (lane & 3);
  if constexpr (EPI == EPI_BF16) {
    __nv_bfloat16* out = (__nv_bfloat16*)args.out;
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) {
      const int m = mr + 8 * ((i >> 1) & 1), n = nc + 8 * (i >> 2) + (i & 1);
      if (n < n_valid && m < args.M) out[(size_t)(row_off + n) * args.ld + m] = __float2bfloat16_rn(d[i]);
    }
  } else if constexpr (EPI == EPI_F32) {
    float* out = (float*)args.out;
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) {
      const int m = mr + 8 * ((i >> 1) & 1), n = nc + 8 * (i >> 2) + (i & 1);
      if (n < n_valid && m < args.M) out[((size_t)split * args.n_cap + n) * args.ld + m] = d[i];
    }
  } else if constexpr (EPI == EPI_SWIGLU) {
    // W rows are stored interleaved: even row = gate_j, odd row = up_j (j = row / 2), so the pair of one
    // output sits in lanes l and l ^ 4.  The two lanes split the two tokens they both hold: the gate lane
    // finishes the first, the up lane the second, so one exchange serves two outputs.
    __nv_bfloat16* out = (__nv_bfloat16*)args.out + (size_t)row_off * args.ld;
    const bool odd = (lane >> 2) & 1;
#pragma unroll
    for (int i = 0; i < BN / 2; i += 2) {
      const float mine0 = bf16_round(d[i]);       // the GEMM's bf16 rounding point
      const float mine1 = bf16_round(d[i + 1]);
      const float got = __shfl_xor_sync(0xffffffffu, odd ? mine0 : mine1, 4);
      const float g = odd ? got : mine0;     // up lane: partner's gate of the second token
      const float u = odd ? mine1 : got;     // gate lane: partner's up of the first token
      const int m = mr + 8 * ((i >> 1) & 1), n = nc + 8 * (i >> 2) + (odd ? 1 : 0);
      if (n < n_valid && m < args.M) {
        const float act = bf16_round(g / (1.0f + expf(-g)));
        out[(size_t)n * args.ld + (m >> 1)] = __float2bfloat16_rn(act * u);
      }
    }
  }
}

// arg-max over the 128 rows of the tile for every column, lowest index on ties (deterministic);
// `red` = 8 warps x BN candidates (value, index) in shared memory no MMA reads any more.
template <int BN>
__device__ __forceinline__ void gemm_store_argmax(const float (&d)[BN / 2], const GemmArgs& args, int m_base, int n0,
                                                  int n_valid, int m_tile, int cw, int lane, uint8_t* red) {
  float* red_v = (float*)red;
  int* red_i = (int*)(red + 8 * BN * sizeof(float));
  float* out = (float*)args.out;
  const int mr = m_base + (lane >> 2);
#pragma unroll
  for (int i = 0; i < BN / 2; i += 4) {
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int n = n0 + 8 * (i >> 2) + 2 * (lane & 3) + e;
      float v = mr < args.M ? d[i + e] : -INFINITY;
      int idx = mr;
      const float v8 = mr + 8 < args.M ? d[i + 2 + e] : -INFINITY;
      if (out != nullptr && n < n_valid) {
        if (mr < args.M) out[(size_t)n * args.ld + mr] = d[i + e];
        if (mr + 8 < args.M) out[(size_t)n * args.ld + mr + 8] = d[i + 2 + e];
      }
      if (v8 > v) { v = v8; idx = mr + 8; }
#pragma unroll
      for (int o = 4; o < 32; o <<= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, v, o);
        const int oi = __shfl_xor_sync(0xffffffffu, idx, o);
        if (ov > v || (ov == v && oi < idx)) { v = ov; idx = oi; }
      }
      if (lane < 4) {
        const int c = 8 * (i >> 2) + 2 * lane + e;
        red_v[cw * BN + c] = v;
        red_i[cw * BN + c] = idx;
      }
    }
  }
  asm volatile("bar.sync 1, 256;" ::: "memory");   // the 8 consumer warps
  const int t = cw * 32 + lane;
  if (t < BN) {
    float v = red_v[t];
    int idx = red_i[t];
#pragma unroll
    for (int w = 1; w < 8; ++w) {
      const float ov = red_v[w * BN + t];
      const int oi = red_i[w * BN + t];
      if (ov > v || (ov == v && oi < idx)) { v = ov; idx = oi; }
    }
    const int n = n0 + t;
    if (n < n_valid) {
      args.amax_val[(size_t)n * gridDim.y + m_tile] = v;
      args.amax_idx[(size_t)n * gridDim.y + m_tile] = idx;
    }
  }
}

// Tiled kernel: one CTA per (n-tile, m-tile, k-split).
template <int BN, int EPI>
__global__ void __launch_bounds__(GEMM_THREADS, GemmCfg<BN>::kMinBlocks)
gemm_wx_kernel(const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ CUtensorMap tmap_x,
               GemmArgs args) {
  using Cfg = GemmCfg<BN>;
  constexpr int STAGES = Cfg::kStages;
  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment is required by the 128B swizzle atom (8 rows x 128 B).
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint64_t* full_bar = (uint64_t*)(smem + STAGES * Cfg::kStageBytes);
  uint64_t* empty_bar = full_bar + STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  // blockIdx.x = n-tile (fastest): the CTAs that run together share ONE weight tile and sweep the
  // activation rows, so W streams from HBM once and X is served by L2.
  int n0 = blockIdx.x * BN;
  const int m0 = blockIdx.y * GEMM_BM;
  const int m_tiles = gridDim.y;
  const bool grouped = args.group_ranges != nullptr;
  int m_tile = blockIdx.y;            // weight m-tile (global index over all groups)
  int split = blockIdx.z;
  int row_off = 0, group_rows = 0;
  pdl_launch_dependents();
  if (grouped) {
    pdl_wait();                        // the ranges come from the previous kernel (moe_dispatch)
    if ((int)blockIdx.x >= args.group_ranges[GEMM_GROUP_TILES]) return;   // whole CTA, before any barrier
    const int group = args.group_ranges[GEMM_GROUP_TILES + 2 + 2 * blockIdx.x];
    n0 = args.group_ranges[GEMM_GROUP_TILES + 2 + 2 * blockIdx.x + 1];
    row_off = args.group_ranges[2 * group];
    group_rows = args.group_ranges[2 * group + 1];
    m_tile = group * m_tiles + (int)blockIdx.y;
    split = 0;
  }
  const int nkb_total = (args.K + GEMM_BK - 1) / GEMM_BK;
  const int kb_begin = (int)(((long long)nkb_total * split) / args.splits);
  const int kb_end = (int)(((long long)nkb_total * (split + 1)) / args.splits);
  const int nkb = kb_end - kb_begin;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_w);
    tma_prefetch_desc(&tmap_x);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp < 4) {
    // ===== TMA producer =====
    if (threadIdx.x == 0) {
      // Phase A: the first ring-full of WEIGHT tiles does not depend on the previous kernel, so
      // it is issued before the grid-dependency wait (hides the HBM ramp under that kernel's tail).
      const int pre = nkb < STAGES ? nkb : STAGES;
      const int w_row0 = m_tile * nkb_total * GEMM_BM;
      for (int kb = 0; kb < pre; ++kb) {
        mbar_arrive_expect_tx(&full_bar[kb], Cfg::kStageBytes);
        // weights are read once per step: evict-first (one contiguous 16 KiB tile)
        tma_load_2d(smem + kb * Cfg::kStageBytes, &tmap_w, &full_bar[kb], 0, w_row0 + (kb_begin + kb) * GEMM_BM, kEvictFirst);
      }
      pdl_wait();  // activations come from the previous kernel
      // activations are re-read by every m-tile: evict-last
      for (int kb = 0; kb < pre; ++kb)
        tma_load_2d(smem + kb * Cfg::kStageBytes + Cfg::kABytes, &tmap_x, &full_bar[kb],
                    (kb_begin + kb) * GEMM_BK, row_off + n0, kEvictLast);
      int s = pre % STAGES;
      uint32_t ph = (pre == STAGES) ? 1u : 0u;
      gemm_produce<BN, STAGES>(smem, full_bar, empty_bar, s, ph, &tmap_w, &tmap_x, w_row0, kb_begin + pre, nkb - pre,
                               row_off + n0, kEvictFirst);
    }
  } else {
    // ===== consumer warpgroups 1, 2 =====
    const int wg = (warp >> 2) - 1, cw = warp - 4;
    pdl_wait();  // outputs may still be read by the previous kernels until they complete
    const int n_valid = grouped ? group_rows : (args.n_dev ? *args.n_dev : args.N);
    float d[BN / 2];
    int s = 0;
    uint32_t ph = 0;
    gemm_consume<BN, STAGES>(d, smem, full_bar, empty_bar, s, ph, nkb, wg, lane);
    const int m_base = m0 + cw * 16;
    if constexpr (EPI == EPI_ARGMAX) {
      asm volatile("bar.sync 1, 256;" ::: "memory");   // every MMA has read the ring: reuse it
      gemm_store_argmax<BN>(d, args, m_base, n0, n_valid, m_tile, cw, lane, smem);
    } else {
      gemm_store<BN, EPI>(d, args, m_base, n0, row_off, n_valid, split, lane);
    }
  }
}

// Persistent kernel (prefill): grid = min(tiles, SMs); tile t = (m-tile t / n_tiles, n-tile t % n_tiles),
// n-tile fastest (CTAs running together share a weight tile; X stays in L2).  bf16, SwiGLU or one fp32 plane.
template <int EPI>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_wx_persistent_kernel(const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ CUtensorMap tmap_x,
                          GemmArgs args, int m_tiles, int n_tiles) {
  constexpr int BN = PGEMM_BN;
  constexpr int STAGES = PGemmCfg::kStages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint64_t* full_bar = (uint64_t*)(smem + STAGES * PGemmCfg::kStageBytes);
  uint64_t* empty_bar = full_bar + STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int nkb = (args.K + GEMM_BK - 1) / GEMM_BK;
  const int num_tiles = m_tiles * n_tiles;

  pdl_launch_dependents();
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_w);
    tma_prefetch_desc(&tmap_x);
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 8); }
    fence_mbar_init();
  }
  __syncthreads();

  int s = 0;
  uint32_t ph = 0;
  if (warp < 4) {
    if (threadIdx.x == 0) {
      pdl_wait();  // activations come from the previous kernel
      for (int t = blockIdx.x; t < num_tiles; t += gridDim.x)
        gemm_produce<BN, STAGES>(smem, full_bar, empty_bar, s, ph, &tmap_w, &tmap_x, (t / n_tiles) * nkb * GEMM_BM, 0, nkb,
                                 (t % n_tiles) * BN, kEvictNormal);
    }
  } else {
    const int wg = (warp >> 2) - 1, cw = warp - 4;
    pdl_wait();
    const int n_valid = args.n_dev ? *args.n_dev : args.N;
    for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
      float d[BN / 2];
      gemm_consume<BN, STAGES>(d, smem, full_bar, empty_bar, s, ph, nkb, wg, lane);
      gemm_store<BN, EPI>(d, args, (t / n_tiles) * GEMM_BM + cw * 16, (t % n_tiles) * BN, 0, n_valid, 0, lane);
    }
  }
}

}  // namespace acp
