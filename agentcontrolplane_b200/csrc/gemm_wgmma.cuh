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
// Persistent flavour (prefill, N > 256): 2-CTA clusters, one CTA per SM, walk pairs of m-tiles of one
// 256-token n-tile; each CTA loads its own weight tile and half of the activation tile, TMA-multicast to both
// (each CTA reads 32 KiB from L2 per 64-wide k-block instead of 48: W 16 + its X half 16).  For bf16 and
// SwiGLU outputs the consumers only write the finished tile, bf16-rounded, into a whole-tile shared-memory
// staging buffer (stmatrix .trans) and go on to the next tile's MMAs; warps 1-3 of warpgroup 0 (the
// epilogue role) read it back, apply SwiGLU, and store 16-byte row pieces while that mainloop runs.  Both
// flavours accumulate K in the same order and round the same way, so they agree bit for bit.
//
// FP8 flavour (template flag FP8, the `-fp8` presets): W and X hold e4m3 codes, a k-block is still one
// 128-byte swizzle row (now 128 elements) and a tile still 128 rows x 128 B, so the ring is unchanged;
// each k-block issues four m64nBNk32 e4m3 MMAs into a scratch accumulator that is added to the fp32
// accumulator on the CUDA cores once per k-block (DESIGN.md §4: FP8 wgmma keeps fewer accumulator bits
// than fp32).  The epilogue scales by s_w[m] and then s_x[n] before the bf16 / fp32 / SwiGLU store.
// The scratch accumulator doubles the registers, so FP8 tiles are at most 128 tokens wide.
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
  // FP8: per-row weight scales [M] and per-token activation scales (indexed like the activation rows)
  const float* w_scale;
  const float* x_scale;
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
constexpr int GEMM_BK_E4M3 = 128;   // e4m3 elements per k-block (the same 128-byte swizzle row)
constexpr int PGEMM_BN_E4M3 = 128;
constexpr int PGEMM_EPI_THREADS = 96;   // the epilogue role of the persistent kernel: warps 1-3 of warpgroup 0
// Persistent kernel, per instantiation: ring depth and the whole-tile staging buffer (128 features x BN tokens
// of bf16, one [token][64 features] half per consumer warpgroup).  The fp32 plane is stored from registers and
// has no buffer.  Dynamic shared memory = ring, barriers (<= 256 B), staging buffer, of the 227 KiB an SM allows:
//   bf16 / SwiGLU  3 x 48 KiB + 64 KiB + 1.25 KiB = 209.25 KiB   (a 4th stage would not fit beside the buffer)
//   FP8            6 x 32 KiB + 32 KiB + 1.25 KiB = 225.25 KiB
//   fp32 plane     the tiled kernel's ring (4 stages bf16, 6 FP8), no buffer
template <int EPI, bool FP8>
constexpr int PGemmStages = (EPI == EPI_F32 || FP8) ? GemmCfg<FP8 ? PGEMM_BN_E4M3 : PGEMM_BN>::kStages : 3;
template <int EPI, bool FP8>
constexpr int PGemmStagingBytes = EPI == EPI_F32 ? 0 : GEMM_BM * (FP8 ? PGEMM_BN_E4M3 : PGEMM_BN) * 2;
template <int EPI, bool FP8>
constexpr int PGemmSmem = PGemmStages<EPI, FP8> * GemmCfg<FP8 ? PGEMM_BN_E4M3 : PGEMM_BN>::kStageBytes + 1024 /*align*/ +
                          256 /*barriers*/ + PGemmStagingBytes<EPI, FP8>;
static_assert(PGemmSmem<EPI_BF16, false> <= 227 * 1024 && PGemmSmem<EPI_SWIGLU, true> <= 227 * 1024, "persistent GEMM smem");

// ---------------------------------------------------------------------------------
// producer: the k-blocks [kb_begin, kb_end) of one tile into the ring (one thread)
// ---------------------------------------------------------------------------------
template <int BN, int STAGES, int BK = GEMM_BK>
__device__ __forceinline__ void gemm_produce(uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar, int& s, uint32_t& ph,
                                             const CUtensorMap* tmap_w, const CUtensorMap* tmap_x, int w_row0, int kb_begin,
                                             int nkb, int x_row, uint64_t w_hint) {
  using Cfg = GemmCfg<BN>;
  for (int kb = 0; kb < nkb; ++kb) {
    mbar_wait_mma(&empty_bar[s], ph ^ 1);
    uint8_t* a_dst = smem + s * Cfg::kStageBytes;
    mbar_arrive_expect_tx(&full_bar[s], Cfg::kStageBytes);
    tma_load_2d(a_dst, tmap_w, &full_bar[s], 0, w_row0 + (kb_begin + kb) * GEMM_BM, w_hint);
    tma_load_2d(a_dst + Cfg::kABytes, tmap_x, &full_bar[s], (kb_begin + kb) * BK, x_row, kEvictLast);
    if (++s == STAGES) { s = 0; ph ^= 1; }
  }
}

// Producer of one CTA of a 2-CTA cluster (persistent kernel): the two CTAs work on m-tiles 2p, 2p+1 of the
// same n-tile.  Each loads its own W tile and half of the X box (BN/2 token rows, `rank` picks the half),
// multicast to both CTAs at the same offset, so every stage still holds W + the whole X tile.  A stage is
// refilled once the consumers of BOTH CTAs have released it (the empty barriers count 16 warps).  `has_w`
// false: the second CTA of a last, odd m-tile has no W tile; it still loads its X half, and expects only X.
template <int BN, int STAGES, int BK>
__device__ __forceinline__ void gemm_produce_pair(uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar, int& s, uint32_t& ph,
                                                  const CUtensorMap* tmap_w, const CUtensorMap* tmap_xh, int w_row0, bool has_w,
                                                  int nkb, int x_row, uint32_t rank) {
  using Cfg = GemmCfg<BN>;
  constexpr int kHalfBytes = Cfg::kBBytes / 2;
  for (int kb = 0; kb < nkb; ++kb) {
    mbar_wait_mma(&empty_bar[s], ph ^ 1);
    uint8_t* a_dst = smem + s * Cfg::kStageBytes;
    mbar_arrive_expect_tx(&full_bar[s], has_w ? Cfg::kStageBytes : Cfg::kBBytes);
    if (has_w) tma_load_2d(a_dst, tmap_w, &full_bar[s], 0, w_row0 + kb * GEMM_BM, kEvictNormal);
    tma_load_2d_multicast(a_dst + Cfg::kABytes + rank * kHalfBytes, tmap_xh, &full_bar[s], kb * BK, x_row + (int)rank * (BN / 2),
                          0x3, kEvictNormal);
    if (++s == STAGES) { s = 0; ph ^= 1; }
  }
}

// A consumer warp releases stage `bar`: its own CTA's empty barrier, and with PAIR also the cluster peer's
// (rank ^ 1), whose producer multicasts into this CTA's stages too.
template <bool PAIR>
__device__ __forceinline__ void gemm_release(uint64_t* bar, uint32_t rank) {
  mbar_arrive(bar);
  if constexpr (PAIR) mbar_arrive_cluster(bar, rank ^ 1u);
}

// ---------------------------------------------------------------------------------
// consumer warpgroup `wg` (0/1): d = W[rows 64*wg ..][k-blocks] x X^T over nkb ring stages.
// Every warp releases a stage once its own MMAs have read it (empty barriers count 8 warps, 16 with PAIR).
// ---------------------------------------------------------------------------------
template <int BN, int STAGES, bool PAIR = false>
__device__ __forceinline__ void gemm_consume(float (&d)[BN / 2], uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar,
                                             int& s, uint32_t& ph, int nkb, int wg, int lane, uint32_t rank = 0) {
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
    if (prev >= 0 && lane == 0) gemm_release<PAIR>(&empty_bar[prev], rank);
    prev = s;
    if (++s == STAGES) { s = 0; ph ^= 1; }
  }
  wgmma_wait<0>();
  wgmma_fence_regs(d);
  if (prev >= 0 && lane == 0) gemm_release<PAIR>(&empty_bar[prev], rank);
}

// FP8 consumer: per k-block, four k32 MMAs into the scratch accumulator t (the first overwrites it), then
// d += t in fp32 once they are done.  The stage is released right after the wait, before the adds.
template <int BN, int STAGES, bool PAIR = false>
__device__ __forceinline__ void gemm_consume_e4m3(float (&d)[BN / 2], uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar,
                                                  int& s, uint32_t& ph, int nkb, int wg, int lane, uint32_t rank = 0) {
  using Cfg = GemmCfg<BN>;
  float t[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) d[i] = 0.f;
  for (int kb = 0; kb < nkb; ++kb) {
    mbar_wait_mma(&full_bar[s], ph);
    const uint32_t a_addr = smem_u32(smem + s * Cfg::kStageBytes) + (uint32_t)wg * (64 * 128);
    const uint64_t a_desc = gmma_desc_k_sw128(a_addr);
    const uint64_t b_desc = gmma_desc_k_sw128(smem_u32(smem + s * Cfg::kStageBytes + Cfg::kABytes));
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < GEMM_BK_E4M3 / 32; ++k)
      // 32 e4m3 = 32 bytes along K per MMA: +2 in the (addr >> 4) field, as for bf16
      wgmma_e4m3_ss<BN>(t, a_desc + (uint64_t)(k * 2), b_desc + (uint64_t)(k * 2), k > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(t);
    if (lane == 0) gemm_release<PAIR>(&empty_bar[s], rank);
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) d[i] += t[i];
    if (++s == STAGES) { s = 0; ph ^= 1; }
  }
}

// FP8 dequantisation in the accumulator layout: d = fp32(fp32(d * s_w[m]) * s_x[n]) (rows / tokens past the
// end are never stored, their scales are not read)
template <int BN>
__device__ __forceinline__ void gemm_scale_e4m3(float (&d)[BN / 2], const GemmArgs& args, int m_base, int n0, int row_off,
                                                int n_valid, int lane) {
  const int mr = m_base + (lane >> 2);
  const int nc = n0 + 2 * (lane & 3);
  const float sw0 = mr < args.M ? args.w_scale[mr] : 0.f;
  const float sw8 = mr + 8 < args.M ? args.w_scale[mr + 8] : 0.f;
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) {
    const int n = nc + 8 * (i >> 2) + (i & 1);
    const float sx = n < n_valid ? args.x_scale[row_off + n] : 0.f;
    d[i] = __fmul_rn(__fmul_rn(d[i], ((i >> 1) & 1) ? sw8 : sw0), sx);
  }
}

// bf16(bf16(silu(g)) * u) of one (gate, up) pair, g and u already bf16-rounded: the one SwiGLU expression of
// both kernels (accurate expf and IEEE division; DESIGN.md §5)
__device__ __forceinline__ uint16_t swiglu_bf16_bits(float g, float u) {
  const float act = bf16_round(g / (1.0f + expf(-g)));
  return f32_to_bf16_bits(act * u);
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
      if (n < n_valid && m < args.M) out[(size_t)n * args.ld + (m >> 1)] = __ushort_as_bfloat16(swiglu_bf16_bits(g, u));
    }
  }
}

// ---------------------------------------------------------------------------------
// persistent-kernel epilogue through shared memory (bf16 and SwiGLU outputs), split in two halves:
//   gemm_stage_tile     consumer warpgroup `wg`: its 64 features x BN tokens of the finished tile, bf16-rounded
//                       (the GEMM's own rounding point: pack_bf16x2), into its half of the staging buffer
//   gemm_epilogue_tile  the epilogue warps: read the tile back, apply SwiGLU, store 16-byte pieces of output rows
// Every value and rounding is the one gemm_store computes; only the way it reaches global memory differs (from
// registers each warp store touches 4-8 rows with 2 bytes per lane).  A half is [token][64 features] rows of
// 128 B whose 16-byte chunk c sits at chunk c ^ (row & 7), so that the stmatrix writes and the 16-byte row reads
// are free of bank conflicts.  W rows are interleaved (gate_j, up_j), so for SwiGLU each staged gate value sits
// next to its up value.
// ---------------------------------------------------------------------------------
// one piece of 8 outputs, columns [col, col + 8) of an output row: one 16-byte store, or element by element
// where the piece runs past the last column (ragged M) or rows are not 16-byte aligned (!vec_ok)
__device__ __forceinline__ void gemm_store_piece(__nv_bfloat16* row, int col, int ncols, bool vec_ok, uint4 v) {
  if (vec_ok && col + 8 <= ncols) {
    *(uint4*)(row + col) = v;
  } else {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int q = 0; q < 8; ++q)
      if (col + q < ncols) row[col + q] = __ushort_as_bfloat16((unsigned short)(w[q >> 1] >> (16 * (q & 1))));
  }
}
// `st` = the warpgroup's half of the buffer, `w4` = warp in the warpgroup (stmatrix .trans turns the [m][n]
// accumulator fragments into [n][m] rows)
template <int BN>
__device__ __forceinline__ void gemm_stage_tile(const float (&d)[BN / 2], uint32_t st, int w4, int lane) {
#pragma unroll
  for (int j = 0; j < BN / 8; j += 2) {
    // matrices (features 8h.., tokens 8j'..) for h = i & 1, j' = j + (i >> 1); this lane addresses token row k
    const int i = lane >> 3, k = lane & 7;
    const int n = 8 * (j + (i >> 1)) + k, c = 2 * w4 + (i & 1);
    stmatrix_x4_trans(st + n * 128 + ((c ^ (n & 7)) << 4), pack_bf16x2(d[4 * j], d[4 * j + 1]),
                      pack_bf16x2(d[4 * j + 2], d[4 * j + 3]), pack_bf16x2(d[4 * j + 4], d[4 * j + 5]),
                      pack_bf16x2(d[4 * j + 6], d[4 * j + 7]));
  }
}
// Tile (features m0 .. m0 + 127, tokens n0 .. n0 + BN - 1) from the buffer at `st`; `et` = epilogue thread (0..95).
// bf16: a token row is 16 pieces (8 per half).  SwiGLU: a piece of 8 outputs is two adjacent staged chunks of
// 4 (gate, up) pairs; threads 4r.. take rows 2r, 2r + 1 so that a phase of 8 lanes reads distinct banks.
template <int BN, int EPI>
__device__ __forceinline__ void gemm_epilogue_tile(const GemmArgs& args, uint32_t st, int m0, int n0, int n_valid, bool vec_ok,
                                                   int et) {
  constexpr uint32_t HALF = BN * 128;
  const int rows = min(BN, n_valid - n0);
  __nv_bfloat16* out = (__nv_bfloat16*)args.out;
  if constexpr (EPI == EPI_BF16) {
    for (int idx = et; idx < rows * 16; idx += PGEMM_EPI_THREADS) {
      const int n = idx >> 4, h = (idx >> 3) & 1, c = idx & 7;
      gemm_store_piece(out + (size_t)(n0 + n) * args.ld, m0 + 64 * h + 8 * c, args.M, vec_ok,
                       lds_v4(st + h * HALF + n * 128 + ((c ^ (n & 7)) << 4)));
    }
  } else {
    static_assert(EPI == EPI_SWIGLU, "bf16 or SwiGLU");
    for (int idx = et; idx < ((rows + 1) & ~1) * 8; idx += PGEMM_EPI_THREADS) {
      const int c = idx & 3, h = (idx >> 3) & 1, n = 2 * (idx >> 4) + ((idx >> 2) & 1);
      if (n >= rows) continue;
      const uint32_t row = st + h * HALF + n * 128;
      const uint4 a = lds_v4(row + (((2 * c) ^ (n & 7)) << 4)), b = lds_v4(row + (((2 * c + 1) ^ (n & 7)) << 4));
      const uint32_t gu[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};   // output 8c + q: gate low, up high half
      uint32_t o[4];
#pragma unroll
      for (int q = 0; q < 4; ++q)
        o[q] = (uint32_t)swiglu_bf16_bits(bf16_lo(gu[2 * q]), bf16_hi(gu[2 * q])) |
               ((uint32_t)swiglu_bf16_bits(bf16_lo(gu[2 * q + 1]), bf16_hi(gu[2 * q + 1])) << 16);
      gemm_store_piece(out + (size_t)(n0 + n) * args.ld, ((m0 + 64 * h) >> 1) + 8 * c, args.M >> 1, vec_ok,
                       make_uint4(o[0], o[1], o[2], o[3]));
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
template <int BN, int EPI, bool FP8 = false>
__global__ void __launch_bounds__(GEMM_THREADS, GemmCfg<BN>::kMinBlocks)
gemm_wx_kernel(const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ CUtensorMap tmap_x,
               GemmArgs args) {
  using Cfg = GemmCfg<BN>;
  constexpr int STAGES = Cfg::kStages;
  constexpr int BK = FP8 ? GEMM_BK_E4M3 : GEMM_BK;
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
  const int nkb_total = (args.K + BK - 1) / BK;
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
                    (kb_begin + kb) * BK, row_off + n0, kEvictLast);
      int s = pre % STAGES;
      uint32_t ph = (pre == STAGES) ? 1u : 0u;
      gemm_produce<BN, STAGES, BK>(smem, full_bar, empty_bar, s, ph, &tmap_w, &tmap_x, w_row0, kb_begin + pre, nkb - pre,
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
    if constexpr (FP8) gemm_consume_e4m3<BN, STAGES>(d, smem, full_bar, empty_bar, s, ph, nkb, wg, lane);
    else gemm_consume<BN, STAGES>(d, smem, full_bar, empty_bar, s, ph, nkb, wg, lane);
    const int m_base = m0 + cw * 16;
    if constexpr (FP8) gemm_scale_e4m3<BN>(d, args, m_base, n0, row_off, n_valid, lane);
    if constexpr (EPI == EPI_ARGMAX) {
      asm volatile("bar.sync 1, 256;" ::: "memory");   // every MMA has read the ring: reuse it
      gemm_store_argmax<BN>(d, args, m_base, n0, n_valid, m_tile, cw, lane, smem);
    } else {
      gemm_store<BN, EPI>(d, args, m_base, n0, row_off, n_valid, split, lane);
    }
  }
}

// Persistent kernel (prefill), launched as 2-CTA clusters: grid = 2 x min(tile pairs, co-resident clusters).
// Pair p = (m-tiles 2(p / n_tiles) and 2(p / n_tiles) + 1, n-tile p % n_tiles), n-tile fastest (clusters
// running together share weight tiles; X stays in L2); cluster CTA `rank` takes m-tile 2(p / n_tiles) + rank.
// Both CTAs walk the same pairs in lockstep, so their rings advance stage for stage: each loads its own W
// tile and multicasts half of the X tile to both (`tmap_xh`: a box of BN/2 token rows; gemm_produce_pair).
// bf16, SwiGLU or one fp32 plane.
// Roles: thread 0 is the producer; warps 1-3 (bf16 and SwiGLU) are the epilogue role, which stores tile t from the
// staging buffer while the consumer warpgroups (warps 4-11) run tile t + 1's MMAs.  Two mbarriers hand the buffer
// back and forth: `staged` (256 consumer threads arrive once the tile is written) and `released` (96 epilogue
// threads arrive once it is read).  The fp32 plane is stored by the consumers from registers.
template <int EPI, bool FP8 = false>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_wx_persistent_kernel(const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ CUtensorMap tmap_xh,
                          GemmArgs args, int m_tiles, int n_tiles) {
  constexpr int BN = FP8 ? PGEMM_BN_E4M3 : PGEMM_BN;
  using Cfg = GemmCfg<BN>;
  constexpr int STAGES = PGemmStages<EPI, FP8>;
  constexpr int BK = FP8 ? GEMM_BK_E4M3 : GEMM_BK;
  constexpr bool STAGED = EPI != EPI_F32;
  extern __shared__ uint8_t smem_raw[];
  // the same alignment in both CTAs of the cluster (the dynamic shared window starts at the same offset), so
  // a multicast box lands at the same offset of the ring in each
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint64_t* full_bar = (uint64_t*)(smem + STAGES * Cfg::kStageBytes);
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* staged_bar = empty_bar + STAGES;
  uint64_t* released_bar = staged_bar + 1;
  const uint32_t staging = smem_u32(smem + STAGES * Cfg::kStageBytes + 256);   // PGemmSmem: past the barriers

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const uint32_t rank = cluster_ctarank();
  const int cluster = (int)blockIdx.x >> 1, clusters = (int)gridDim.x >> 1;
  const int nkb = (args.K + BK - 1) / BK;
  const int num_pairs = ((m_tiles + 1) >> 1) * n_tiles;
  // 16-byte stores need output rows that start 16-byte aligned
  const bool vec_ok = args.ld % 8 == 0 && ((uintptr_t)args.out & 15) == 0;

  pdl_launch_dependents();
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_w);
    tma_prefetch_desc(&tmap_xh);
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 16); }
    mbar_init(staged_bar, 256);
    mbar_init(released_bar, PGEMM_EPI_THREADS);
    fence_mbar_init();
  }
  cluster_sync_relaxed();   // both CTAs' barriers are initialised before either multicasts or arrives on them

  int s = 0;
  uint32_t ph = 0;
  if (warp < 4) {
    if (threadIdx.x == 0) {
      pdl_wait();  // activations come from the previous kernel
      for (int p = cluster; p < num_pairs; p += clusters) {
        const int m_tile = 2 * (p / n_tiles) + (int)rank;
        gemm_produce_pair<BN, STAGES, BK>(smem, full_bar, empty_bar, s, ph, &tmap_w, &tmap_xh, m_tile * nkb * GEMM_BM,
                                          m_tile < m_tiles, nkb, (p % n_tiles) * BN, rank);
      }
    } else if constexpr (STAGED) {
      if (warp > 0) {
        // ===== epilogue role: the tiles with a W tile, in the consumers' order =====
        pdl_wait();   // the previous kernel may still read the output buffer
        const int n_valid = args.n_dev ? *args.n_dev : args.N;
        uint32_t eph = 0;
        for (int p = cluster; p < num_pairs; p += clusters) {
          const int m_tile = 2 * (p / n_tiles) + (int)rank;
          if (m_tile >= m_tiles) continue;
          mbar_wait_mma(staged_bar, eph);
          gemm_epilogue_tile<BN, EPI>(args, staging, m_tile * GEMM_BM, (p % n_tiles) * BN, n_valid, vec_ok, threadIdx.x - 32);
          mbar_arrive(released_bar);
          eph ^= 1;
        }
      }
    }
  } else {
    const int wg = (warp >> 2) - 1, cw = warp - 4;
    pdl_wait();
    const int n_valid = args.n_dev ? *args.n_dev : args.N;
    uint32_t eph = 0;   // parity of the staging-buffer hand-over
    for (int p = cluster; p < num_pairs; p += clusters) {
      const int m_tile = 2 * (p / n_tiles) + (int)rank, m_base = m_tile * GEMM_BM + cw * 16, n0 = (p % n_tiles) * BN;
      float d[BN / 2];
      // a CTA without a W tile still consumes (and releases) every stage: its peer's X half needs the slot
      if constexpr (FP8) gemm_consume_e4m3<BN, STAGES, true>(d, smem, full_bar, empty_bar, s, ph, nkb, wg, lane, rank);
      else gemm_consume<BN, STAGES, true>(d, smem, full_bar, empty_bar, s, ph, nkb, wg, lane, rank);
      if (m_tile < m_tiles) {
        if constexpr (FP8) gemm_scale_e4m3<BN>(d, args, m_base, n0, 0, n_valid, lane);
        if constexpr (STAGED) {
          mbar_wait_mma(released_bar, eph ^ 1);   // the epilogue warps have read the previous tile
          gemm_stage_tile<BN>(d, staging + wg * (BN * 128), cw & 3, lane);
          mbar_arrive(staged_bar);
          eph ^= 1;
        } else {
          gemm_store<BN, EPI>(d, args, m_base, n0, 0, n_valid, 0, lane);   // the fp32 plane, from registers
        }
      }
    }
  }
  cluster_sync();   // no CTA exits while its peer may still multicast into it or arrive on its barriers
}

}  // namespace acp
