// attention_prefill_tc.cu — causal paged-KV GQA attention for PREFILL steps on the Hopper tensor
// cores: S = Q K^T and O += P V are wgmma warpgroup MMAs with the accumulators in registers.
//
// CTA = 128 query rows x one KV head.  GQA packs the G = heads / kv_heads query heads that share
// the KV head into the rows: row r = (token r / G, head r % G), i.e. 128 / G consecutive new tokens
// of ONE sequence, so every K/V byte staged in shared memory serves G heads.  Keys are walked in
// 64-key tiles (two 32-token pages) from key 0 up to the block's last query position; tile
// boundaries are ABSOLUTE key indices, so a row's arithmetic depends only on its own sequence
// (chunked prefill == single shot, batch invariance).
//
//   warpgroups 0, 1  rows 0..63 / 64..127.  Per tile:
//                S  = Q K_j^T  m64n64k16 x 8   (A = Q, B = K, both from smem, K-major, SW128)
//                softmax in registers (a thread owns 2 rows x 16 keys; row max / sum over the 4-lane quad):
//                causal mask on diagonal tiles, running max with LAZY rescale (O and l are only rescaled
//                when the max grows by more than 2^8; exact, the normaliser carries the same stale max),
//                exp2, P = bf16 hi + bf16 lo (two PV MMAs ~ fp32 P, so no P rounding has to be mirrored
//                by the oracle — same policy as the decode kernels)
//                O += P V_j    m64n128k16 x 4 x 2 (A = P from registers, B = V from smem, MN-major)
//   warp 8      TMA producer: Q tile once (3-D map over qbuf [T][heads][128], box {64, G, 128/G}),
//               then per tile K and V as four {64 dims x 32 tokens} boxes each (page x dim-half),
//               two 2-deep rings with their own full/empty mbarriers; the V tile that holds the sequence's end
//               lands on v_land, the warp zeroes the rows past the end (stale bytes of a recycled page), then
//               completes v_full, so the consumers never see those bytes
// The two warpgroups interleave on the SM: one's MMAs overlap the other's softmax.
//
// Reference boundary: part of the arithmetic behind langchaingo_client.go:102 (DESIGN.md §1).
#include "attention.h"
#include "common.cuh"
#include "gemm.h"

namespace acp {

namespace {

constexpr int PF_ROWS = 128;                     // query rows per CTA
constexpr int PF_KEYS = 64;                      // keys per tile (2 pages)
constexpr int PF_STAGES = 2;
constexpr int PF_Q_BYTES = 2 * PF_ROWS * 128;    // 2 k-blocks (64 dims) of [128 rows][128 B]
constexpr int PF_KT_BYTES = 2 * PF_KEYS * 128;   // 2 dim-halves of [64 keys][128 B] = 16 KiB
constexpr int PF_HALF_BYTES = PF_KEYS * 128;     // 8 KiB
constexpr int PF_PAGE_BYTES = KV_PAGE * 128;     // one {64 x 32} box = 4 KiB
constexpr int PF_THREADS = 288;                  // 2 consumer warpgroups + 1 producer warp
constexpr int PF_SMEM = 1024 + PF_Q_BYTES + 2 * PF_STAGES * PF_KT_BYTES + 256;
constexpr float PF_RESCALE_LOG2 = 8.0f;          // lazy rescale threshold (log2 units)

// two fp32 -> packed bf16x2 (round to nearest even) in ONE conversion instruction; `lo` lands in bits 0..15
ACP_DEVINL uint32_t cvt_bf16x2(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
// 2^x on the SFU without the denormal fix-up sequence (inputs here are <= 8 and -inf maps to +0)
ACP_DEVINL float ex2_ftz(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// P = hi + lo with hi = bf16(p), lo = bf16(p - hi): two PV MMAs carry ~16 mantissa bits of P
ACP_DEVINL void split_hi_lo(float p0, float p1, uint32_t& hi, uint32_t& lo) {
  hi = cvt_bf16x2(p0, p1);
  lo = cvt_bf16x2(p0 - __uint_as_float(hi << 16), p1 - __uint_as_float(hi & 0xffff0000u));
}

ACP_DEVINL void tma_load_3d(void* smem_dst, const void* tmap, uint64_t* bar, int c0, int c1, int c2, uint64_t hint) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4, %5}], [%2], %6;"
      :
      : "r"(smem_u32(smem_dst)), "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "l"(hint)
      : "memory");
}

struct PfBars {
  uint64_t q_full;
  uint64_t v_land;     // the sequence's last V tile landed (v_full follows once its tail is zeroed)
  uint64_t k_full[PF_STAGES], k_empty[PF_STAGES], v_full[PF_STAGES], v_empty[PF_STAGES];
};

__global__ void __launch_bounds__(PF_THREADS, 1)
attn_prefill_tc_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_k,
                       const __grid_constant__ CUtensorMap tm_v, AttnPrefillArgs a, int num_blocks) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint8_t* q_smem = smem;
  uint8_t* k_smem = smem + PF_Q_BYTES;
  uint8_t* v_smem = k_smem + PF_STAGES * PF_KT_BYTES;
  PfBars* bars = (PfBars*)(v_smem + PF_STAGES * PF_KT_BYTES);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // heaviest blocks first: later blocks of a sequence see more keys
  const int blk = num_blocks - 1 - (int)blockIdx.x, kh = blockIdx.y;
  const int G = a.heads / a.kv_heads;
  const int tpb = PF_ROWS / G;                 // query tokens per CTA
  const int b = a.blk_seq[blk];
  const int tq0 = a.blk_tok0[blk];             // first query token (index within the new tokens)
  const int q_len = a.q_len[b], ctx = a.ctx_len[b];
  const int pos0 = ctx - q_len;                // absolute position of new token 0
  const int blk_tokens = min(tpb, q_len - tq0);
  const int last_pos = pos0 + tq0 + blk_tokens - 1;
  const int n_tiles = last_pos / PF_KEYS + 1;

  pdl_launch_dependents();
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_q);
    tma_prefetch_desc(&tm_k);
    tma_prefetch_desc(&tm_v);
    mbar_init(&bars->q_full, 1);
    mbar_init(&bars->v_land, 1);
    for (int s = 0; s < PF_STAGES; ++s) {
      mbar_init(&bars->k_full[s], 1); mbar_init(&bars->k_empty[s], 8);
      mbar_init(&bars->v_full[s], 1); mbar_init(&bars->v_empty[s], 8);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == 8) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      pdl_wait();   // q and the K/V pages of this step come from the previous kernel (rope_kv)
      mbar_arrive_expect_tx(&bars->q_full, PF_Q_BYTES);
      const int row0 = a.q_start[b] + tq0;
      tma_load_3d(q_smem, &tm_q, &bars->q_full, 0, kh * G, row0, kEvictFirst);
      tma_load_3d(q_smem + PF_ROWS * 128, &tm_q, &bars->q_full, 64, kh * G, row0, kEvictFirst);
      const int* pt_row = a.page_table + a.page_off[b];
      const int n_pages = a.page_off[b + 1] - a.page_off[b];
      int jk = 0, jv = 0;
      uint64_t t0 = 0;
      while (jv < n_tiles) {
        bool progressed = false;
        // K runs up to two tiles ahead of the MMAs, V follows K; neither blocks the other
        if (jk < n_tiles && mbar_try_wait(&bars->k_empty[jk % PF_STAGES], (((uint32_t)(jk / PF_STAGES)) & 1u) ^ 1u)) {
          const int s = jk % PF_STAGES;
          mbar_arrive_expect_tx(&bars->k_full[s], PF_KT_BYTES);
          for (int p = 0; p < 2; ++p) {
            const int pi = jk * 2 + p;
            const int page = pi < n_pages ? pt_row[pi] : 0;   // page 0 is the reserved all-zero page
            const int row = (page * a.kv_heads + kh) * 2 * KV_PAGE;
            uint8_t* dst = k_smem + s * PF_KT_BYTES + p * PF_PAGE_BYTES;
            tma_load_2d(dst, &tm_k, &bars->k_full[s], 0, row, kEvictNormal);
            tma_load_2d(dst + PF_HALF_BYTES, &tm_k, &bars->k_full[s], 0, row + KV_PAGE, kEvictNormal);
          }
          ++jk;
          progressed = true;
        }
        if (jv < jk && mbar_try_wait(&bars->v_empty[jv % PF_STAGES], (((uint32_t)(jv / PF_STAGES)) & 1u) ^ 1u)) {
          const int s = jv % PF_STAGES;
          // the tile that holds the sequence's end lands on v_land: the tail below zeroes it, then fills v_full
          uint64_t* bar = (jv * PF_KEYS + PF_KEYS > ctx) ? &bars->v_land : &bars->v_full[s];
          mbar_arrive_expect_tx(bar, PF_KT_BYTES);
          for (int p = 0; p < 2; ++p) {
            const int pi = jv * 2 + p;
            const int page = pi < n_pages ? pt_row[pi] : 0;
            const int row = (page * a.kv_heads + kh) * 2 * KV_PAGE;
            uint8_t* dst = v_smem + s * PF_KT_BYTES + p * PF_PAGE_BYTES;
            tma_load_2d(dst, &tm_v, bar, 0, row, kEvictNormal);
            tma_load_2d(dst + PF_HALF_BYTES, &tm_v, bar, 0, row + KV_PAGE, kEvictNormal);
          }
          ++jv;
          progressed = true;
        }
        // the bound of mbar_wait_mma (no printf: it would serialize the kernel's wgmma)
        if (progressed) t0 = 0;
        else if (t0 == 0) t0 = global_timer_ns();
        else if (global_timer_ns() - t0 > 20000000000ull) __trap();
      }
    }
    __syncwarp();
    const int tile0 = (n_tiles - 1) * PF_KEYS;
    if (tile0 + PF_KEYS > ctx) {
      // The sequence's last tile: its V rows past the end hold whatever the page's previous owner wrote there.
      // Their P is 0, but 0 * NaN = NaN, so the producer warp zeroes them once the tile has landed, makes the
      // stores visible to the async proxy wgmma reads shared memory through, and only then completes v_full.
      const int s = (n_tiles - 1) % PF_STAGES;
      mbar_wait_mma(&bars->v_land, 0);
      uint8_t* vt = v_smem + s * PF_KT_BYTES;
      const int first = ctx - tile0, chunks = (PF_KEYS - first) * 8;   // 16-byte chunks per dim half
      for (int i = lane; i < 2 * chunks; i += 32) {
        const int h = i / chunks, c = i % chunks;
        *reinterpret_cast<uint4*>(vt + h * PF_HALF_BYTES + (first + c / 8) * 128 + (c % 8) * 16) = make_uint4(0, 0, 0, 0);
      }
      fence_proxy_async();
      __syncwarp();
      if (lane == 0) mbar_arrive(&bars->v_full[s]);
    }
  } else {
    // ============ consumer warpgroups: thread owns rows rb and rb + 8, keys 8c + 2(lane % 4) + {0, 1} ============
    const int wg = warp >> 2;
    const int rb = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    int limit[2], tok[2], head[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = rb + 8 * h;
      tok[h] = r / G;
      head[h] = r % G;
      limit[h] = tok[h] < blk_tokens ? pos0 + tq0 + tok[h] + 1 : 0;   // keys with index < limit are visible
    }
    const int first_limit = pos0 + tq0 + 1;        // smallest limit among the valid rows of this CTA
    const float sl2e = a.scale * 1.4426950408889634f;
    pdl_wait();
    float m_run[2] = {-INFINITY, -INFINITY};   // running max, log2 units (score * sl2e); stale by at most PF_RESCALE_LOG2
    float l_run[2] = {0.f, 0.f};               // this thread's share of the row sums
    float o[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) o[i] = 0.f;
    const uint32_t q_addr = smem_u32(q_smem) + (uint32_t)wg * (64 * 128);
    mbar_wait_mma(&bars->q_full, 0);
    for (int j = 0; j < n_tiles; ++j) {
      const int s = j % PF_STAGES;
      const uint32_t par = ((uint32_t)(j / PF_STAGES)) & 1u;
      float sc[32];
      mbar_wait_mma(&bars->k_full[s], par);
      {
        const uint32_t k_addr = smem_u32(k_smem + s * PF_KT_BYTES);
        wgmma_fence();
#pragma unroll
        for (int h = 0; h < 2; ++h) {     // dim halves = 64-wide k-blocks
          const uint64_t a_desc = gmma_desc_k_sw128(q_addr + h * (PF_ROWS * 128));
          const uint64_t b_desc = gmma_desc_k_sw128(k_addr + h * PF_HALF_BYTES);
#pragma unroll
          for (int k = 0; k < 4; ++k)
            wgmma_bf16_ss<PF_KEYS>(sc, a_desc + (uint64_t)(k * 2), b_desc + (uint64_t)(k * 2), (h | k) ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(sc);
      }
      if (lane == 0) mbar_arrive(&bars->k_empty[s]);
      const int tile0 = j * PF_KEYS;
      if (tile0 + PF_KEYS > first_limit) {   // diagonal tile: causal mask (CTA-uniform branch)
#pragma unroll
        for (int i = 0; i < 32; ++i)
          if (tile0 + 8 * (i >> 2) + 2 * (lane & 3) + (i & 1) >= limit[(i >> 1) & 1]) sc[i] = -INFINITY;
      }
      float base[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float mx = -INFINITY;
#pragma unroll
        for (int c = 0; c < 8; ++c) mx = fmaxf(mx, fmaxf(sc[4 * c + 2 * h], sc[4 * c + 2 * h + 1]));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
        const float cand = mx * sl2e;
        // lazy rescale: keep the old base unless the max grew by more than 2^8 (or there was none)
        if (m_run[h] == -INFINITY) {
          m_run[h] = cand;                   // first visible key of this row (O and l are still 0)
        } else if (cand > m_run[h] + PF_RESCALE_LOG2) {
          const float corr = ex2_ftz(m_run[h] - cand);
          m_run[h] = cand;
          l_run[h] *= corr;
#pragma unroll
          for (int c = 0; c < 16; ++c) { o[4 * c + 2 * h] *= corr; o[4 * c + 2 * h + 1] *= corr; }
        }
        base[h] = (m_run[h] == -INFINITY) ? 0.f : m_run[h];
      }
      // P as the A fragments of four k16 MMAs: keys 16kk..16kk+15 = score registers 8kk..8kk+7
      uint32_t ph[16], pl[16];
#pragma unroll
      for (int i = 0; i < 32; i += 2) {
        const int h = (i >> 1) & 1;
        const float p0 = ex2_ftz(fmaf(sc[i], sl2e, -base[h]));
        const float p1 = ex2_ftz(fmaf(sc[i + 1], sl2e, -base[h]));
        l_run[h] += p0 + p1;
        split_hi_lo(p0, p1, ph[i >> 1], pl[i >> 1]);
      }
      mbar_wait_mma(&bars->v_full[s], par);
      {
        const uint32_t v_addr = smem_u32(v_smem + s * PF_KT_BYTES);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < PF_KEYS / 16; ++kk) {   // 16 keys per MMA
          // V tile: [64 keys][64 dims] per dim half, dims contiguous (MN-major): LBO = the next 64 dims,
          // SBO = the next 8 keys
          const uint64_t b_desc = gmma_desc_sw128(v_addr + kk * 16 * 128, PF_HALF_BYTES, 1024);
          const uint32_t fh[4] = {ph[4 * kk], ph[4 * kk + 1], ph[4 * kk + 2], ph[4 * kk + 3]};
          const uint32_t fl[4] = {pl[4 * kk], pl[4 * kk + 1], pl[4 * kk + 2], pl[4 * kk + 3]};
          wgmma_bf16_rs_n128_mn(o, fh, b_desc, 1u);
          wgmma_bf16_rs_n128_mn(o, fl, b_desc, 1u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(o);
      }
      if (lane == 0) mbar_arrive(&bars->v_empty[s]);
    }
    // ---- epilogue: O / l -> bf16 -> global ----
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float l = l_run[h];
      l += __shfl_xor_sync(0xffffffffu, l, 1);
      l += __shfl_xor_sync(0xffffffffu, l, 2);
      if (limit[h] == 0) continue;
      const float inv = 1.0f / l;
      __nv_bfloat16* orow = a.out + ((size_t)(a.q_start[b] + tq0 + tok[h]) * a.heads + (kh * G + head[h])) * HEAD_DIM;
#pragma unroll
      for (int c = 0; c < 16; ++c)
        *reinterpret_cast<uint32_t*>(orow + 8 * c + 2 * (lane & 3)) =
            pack_bf16x2(o[4 * c + 2 * h] * inv, o[4 * c + 2 * h + 1] * inv);
    }
  }
}

}  // namespace

int attn_prefill_tc_setup() {
  if (cudaFuncSetAttribute(attn_prefill_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, PF_SMEM) != cudaSuccess) {
    fprintf(stderr, "[acp_infer] attn_prefill_tc cudaFuncSetAttribute failed\n");
    return -5;
  }
  return 0;
}

int attn_prefill_tc_block_tokens(int heads, int kv_heads) { return PF_ROWS / (heads / kv_heads); }

// K/V of one (page, kv head, dim half): {64 dims x 32 tokens}, 4 KiB, 128-byte swizzle
int attn_make_kv_half_map(CUtensorMap* out, const void* base, uint64_t num_pages, int kv_heads) {
  return tma_encode_2d_bf16(out, base, num_pages * (uint64_t)kv_heads * 2 * KV_PAGE, 64, KV_PAGE);
}

// Q of a step: qbuf [T][heads][128] seen as a 3-D tensor {128 dims, heads, T}; one box =
// {64 dims, G heads of a KV group, 128 / G tokens} = one k-block of the [128 rows][64] A operand
int attn_make_q_map(CUtensorMap* out, const void* qbuf, uint64_t rows, int heads, int kv_heads) {
  const int G = heads / kv_heads;
  if (heads % kv_heads != 0 || G > 128 || (PF_ROWS % G) != 0) return -1;
  return tma_encode_3d_bf16(out, qbuf, HEAD_DIM, (uint64_t)heads, rows, 64, (uint32_t)G, (uint32_t)(PF_ROWS / G));
}

int launch_attn_prefill_tc(const CUtensorMap& tm_q, const CUtensorMap& tm_k, const CUtensorMap& tm_v,
                           const AttnPrefillArgs& a, int num_blocks, cudaStream_t s) {
  if (num_blocks <= 0) return 0;
  const int G = a.heads / a.kv_heads;
  if (a.heads % a.kv_heads != 0 || G > 128 || (PF_ROWS % G) != 0) return -1;
  dim3 grid(num_blocks, a.kv_heads);
  cudaError_t e = acp_launch(attn_prefill_tc_kernel, grid, dim3(PF_THREADS), PF_SMEM, s, tm_q, tm_k, tm_v, a, num_blocks);
  if (e != cudaSuccess) { fprintf(stderr, "[acp_infer] attn_prefill_tc launch: %s\n", cudaGetErrorString(e)); return -5; }
  return 0;
}

}  // namespace acp
