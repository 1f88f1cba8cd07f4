// attention.cu — paged-KV GQA attention for the decode engine (decode + causal prefill).
//
// KV cache layout per layer:  K, V : [num_pages][kv_heads][2 dim-halves][KV_PAGE=32][64] bf16: the
// block of one (page, kv head) is 8 KiB CONTIGUOUS.  Seen by TMA as a 2-D tensor
// [num_pages*kv_heads*64 rows][64 cols]; one box {64 cols x 64 rows} with the 128-byte swizzle
// fetches the whole block, which lands in shared memory as two [32 rows][128 B] halves with
// 16-byte chunks XOR-ed by (row & 7): ldmatrix reads are bank-conflict free with no padding.
//
// A CTA stages 64-token tiles (2 pages: K 16 KiB + V 16 KiB per stage) through a 3-deep ring
// filled by a dedicated producer warp (cp.async.bulk.tensor + mbarrier complete_tx); consumer
// warps run mma.sync m16n8k16 (bf16 in, fp32 accumulate) with an online softmax:
//   rows of the 16-row MMA tile = (query token, head-in-group); GQA packs the G query heads that
//   share one KV head into one tile, so K/V bytes are read once per KV head.
//   P is split into bf16 hi + lo parts (two PV MMAs) so that P keeps ~16 mantissa bits: the
//   result matches an fp32-softmax oracle to ~1e-6 and no bf16 rounding of P needs mirroring.
//
// decode  : CTA = (sequence, kv head[, chunk of 1024 tokens]); the 4 consumer warps each take a
//           16-token slice of every tile.  Short contexts: one CTA per item, warps merged in shared
//           memory, output written directly.  Long contexts: fixed 1024-token chunks (boundaries
//           depend only on the sequence itself => batch invariant), per-warp partial (m, l, O) to
//           a workspace, attn_merge_kernel combines them in fixed order.
// prefill : CTA = (16/G*4 query tokens of one sequence, kv head); every warp owns 16 rows
//           (16/G tokens x G heads) and all warps walk the causal range of tiles together.
//
// This is HBM/L2-bound byte movement (4..8 useful rows per MMA): tensor-core use here is only to
// keep the issue slots free, the roofline is bytes of K/V per second (DESIGN.md §4).
#include "attention.h"
#include "common.cuh"
#include "gemm.h"
#include "gemm_out.cuh"

namespace acp {

namespace {

constexpr int TILE_TOK = 64;                 // tokens per staged tile (2 pages)
constexpr int BLOCK_BYTES = KV_PAGE * 128;   // one {64 cols x 32 rows} box = 4 KiB
constexpr int K_TILE_BYTES = 4 * BLOCK_BYTES;  // 2 pages x 2 halves
constexpr int STAGE_BYTES = 2 * K_TILE_BYTES;  // K + V = 32 KiB
constexpr int STAGES = 3;
constexpr int CONSUMER_WARPS = 4;
constexpr int ATTN_THREADS = (CONSUMER_WARPS + 1) * 32;

ACP_DEVINL void mma_bf16_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
      "{%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
ACP_DEVINL void ldmatrix_x4(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}
ACP_DEVINL void ldmatrix_x4_trans(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}

// byte offset of (token-in-tile, dim) inside a staged K or V tile
ACP_DEVINL uint32_t tile_off(int tok, int dim) {
  const int page = tok >> 5, r = tok & 31, hf = dim >> 6, c = (dim & 63) >> 3;
  return (uint32_t)((page * 2 + hf) * BLOCK_BYTES + r * 128 + ((c ^ (r & 7)) << 4));
}

struct WarpState {
  float o[16][4];   // 16 dim-tiles of 8: c0,c1 -> row lane/4 ; c2,c3 -> row lane/4+8
  float m[2];       // running max (raw score units) for the two rows of this thread
  float l[2];       // per-thread partial row sums
};

// One 64-token tile for one warp.  key_limit[r] = number of visible keys for row r (keys with
// absolute index < key_limit are visible), tile_tok0 = absolute index of the tile's first key.
// NT = number of 8-token n-tiles this warp handles, starting at token `tok_off` of the tile
// (prefill: NT = 8, the whole tile; decode: NT = 2, the warp's 16-token slice).
template <int NT>
ACP_DEVINL void process_tile(WarpState& st, const uint32_t (&qf)[8][4], uint32_t k_base,
                             uint32_t v_base, int tile_tok0, int tok_off, int key_limit_lo,
                             int key_limit_hi, float sl2e, int lane) {
  float s[NT][4];
#pragma unroll
  for (int j = 0; j < NT; ++j) { s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f; }
  const int mi = lane >> 3, rr = lane & 7;
  // ---- S = Q K^T ----
#pragma unroll
  for (int j = 0; j < NT; ++j) {         // key n-tiles of 8 tokens
#pragma unroll
    for (int kp = 0; kp < 4; ++kp) {     // 4 pairs of k-steps (32 dims each)
      uint32_t b[4];
      ldmatrix_x4(b, k_base + tile_off(tok_off + j * 8 + rr, kp * 32 + mi * 8));
      mma_bf16_16816(s[j], qf[kp * 2], b[0], b[1]);
      mma_bf16_16816(s[j], qf[kp * 2 + 1], b[2], b[3]);
    }
  }
  // ---- mask + online softmax ----
  float mx_lo = -INFINITY, mx_hi = -INFINITY;
#pragma unroll
  for (int j = 0; j < NT; ++j) {
    const int t0 = tile_tok0 + tok_off + j * 8 + 2 * (lane & 3);
    if (t0 >= key_limit_lo) s[j][0] = -INFINITY;
    if (t0 + 1 >= key_limit_lo) s[j][1] = -INFINITY;
    if (t0 >= key_limit_hi) s[j][2] = -INFINITY;
    if (t0 + 1 >= key_limit_hi) s[j][3] = -INFINITY;
    mx_lo = fmaxf(mx_lo, fmaxf(s[j][0], s[j][1]));
    mx_hi = fmaxf(mx_hi, fmaxf(s[j][2], s[j][3]));
  }
  mx_lo = fmaxf(mx_lo, __shfl_xor_sync(0xffffffffu, mx_lo, 1));
  mx_lo = fmaxf(mx_lo, __shfl_xor_sync(0xffffffffu, mx_lo, 2));
  mx_hi = fmaxf(mx_hi, __shfl_xor_sync(0xffffffffu, mx_hi, 1));
  mx_hi = fmaxf(mx_hi, __shfl_xor_sync(0xffffffffu, mx_hi, 2));
  const float mn_lo = fmaxf(st.m[0], mx_lo), mn_hi = fmaxf(st.m[1], mx_hi);
  // rows with nothing visible yet keep m = -inf; use 0 as the exponent base there (all p = 0)
  const float base_lo = (mn_lo == -INFINITY) ? 0.f : mn_lo * sl2e;
  const float base_hi = (mn_hi == -INFINITY) ? 0.f : mn_hi * sl2e;
  const float corr_lo = (st.m[0] == -INFINITY) ? 0.f : exp2f(st.m[0] * sl2e - base_lo);
  const float corr_hi = (st.m[1] == -INFINITY) ? 0.f : exp2f(st.m[1] * sl2e - base_hi);
  st.m[0] = mn_lo; st.m[1] = mn_hi;
  st.l[0] *= corr_lo; st.l[1] *= corr_hi;
#pragma unroll
  for (int d = 0; d < 16; ++d) {
    st.o[d][0] *= corr_lo; st.o[d][1] *= corr_lo;
    st.o[d][2] *= corr_hi; st.o[d][3] *= corr_hi;
  }
  uint32_t p_hi[NT / 2][4], p_lo[NT / 2][4];  // A fragments for the PV k-steps (16 tokens each)
#pragma unroll
  for (int j = 0; j < NT; ++j) {
    float p[4];
    p[0] = exp2f(s[j][0] * sl2e - base_lo);
    p[1] = exp2f(s[j][1] * sl2e - base_lo);
    p[2] = exp2f(s[j][2] * sl2e - base_hi);
    p[3] = exp2f(s[j][3] * sl2e - base_hi);
    st.l[0] += p[0] + p[1];
    st.l[1] += p[2] + p[3];
    float h[4], lo[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) { h[e] = bf16_round(p[e]); lo[e] = p[e] - h[e]; }
    const int kt = j >> 1, half = j & 1;
    p_hi[kt][half * 2 + 0] = pack_bf16x2(h[0], h[1]);
    p_hi[kt][half * 2 + 1] = pack_bf16x2(h[2], h[3]);
    p_lo[kt][half * 2 + 0] = pack_bf16x2(lo[0], lo[1]);
    p_lo[kt][half * 2 + 1] = pack_bf16x2(lo[2], lo[3]);
  }
  // ---- O += P V ----
#pragma unroll
  for (int kt = 0; kt < NT / 2; ++kt) {  // 16 tokens per k-step
#pragma unroll
    for (int nd = 0; nd < 8; ++nd) {     // 16 dims per ldmatrix.x4.trans
      uint32_t b[4];
      ldmatrix_x4_trans(b, v_base + tile_off(tok_off + kt * 16 + (mi & 1) * 8 + rr, nd * 16 + (mi >> 1) * 8));
      mma_bf16_16816(st.o[nd * 2], p_hi[kt], b[0], b[1]);
      mma_bf16_16816(st.o[nd * 2], p_lo[kt], b[0], b[1]);
      mma_bf16_16816(st.o[nd * 2 + 1], p_hi[kt], b[2], b[3]);
      mma_bf16_16816(st.o[nd * 2 + 1], p_lo[kt], b[2], b[3]);
    }
  }
}

// V rows of tokens that do not exist yet may hold stale bytes (NaN patterns): zero them so that
// 0 * garbage cannot poison the accumulators.  Called by the consuming warp on a landed tile.
ACP_DEVINL void zero_v_tail(uint8_t* v_tile, int first_invalid_tok, int end_tok, int lane) {
  for (int t = first_invalid_tok; t < end_tok; ++t) {
    const int page = t >> 5, r = t & 31;
    // 2 halves x 128 B per row = 16 uint4; lanes 0..15 write one each
    if (lane < 16) {
      const int hf = lane >> 3, c = lane & 7;
      *reinterpret_cast<uint4*>(v_tile + (page * 2 + hf) * BLOCK_BYTES + r * 128 + c * 16) =
          make_uint4(0, 0, 0, 0);
    }
  }
  __syncwarp();
}

ACP_DEVINL void load_q_frags(uint32_t (&qf)[8][4], const __nv_bfloat16* q_lo,
                             const __nv_bfloat16* q_hi, int lane) {
  const int c = 2 * (lane & 3);
#pragma unroll
  for (int ks = 0; ks < 8; ++ks) {
    qf[ks][0] = q_lo ? *reinterpret_cast<const uint32_t*>(q_lo + ks * 16 + c) : 0u;
    qf[ks][1] = q_hi ? *reinterpret_cast<const uint32_t*>(q_hi + ks * 16 + c) : 0u;
    qf[ks][2] = q_lo ? *reinterpret_cast<const uint32_t*>(q_lo + ks * 16 + 8 + c) : 0u;
    qf[ks][3] = q_hi ? *reinterpret_cast<const uint32_t*>(q_hi + ks * 16 + 8 + c) : 0u;
  }
}

// Producer: stage tiles [tile_begin, tile_end) of sequence `seq`, kv head `kh`.
template <int NS = STAGES>
ACP_DEVINL void produce_tiles(const CUtensorMap* tm_k, const CUtensorMap* tm_v, uint8_t* stages,
                              uint64_t* full_bar, uint64_t* empty_bar, const int* pt_row, int kh,
                              int kv_heads, int tile_begin, int tile_end, int last_tok /*exclusive*/) {
  int it = 0;
  for (int tile = tile_begin; tile < tile_end; ++tile, ++it) {
    const int s = it % NS;
    const uint32_t ph = (uint32_t)(it / NS) & 1u;
    mbar_wait(&empty_bar[s], ph ^ 1u);
    const int tok0 = tile * TILE_TOK;
    const int n_pages = (last_tok - tok0 > KV_PAGE) ? 2 : 1;
    mbar_arrive_expect_tx(&full_bar[s], (uint32_t)(n_pages * 4 * BLOCK_BYTES));
    uint8_t* kdst = stages + s * STAGE_BYTES;
    uint8_t* vdst = kdst + K_TILE_BYTES;
    for (int p = 0; p < n_pages; ++p) {
      const int page = pt_row[tok0 / KV_PAGE + p];
      const int row = (page * kv_heads + kh) * 2 * KV_PAGE;  // one contiguous 8 KiB block: both dim-halves
      tma_load_2d(kdst + p * 2 * BLOCK_BYTES, tm_k, &full_bar[s], 0, row, kEvictFirst);
      tma_load_2d(vdst + p * 2 * BLOCK_BYTES, tm_v, &full_bar[s], 0, row, kEvictFirst);
    }
  }
}

struct SmemLayout {
  uint8_t* stages;
  uint64_t* full_bar;
  uint64_t* empty_bar;
  __nv_bfloat16* nq;  // [16][128] rotated query heads of the new token (rows >= G unused)
  float* nk;          // [128] rotated key of the new token (bf16-rounded values)
  float* nv;          // [128]
  float* ns;          // [16] q . k_new per head (raw score units)
};
template <int NS = STAGES>
ACP_DEVINL SmemLayout carve(uint8_t* raw) {
  SmemLayout L;
  uint8_t* base = (uint8_t*)(((uintptr_t)raw + 1023) & ~(uintptr_t)1023);
  L.stages = base;
  L.full_bar = (uint64_t*)(base + NS * STAGE_BYTES);
  L.empty_bar = L.full_bar + NS;
  uint8_t* extra = (uint8_t*)(((uintptr_t)(L.empty_bar + NS) + 63) & ~(uintptr_t)63);
  L.nq = (__nv_bfloat16*)extra;
  L.nk = (float*)(extra + 16 * HEAD_DIM * 2);
  L.nv = L.nk + HEAD_DIM;
  L.ns = L.nv + HEAD_DIM;
  return L;
}
// decode cross-warp merge scratch [4 warps][16 rows][130] aliases the (drained) stage ring
constexpr int SCRATCH_FLOATS = CONSUMER_WARPS * 16 * 130;
static_assert(SCRATCH_FLOATS * 4 <= STAGES * STAGE_BYTES, "scratch must fit in the ring");
// new-token scratch of the decode kernels: q[16 rows][128] bf16 (4 KiB) + k[128] + v[128] + s[16] fp32
constexpr int NEWTOK_BYTES = 16 * HEAD_DIM * 2 + (2 * HEAD_DIM + 16) * 4;
constexpr int ATTN_SMEM = STAGES * STAGE_BYTES + 1024 + 2 * STAGES * 8 + 16 + NEWTOK_BYTES + 64;

// ---------------------------------------------------------------------------------
// New-token prologue of the decode kernels (128 consumer threads): reduce the QKV split-K planes
// for this (sequence, kv head), apply RoPE with the same explicit-rn arithmetic as rope_kv_kernel,
// keep q (bf16) / k / v in shared memory, append K/V to the cache (if `write_kv`), and compute the
// G scores q . k_new.  Ends with a consumer-only barrier.
// ---------------------------------------------------------------------------------
ACP_DEVINL void new_token_prologue(const AttnDecodeArgs& a, const SmemLayout& L, int b, int kh, int ctx,
                                   bool write_kv) {
  const int G = a.heads / a.kv_heads;
  const int tid = threadIdx.x;  // 0..127
  const int pos = ctx - 1;
  const GemmOutDev qkv{a.qkv_ptr, a.qkv_splits, a.qkv_n_cap, a.qkv_ld};
  const int q_dim = a.heads * HEAD_DIM, kv_dim = a.kv_heads * HEAD_DIM;
  const float* ct = a.cos_tab + (size_t)pos * (HEAD_DIM / 2);
  const float* st = a.sin_tab + (size_t)pos * (HEAD_DIM / 2);
  const int page = a.page_table[(size_t)b * a.max_pages + pos / KV_PAGE];
  const size_t blk = ((size_t)page * a.kv_heads + kh) * (KV_PAGE * HEAD_DIM) + (size_t)(pos % KV_PAGE) * 64;
  // rotated vectors: G query heads then the key head; 16 work items (4 frequency pairs) per head
  for (int w = tid; w < (G + 1) * 16; w += 128) {
    const int hv = w >> 4, i0 = (w & 15) * 4;
    const int col = hv < G ? (kh * G + hv) * HEAD_DIM : q_dim + kh * HEAD_DIM;
    float x1[4], x2[4];
    gemm_out_load4(qkv, b, col + i0, x1);
    gemm_out_load4(qkv, b, col + 64 + i0, x2);
    const float4 c = *reinterpret_cast<const float4*>(ct + i0);
    const float4 s = *reinterpret_cast<const float4*>(st + i0);
    const float cc[4] = {c.x, c.y, c.z, c.w}, sn[4] = {s.x, s.y, s.z, s.w};
    float lo[4], hi[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      lo[j] = bf16_round(__fsub_rn(__fmul_rn(x1[j], cc[j]), __fmul_rn(x2[j], sn[j])));
      hi[j] = bf16_round(__fadd_rn(__fmul_rn(x2[j], cc[j]), __fmul_rn(x1[j], sn[j])));
    }
    if (hv < G) {
      __nv_bfloat16* d = L.nq + hv * HEAD_DIM;
      *reinterpret_cast<uint2*>(d + i0) = make_uint2(pack_bf16x2(lo[0], lo[1]), pack_bf16x2(lo[2], lo[3]));
      *reinterpret_cast<uint2*>(d + 64 + i0) = make_uint2(pack_bf16x2(hi[0], hi[1]), pack_bf16x2(hi[2], hi[3]));
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j) { L.nk[i0 + j] = lo[j]; L.nk[64 + i0 + j] = hi[j]; }
      if (write_kv) {
        *reinterpret_cast<uint2*>(a.k_cache + blk + i0) = make_uint2(pack_bf16x2(lo[0], lo[1]), pack_bf16x2(lo[2], lo[3]));
        *reinterpret_cast<uint2*>(a.k_cache + blk + KV_PAGE * 64 + i0) =
            make_uint2(pack_bf16x2(hi[0], hi[1]), pack_bf16x2(hi[2], hi[3]));
      }
    }
  }
  // value head: plain copy (32 work items of 4 elements), done by the upper threads
  if (tid >= 96) {
    const int e = (tid - 96) * 4;
    float v[4];
    gemm_out_load4(qkv, b, q_dim + kv_dim + kh * HEAD_DIM + e, v);
#pragma unroll
    for (int j = 0; j < 4; ++j) L.nv[e + j] = v[j];
    if (write_kv)
      *reinterpret_cast<uint2*>(a.v_cache + blk + (e >> 6) * (KV_PAGE * 64) + (e & 63)) =
          make_uint2(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]));
  }
  asm volatile("bar.sync 1, 128;" ::: "memory");
  // scores of the new token against itself: warp w reduces head w, w+4, ...
  const int warp = tid >> 5, lane = tid & 31;
  for (int g = warp; g < G; g += CONSUMER_WARPS) {
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int d = lane * 4 + j;
      acc += __bfloat162float(L.nq[g * HEAD_DIM + d]) * L.nk[d];
    }
    acc = warp_sum(acc);
    if (lane == 0) L.ns[g] = acc;
  }
  asm volatile("bar.sync 1, 128;" ::: "memory");
}

// Warp 0 folds the new token (one extra key, kept in shared memory) into its running softmax.
ACP_DEVINL void fold_new_token(WarpState& st, const SmemLayout& L, int G, float sl2e, int lane) {
  const int r_lo = lane >> 2;
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int row = r_lo + hh * 8;
    if (row < G) {
      const float s = L.ns[row];
      const float mn = fmaxf(st.m[hh], s);
      const float corr = (st.m[hh] == -INFINITY) ? 0.f : exp2f((st.m[hh] - mn) * sl2e);
      const float p = exp2f((s - mn) * sl2e);
      st.m[hh] = mn;
      st.l[hh] = st.l[hh] * corr + (((lane & 3) == 0) ? p : 0.f);  // l is quad-reduced later
#pragma unroll
      for (int d = 0; d < 16; ++d) {
        const int dim = d * 8 + 2 * (lane & 3);
        st.o[d][hh * 2] = st.o[d][hh * 2] * corr + p * L.nv[dim];
        st.o[d][hh * 2 + 1] = st.o[d][hh * 2 + 1] * corr + p * L.nv[dim + 1];
      }
    }
  }
}

// =================================================================================
// decode, chunked: CTA = (sequence, kv head, chunk of ATTN_CHUNK_TILES tiles).  The chunk
// boundaries depend ONLY on the sequence's own length, so a sequence's result is bit-identical
// whatever it is batched with (batch invariance); long contexts are cut into many CTAs, which is
// what balances a mix of context lengths.  attn_merge_kernel combines the chunks in order.
// =================================================================================
ACP_DEVINL int find_seq(const int* cum, int n, long long f, int kvh) {  // cum[b]*kvh <= f < cum[b+1]*kvh
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if ((long long)cum[mid] * kvh <= f) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__global__ void __launch_bounds__(ATTN_THREADS, 2)
attn_decode_kernel(const __grid_constant__ CUtensorMap tm_k, const __grid_constant__ CUtensorMap tm_v,
                   AttnDecodeArgs a) {
  extern __shared__ uint8_t smem_raw[];
  SmemLayout L = carve(smem_raw);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int G = a.heads / a.kv_heads;
  // linear CTA index -> (sequence b, kv head kh, chunk)
  const long long f = blockIdx.x;
  const int b = find_seq(a.chunk_cum, a.num_seqs, f, a.kv_heads);
  const int nc = a.chunk_cum[b + 1] - a.chunk_cum[b];
  const long long r = f - (long long)a.chunk_cum[b] * a.kv_heads;
  const int kh = (int)(r / nc), chunk = (int)(r % nc);
  const int ctx = a.ctx_len[b];
  // keys 0..ctx-2 are in the cache; the new token (position ctx-1) is handled from shared memory
  const int tile_begin = chunk * ATTN_CHUNK_TILES;
  const int tok_end = min(ctx - 1, (chunk + 1) * ATTN_CHUNK_TILES * TILE_TOK);
  const int tile_end = max(tile_begin, (tok_end + TILE_TOK - 1) / TILE_TOK);
  const int n_tiles = tile_end - tile_begin;
  const bool last_chunk = (chunk == nc - 1);

  pdl_launch_dependents();
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_k);
    tma_prefetch_desc(&tm_v);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&L.full_bar[s], 1);
      mbar_init(&L.empty_bar[s], CONSUMER_WARPS);
    }
    fence_mbar_init();
  }
  __syncthreads();
  // (Starting the K/V stream BEFORE the grid-dependency wait — legal, the cached keys predate the step — was
  // measured in round 2 and lost: 4.157 vs 4.128 ms per config-1 decode step, 9.44 vs 9.21 ms at B = 256; the
  // early loads compete with the QKV GEMM's weight stream instead of hiding under its tail.)
  pdl_wait();  // the QKV planes of the new token come from the previous kernel
  if (warp == CONSUMER_WARPS) {
    if (lane == 0)
      produce_tiles(&tm_k, &tm_v, L.stages, L.full_bar, L.empty_bar,
                    a.page_table + (size_t)b * a.max_pages, kh, a.kv_heads, tile_begin, tile_end, tok_end);
    return;
  }
  const float sl2e = a.scale * 1.4426950408889634f;
  const int r_lo = lane >> 2;
  const int tok_off = warp * 16;
  new_token_prologue(a, L, b, kh, ctx, last_chunk);  // q/k/v of the new token; K/V appended by the last chunk
  uint32_t qf[8][4];
  load_q_frags(qf, r_lo < G ? L.nq + r_lo * HEAD_DIM : nullptr,
               r_lo + 8 < G ? L.nq + (r_lo + 8) * HEAD_DIM : nullptr, lane);
  WarpState st;
#pragma unroll
  for (int d = 0; d < 16; ++d) st.o[d][0] = st.o[d][1] = st.o[d][2] = st.o[d][3] = 0.f;
  st.m[0] = st.m[1] = -INFINITY;
  st.l[0] = st.l[1] = 0.f;
  for (int it = 0; it < n_tiles; ++it) {
    const int s = it % STAGES;
    const uint32_t ph = (uint32_t)(it / STAGES) & 1u;
    mbar_wait(&L.full_bar[s], ph);
    uint8_t* kt = L.stages + s * STAGE_BYTES;
    uint8_t* vt = kt + K_TILE_BYTES;
    const int tile_tok0 = (tile_begin + it) * TILE_TOK;
    const int valid = tok_end - tile_tok0;   // tokens of this tile that exist
    if (valid > tok_off) {
      if (valid < tok_off + 16) zero_v_tail(vt, valid, tok_off + 16, lane);
      process_tile<2>(st, qf, smem_u32(kt), smem_u32(vt), tile_tok0, tok_off, tok_end, tok_end, sl2e, lane);
    }
    __syncwarp();
    if (lane == 0) { fence_proxy_async(); mbar_arrive(&L.empty_bar[s]); }
  }
  if (last_chunk && warp == 0) fold_new_token(st, L, G, sl2e, lane);
  // per-warp partial (m, l, O) of this chunk -> workspace
  st.l[0] += __shfl_xor_sync(0xffffffffu, st.l[0], 1);
  st.l[0] += __shfl_xor_sync(0xffffffffu, st.l[0], 2);
  st.l[1] += __shfl_xor_sync(0xffffffffu, st.l[1], 1);
  st.l[1] += __shfl_xor_sync(0xffffffffu, st.l[1], 2);
  const size_t item = (size_t)b * a.kv_heads + kh;
  float* base = a.ws + (((item * a.max_chunks + chunk) * CONSUMER_WARPS + warp) * G) * 130;
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int row = r_lo + hh * 8;
    if (row < G) {
      float* dst = base + (size_t)row * 130;
      if ((lane & 3) == 0) { dst[128] = st.m[hh]; dst[129] = st.l[hh]; }
#pragma unroll
      for (int d = 0; d < 16; ++d)
        *reinterpret_cast<float2*>(dst + d * 8 + 2 * (lane & 3)) = make_float2(st.o[d][hh * 2], st.o[d][hh * 2 + 1]);
    }
  }
}

// Finishes every (sequence, head): combines chunks x 4 warp partials in fixed order.  For a
// single-chunk item this is the same arithmetic, in the same order, as attn_decode_item_kernel.
__global__ void __launch_bounds__(128)
attn_merge_kernel(AttnDecodeArgs a) {
  pdl_launch_dependents();
  pdl_wait();
  const int b = blockIdx.x, head = blockIdx.y, d = threadIdx.x;
  const int G = a.heads / a.kv_heads;
  const int kh = head / G, g = head % G;
  const int n_pieces = a.chunk_cum[b + 1] - a.chunk_cum[b];
  const float sl2e = a.scale * 1.4426950408889634f;
  const size_t item = (size_t)b * a.kv_heads + kh;
  const float* base = a.ws + ((item * a.max_chunks) * CONSUMER_WARPS * G) * 130;
  float M = -INFINITY;
  for (int p = 0; p < n_pieces; ++p)
    for (int w = 0; w < CONSUMER_WARPS; ++w)
      M = fmaxf(M, base[(((size_t)p * CONSUMER_WARPS + w) * G + g) * 130 + 128]);
  float num = 0.f, den = 0.f;
  for (int p = 0; p < n_pieces; ++p)
    for (int w = 0; w < CONSUMER_WARPS; ++w) {  // fixed order => deterministic
      const float* src = base + (((size_t)p * CONSUMER_WARPS + w) * G + g) * 130;
      const float mw = src[128];
      const float wgt = (mw == -INFINITY) ? 0.f : exp2f((mw - M) * sl2e);
      num += wgt * src[d];
      den += wgt * src[129];
    }
  a.out[(size_t)b * a.heads * HEAD_DIM + head * HEAD_DIM + d] = __float2bfloat16_rn(num / den);
}

// Per-item variant: CTA = (sequence, kv head), the whole context of the item, cross-warp merge in
// shared memory, final bf16 output written directly (no workspace, no merge kernel).  Used when
// there are enough items to fill the machine and every item is short (launch_attn_decode picks).
__global__ void __launch_bounds__(ATTN_THREADS, 2)
attn_decode_item_kernel(const __grid_constant__ CUtensorMap tm_k, const __grid_constant__ CUtensorMap tm_v,
                        AttnDecodeArgs a) {
  extern __shared__ uint8_t smem_raw[];
  SmemLayout L = carve(smem_raw);
  const int b = blockIdx.x, kh = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int G = a.heads / a.kv_heads;
  const int ctx = a.ctx_len[b];
  const int cached = ctx - 1;  // the new token (position ctx-1) is handled from shared memory
  const int n_tiles = (cached + TILE_TOK - 1) / TILE_TOK;

  pdl_launch_dependents();
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_k);
    tma_prefetch_desc(&tm_v);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&L.full_bar[s], 1);
      mbar_init(&L.empty_bar[s], CONSUMER_WARPS);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();
  if (warp == CONSUMER_WARPS) {
    if (lane == 0)
      produce_tiles(&tm_k, &tm_v, L.stages, L.full_bar, L.empty_bar,
                    a.page_table + (size_t)b * a.max_pages, kh, a.kv_heads, 0, n_tiles, cached);
    return;
  }
  const int r_lo = lane >> 2;
  new_token_prologue(a, L, b, kh, ctx, true);
  uint32_t qf[8][4];
  load_q_frags(qf, r_lo < G ? L.nq + r_lo * HEAD_DIM : nullptr,
               r_lo + 8 < G ? L.nq + (r_lo + 8) * HEAD_DIM : nullptr, lane);
  WarpState st;
#pragma unroll
  for (int d = 0; d < 16; ++d) st.o[d][0] = st.o[d][1] = st.o[d][2] = st.o[d][3] = 0.f;
  st.m[0] = st.m[1] = -INFINITY;
  st.l[0] = st.l[1] = 0.f;
  const float sl2e = a.scale * 1.4426950408889634f;
  const int tok_off = warp * 16;
  for (int it = 0; it < n_tiles; ++it) {
    const int s = it % STAGES;
    const uint32_t ph = (uint32_t)(it / STAGES) & 1u;
    mbar_wait(&L.full_bar[s], ph);
    uint8_t* kt = L.stages + s * STAGE_BYTES;
    uint8_t* vt = kt + K_TILE_BYTES;
    const int tile_tok0 = it * TILE_TOK;
    const int valid = cached - tile_tok0;
    if (valid > tok_off) {
      if (valid < tok_off + 16) zero_v_tail(vt, valid, tok_off + 16, lane);
      process_tile<2>(st, qf, smem_u32(kt), smem_u32(vt), tile_tok0, tok_off, cached, cached, sl2e, lane);
    }
    __syncwarp();
    if (lane == 0) { fence_proxy_async(); mbar_arrive(&L.empty_bar[s]); }
  }
  if (warp == 0) fold_new_token(st, L, G, sl2e, lane);
  // ---- merge the 4 warps through the (drained) ring, rows < G only ----
  st.l[0] += __shfl_xor_sync(0xffffffffu, st.l[0], 1);
  st.l[0] += __shfl_xor_sync(0xffffffffu, st.l[0], 2);
  st.l[1] += __shfl_xor_sync(0xffffffffu, st.l[1], 1);
  st.l[1] += __shfl_xor_sync(0xffffffffu, st.l[1], 2);
  asm volatile("bar.sync 1, 128;" ::: "memory");  // every consumer is done with the ring
  float* scratch = reinterpret_cast<float*>(L.stages);
  float* my = scratch + warp * 16 * 130;
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int r = r_lo + hh * 8;
    if (r < G) {
      if ((lane & 3) == 0) { my[r * 130 + 128] = st.m[hh]; my[r * 130 + 129] = st.l[hh]; }
#pragma unroll
      for (int d = 0; d < 16; ++d) {
        my[r * 130 + d * 8 + 2 * (lane & 3)] = st.o[d][hh * 2];
        my[r * 130 + d * 8 + 2 * (lane & 3) + 1] = st.o[d][hh * 2 + 1];
      }
    }
  }
  asm volatile("bar.sync 1, 128;" ::: "memory");
  const int d = threadIdx.x;  // 128 consumer threads <-> 128 dims
  for (int r = 0; r < G; ++r) {
    float M = -INFINITY;
    for (int w = 0; w < CONSUMER_WARPS; ++w) M = fmaxf(M, scratch[(w * 16 + r) * 130 + 128]);
    float num = 0.f, den = 0.f;
    for (int w = 0; w < CONSUMER_WARPS; ++w) {  // fixed order
      const float mw = scratch[(w * 16 + r) * 130 + 128];
      const float wgt = (mw == -INFINITY) ? 0.f : exp2f((mw - M) * sl2e);
      num += wgt * scratch[(w * 16 + r) * 130 + d];
      den += wgt * scratch[(w * 16 + r) * 130 + 129];
    }
    a.out[(size_t)b * a.heads * HEAD_DIM + (kh * G + r) * HEAD_DIM + d] = __float2bfloat16_rn(num / den);
  }
}

// =================================================================================
// prefill (causal, chunk-capable: queries may start at any position of the sequence)
// =================================================================================
// Round 1's mma.sync prefill kernel: kept ONLY as the A/B baseline of the wgmma kernel
// (attention_prefill_tc.cu; ACP_ATTN_PREFILL_TC=0 and tests/test_attention_gpu.py impl 0).
constexpr int NS = STAGES;
__global__ void __launch_bounds__(ATTN_THREADS, 2)
attn_prefill_kernel(const __grid_constant__ CUtensorMap tm_k, const __grid_constant__ CUtensorMap tm_v,
                    AttnPrefillArgs a) {
  extern __shared__ uint8_t smem_raw[];
  SmemLayout L = carve<NS>(smem_raw);
  const int blk = blockIdx.x, kh = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int G = a.heads / a.kv_heads;
  const int tpw = 16 / G;                    // query tokens per warp
  const int b = a.blk_seq[blk];
  const int tq0 = a.blk_tok0[blk];           // first query token (index within the new tokens)
  const int q_len = a.q_len[b], ctx = a.ctx_len[b];
  const int pos0 = ctx - q_len;              // absolute position of new token 0
  const int blk_tokens = min(tpw * CONSUMER_WARPS, q_len - tq0);
  const int last_pos = pos0 + tq0 + blk_tokens - 1;
  const int n_tiles = last_pos / TILE_TOK + 1;

  pdl_launch_dependents();
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_k);
    tma_prefetch_desc(&tm_v);
    for (int s = 0; s < NS; ++s) {
      mbar_init(&L.full_bar[s], 1);
      mbar_init(&L.empty_bar[s], CONSUMER_WARPS);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();
  if (warp == CONSUMER_WARPS) {
    if (lane == 0)
      produce_tiles<NS>(&tm_k, &tm_v, L.stages, L.full_bar, L.empty_bar,
                    a.page_table + (size_t)b * a.max_pages, kh, a.kv_heads, 0, n_tiles, last_pos + 1);
    return;
  }
  // rows of this warp: r -> token tq0 + warp*tpw + r / G, head kh*G + r % G
  const int r_lo = lane >> 2, r_hi = r_lo + 8;
  const int tq_lo = tq0 + warp * tpw + r_lo / G, tq_hi = tq0 + warp * tpw + r_hi / G;
  const bool v_lo = tq_lo < q_len, v_hi = tq_hi < q_len;
  const size_t row_lo = (size_t)(a.q_start[b] + tq_lo), row_hi = (size_t)(a.q_start[b] + tq_hi);
  const int h_lo = kh * G + r_lo % G, h_hi = kh * G + r_hi % G;
  uint32_t qf[8][4];
  load_q_frags(qf, v_lo ? a.q + (row_lo * a.heads + h_lo) * HEAD_DIM : nullptr,
               v_hi ? a.q + (row_hi * a.heads + h_hi) * HEAD_DIM : nullptr, lane);
  const int lim_lo = v_lo ? pos0 + tq_lo + 1 : 0, lim_hi = v_hi ? pos0 + tq_hi + 1 : 0;
  // this warp needs tiles only up to its own last query position
  const int warp_last = pos0 + min(q_len - 1, tq0 + warp * tpw + tpw - 1);
  const bool warp_active = (tq0 + warp * tpw) < q_len;
  WarpState st;
#pragma unroll
  for (int d = 0; d < 16; ++d) st.o[d][0] = st.o[d][1] = st.o[d][2] = st.o[d][3] = 0.f;
  st.m[0] = st.m[1] = -INFINITY;
  st.l[0] = st.l[1] = 0.f;
  const float sl2e = a.scale * 1.4426950408889634f;
  for (int it = 0; it < n_tiles; ++it) {
    const int s = it % NS;
    const uint32_t ph = (uint32_t)(it / NS) & 1u;
    mbar_wait(&L.full_bar[s], ph);
    uint8_t* kt = L.stages + s * STAGE_BYTES;
    uint8_t* vt = kt + K_TILE_BYTES;
    const int tile_tok0 = it * TILE_TOK;
    if (warp_active && tile_tok0 <= warp_last) {
      // tokens past last_pos were not loaded (or belong to the future): zero V there.  Every
      // active warp writes the same zeros, which is benign.
      if (last_pos + 1 - tile_tok0 < TILE_TOK) zero_v_tail(vt, last_pos + 1 - tile_tok0, TILE_TOK, lane);
      process_tile<8>(st, qf, smem_u32(kt), smem_u32(vt), tile_tok0, 0, lim_lo, lim_hi, sl2e, lane);
    }
    __syncwarp();
    if (lane == 0) { fence_proxy_async(); mbar_arrive(&L.empty_bar[s]); }
  }
  st.l[0] += __shfl_xor_sync(0xffffffffu, st.l[0], 1);
  st.l[0] += __shfl_xor_sync(0xffffffffu, st.l[0], 2);
  st.l[1] += __shfl_xor_sync(0xffffffffu, st.l[1], 1);
  st.l[1] += __shfl_xor_sync(0xffffffffu, st.l[1], 2);
  const int c = 2 * (lane & 3);
  if (v_lo) {
    const float inv = 1.0f / st.l[0];
    __nv_bfloat16* o = a.out + (row_lo * a.heads + h_lo) * HEAD_DIM;
#pragma unroll
    for (int d = 0; d < 16; ++d)
      *reinterpret_cast<uint32_t*>(o + d * 8 + c) = pack_bf16x2(st.o[d][0] * inv, st.o[d][1] * inv);
  }
  if (v_hi) {
    const float inv = 1.0f / st.l[1];
    __nv_bfloat16* o = a.out + (row_hi * a.heads + h_hi) * HEAD_DIM;
#pragma unroll
    for (int d = 0; d < 16; ++d)
      *reinterpret_cast<uint32_t*>(o + d * 8 + c) = pack_bf16x2(st.o[d][2] * inv, st.o[d][3] * inv);
  }
}

}  // namespace

int attn_setup_attributes() {
  if (cudaFuncSetAttribute(attn_decode_item_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, ATTN_SMEM) != cudaSuccess ||
      cudaFuncSetAttribute(attn_decode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, ATTN_SMEM) != cudaSuccess ||
      cudaFuncSetAttribute(attn_prefill_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, ATTN_SMEM) != cudaSuccess) {
    fprintf(stderr, "[acp_infer] attention cudaFuncSetAttribute failed\n");
    return -5;
  }
  return attn_prefill_tc_setup();
}

int attn_make_kv_map(CUtensorMap* out, const void* base, uint64_t num_pages, int kv_heads) {
  // block of a (page, kv head) = [2 dim-halves][32 tokens][64 dims], 8 KiB contiguous; 2-D view
  // [num_pages*kv_heads*64 rows][64 cols], ONE box {64 cols, 64 rows} per block and tensor
  return tma_encode_2d_bf16(out, base, num_pages * (uint64_t)kv_heads * 2 * KV_PAGE, 64, 2 * KV_PAGE);
}

int attn_decode_chunks(int ctx_len) {
  const int tiles = (ctx_len + TILE_TOK - 1) / TILE_TOK;
  return (tiles + ATTN_CHUNK_TILES - 1) / ATTN_CHUNK_TILES;
}
size_t attn_decode_ws_floats(int max_batch, int heads, int kv_heads, int max_chunks) {
  return (size_t)max_batch * kv_heads * max_chunks * CONSUMER_WARPS * (heads / kv_heads) * 130;
}

int launch_attn_decode(const CUtensorMap& tm_k, const CUtensorMap& tm_v, const AttnDecodeArgs& a,
                       cudaStream_t s) {
  if (a.num_seqs <= 0) return 0;
  if (a.heads % a.kv_heads != 0 || a.heads / a.kv_heads > 16) return -1;
  if (a.per_item) {
    cudaError_t e = acp_launch(attn_decode_item_kernel, dim3(a.num_seqs, a.kv_heads), dim3(ATTN_THREADS), ATTN_SMEM, s, tm_k, tm_v, a);
    if (e != cudaSuccess) { fprintf(stderr, "[acp_infer] attn_decode_item launch: %s\n", cudaGetErrorString(e)); return -5; }
    return 0;
  }
  if (a.total_chunks <= 0) return -1;
  cudaError_t e = acp_launch(attn_decode_kernel, dim3((unsigned)(a.total_chunks * a.kv_heads)), dim3(ATTN_THREADS), ATTN_SMEM, s, tm_k, tm_v, a);
  if (e != cudaSuccess) { fprintf(stderr, "[acp_infer] attn_decode launch: %s\n", cudaGetErrorString(e)); return -5; }
  e = acp_launch(attn_merge_kernel, dim3(a.num_seqs, a.heads), dim3(128), 0, s, a);
  if (e != cudaSuccess) { fprintf(stderr, "[acp_infer] attn_merge launch: %s\n", cudaGetErrorString(e)); return -5; }
  return 0;
}

bool attn_prefill_tc_enabled() {
  static const bool on = [] { const char* e = getenv("ACP_ATTN_PREFILL_TC"); return !(e && *e == '0'); }();
  return on;
}
int attn_prefill_block_tokens(int heads, int kv_heads) {
  if (attn_prefill_tc_enabled()) return attn_prefill_tc_block_tokens(heads, kv_heads);
  return (16 / (heads / kv_heads)) * CONSUMER_WARPS;
}

int launch_attn_prefill(const CUtensorMap& tm_k, const CUtensorMap& tm_v, const AttnPrefillArgs& a,
                        int num_blocks, cudaStream_t s) {
  if (num_blocks <= 0) return 0;
  const int G = a.heads / a.kv_heads;
  if (a.heads % a.kv_heads != 0 || G > 16 || (16 % G) != 0) return -1;
  dim3 grid(num_blocks, a.kv_heads);
  cudaError_t e = acp_launch(attn_prefill_kernel, grid, dim3(ATTN_THREADS), ATTN_SMEM, s, tm_k, tm_v, a);
  if (e != cudaSuccess) { fprintf(stderr, "[acp_infer] attn_prefill launch: %s\n", cudaGetErrorString(e)); return -5; }
  return 0;
}

}  // namespace acp
