// kernel_tests.cu — C-ABI per-kernel test hooks (include/acp_infer_kernels.h).
// Host buffers in, host buffers out; used only by tests/ to compare each kernel with oracle/.
#include "acp_infer_kernels.h"
#include "common.cuh"
#include "gemm.h"
#include "gemm_wgmma.cuh"
#include "attention.h"
#include "fp8.h"
#include "moe.h"
#include <string.h>
#include <algorithm>
#include <utility>
#include <vector>

using namespace acp;

namespace {
struct DevBuf {
  void* p = nullptr;
  ~DevBuf() { if (p) cudaFree(p); }
  int alloc(size_t bytes) { return cudaMalloc(&p, bytes ? bytes : 1) == cudaSuccess ? 0 : -5; }
};
// Every output buffer of a hook (GEMM output or split-K planes, attention output, decode merge workspace) is followed
// by kGuardBytes of 0xff: a store past its end changes one, and the hook returns ACP_ERR_GUARD instead of the result.
constexpr size_t kGuardBytes = 4096;
int check_guard(const DevBuf& out, size_t out_bytes) {
  std::vector<uint8_t> g(kGuardBytes);
  if (cudaMemcpy(g.data(), (const uint8_t*)out.p + out_bytes, kGuardBytes, cudaMemcpyDeviceToHost) != cudaSuccess) return -5;
  for (uint8_t b : g)
    if (b != 0xff) {
      fprintf(stderr, "[acp_infer] kernel store past the end of an output buffer (%zu bytes)\n", out_bytes);
      return ACP_ERR_GUARD;
    }
  return 0;
}
__global__ void l2_flush_kernel(float* buf, size_t n) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  size_t stride = (size_t)gridDim.x * blockDim.x;
  for (; i < n; i += stride) buf[i] = buf[i] * 1.0001f + 1.0f;
}
}  // namespace

extern "C" int acp_kernel_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
  return n;
}

extern "C" int acp_kernel_gemm_path(int M, int N, int K, int splits, int epi, int bn) {
  GemmLaunch g;
  g.M = M; g.N = N; g.K = K; g.epi = epi; g.splits = splits;
  g.bn_override = bn;
  return gemm_path(g);
}

extern "C" int acp_kernel_gemm_persistent_clusters(int fp8, int epi) {
  if (acp_kernel_device_count() <= 0 || gemm_setup_attributes() != 0) return -5;
  return gemm_persistent_clusters(fp8 != 0, epi);
}

extern "C" int acp_kernel_gemm(const uint16_t* w, const uint16_t* x, int M, int N, int K,
                               int splits, int epi, int bn, void* out, float* amax_val,
                               int* amax_idx, int iters, float* elapsed_ms) {
  if (acp_kernel_device_count() <= 0) {
    fprintf(stderr, "[acp_infer] no CUDA device: kernels cannot run (no CPU fallback)\n");
    return -5;
  }
  if (gemm_setup_attributes() != 0) return -5;
  const int m_tiles = (M + GEMM_BM - 1) / GEMM_BM;
  DevBuf dw, dx, dout, dval, didx, dflush;
  // activation rows are padded to the largest N tile like the engine's buffers (zero rows)
  const int n_pad = ((N + 255) / 256) * 256;
  // weights: zero-pad to (128, 64) multiples and re-order into the engine's tiled layout
  const int Mp = ((M + GEMM_BM - 1) / GEMM_BM) * GEMM_BM, Kp = ((K + GEMM_BK - 1) / GEMM_BK) * GEMM_BK;
  const int nkb_p = Kp / GEMM_BK;
  std::vector<uint16_t> wt((size_t)Mp * Kp, 0), xp((size_t)N * Kp, 0);
  for (int r = 0; r < M; ++r)
    for (int c = 0; c < K; ++c)
      wt[((size_t)(r / GEMM_BM) * nkb_p + c / GEMM_BK) * 8192 + (size_t)(r % GEMM_BM) * 64 + c % GEMM_BK] =
          w[(size_t)r * K + c];
  for (int r = 0; r < N; ++r) memcpy(&xp[(size_t)r * Kp], &x[(size_t)r * K], (size_t)K * 2);
  if (dw.alloc(wt.size() * 2) || dx.alloc((size_t)n_pad * Kp * 2)) return -5;
  ACP_CUDA_CHECK(cudaMemset(dx.p, 0, (size_t)n_pad * Kp * 2));
  ACP_CUDA_CHECK(cudaMemcpy(dw.p, wt.data(), wt.size() * 2, cudaMemcpyHostToDevice));
  ACP_CUDA_CHECK(cudaMemcpy(dx.p, xp.data(), xp.size() * 2, cudaMemcpyHostToDevice));
  size_t out_bytes = 0;
  if (epi == EPI_BF16) out_bytes = (size_t)N * M * 2;
  else if (epi == EPI_F32) out_bytes = (size_t)splits * N * M * 4;
  else if (epi == EPI_SWIGLU) out_bytes = (size_t)N * (M / 2) * 2;
  else if (out != nullptr) out_bytes = (size_t)N * M * 4;
  if (dout.alloc(out_bytes + kGuardBytes)) return -5;
  ACP_CUDA_CHECK(cudaMemset(dout.p, 0xff, out_bytes + kGuardBytes));
  if (epi == EPI_ARGMAX) {
    if (dval.alloc((size_t)N * m_tiles * 4) || didx.alloc((size_t)N * m_tiles * 4)) return -5;
  }
  TmaMaps mw, mx;
  if (tma_make_weight(&mw, dw.p, Mp, Kp) != 0) return -5;
  if (tma_make_act(&mx, dx.p, n_pad, Kp) != 0) return -5;
  GemmLaunch g;
  g.w = &mw.w; g.x = &mx; g.M = M; g.N = N; g.K = Kp; g.splits = splits; g.epi = epi;
  g.ld = (epi == EPI_SWIGLU) ? M / 2 : M; g.n_cap = N;
  g.out = (epi == EPI_ARGMAX && out == nullptr) ? nullptr : dout.p;
  g.amax_val = (float*)dval.p; g.amax_idx = (int*)didx.p; g.bn_override = bn;   // hook-only: bn -1 forces the persistent prefill kernel
  int rc = gemm_launch(g, 0);
  if (rc != 0) return rc;
  ACP_CUDA_CHECK(cudaDeviceSynchronize());
  if ((rc = check_guard(dout, out_bytes)) != 0) return rc;
  if (out != nullptr && out_bytes)
    ACP_CUDA_CHECK(cudaMemcpy(out, dout.p, out_bytes, cudaMemcpyDeviceToHost));
  if (epi == EPI_ARGMAX) {
    // final reduction over m-tiles on the host for this hook (the engine does it on device)
    std::vector<float> tv((size_t)N * m_tiles);
    std::vector<int> ti((size_t)N * m_tiles);
    ACP_CUDA_CHECK(cudaMemcpy(tv.data(), dval.p, tv.size() * 4, cudaMemcpyDeviceToHost));
    ACP_CUDA_CHECK(cudaMemcpy(ti.data(), didx.p, ti.size() * 4, cudaMemcpyDeviceToHost));
    for (int n = 0; n < N; ++n) {
      float bv = tv[(size_t)n * m_tiles];
      int bi = ti[(size_t)n * m_tiles];
      for (int t = 1; t < m_tiles; ++t) {
        float v = tv[(size_t)n * m_tiles + t];
        int i = ti[(size_t)n * m_tiles + t];
        if (v > bv || (v == bv && i < bi)) { bv = v; bi = i; }
      }
      amax_val[n] = bv;
      amax_idx[n] = bi;
    }
  }
  if (iters < 0 && elapsed_ms != nullptr) {
    // STRESS mode: -iters back-to-back launches (programmatic dependent launch on, no L2 flush, one sync at the
    // end) — what a rare pipeline deadlock needs to show up; a hang ends in the kernels' own bounded waits
    cudaEvent_t e0, e1;
    ACP_CUDA_CHECK(cudaEventCreate(&e0));
    ACP_CUDA_CHECK(cudaEventCreate(&e1));
    ACP_CUDA_CHECK(cudaEventRecord(e0, 0));
    for (int it = 0; it < -iters; ++it) {
      rc = gemm_launch(g, 0);
      if (rc != 0) return rc;
    }
    ACP_CUDA_CHECK(cudaEventRecord(e1, 0));
    ACP_CUDA_CHECK(cudaEventSynchronize(e1));
    float ms = 0.f;
    ACP_CUDA_CHECK(cudaEventElapsedTime(&ms, e0, e1));
    *elapsed_ms = ms / (float)(-iters);
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
  }
  if (iters > 0 && elapsed_ms != nullptr) {
    const size_t flush_n = (size_t)64 << 20;  // 256 MiB of fp32 > 50 MB L2
    if (dflush.alloc(flush_n * 4)) return -5;
    ACP_CUDA_CHECK(cudaMemset(dflush.p, 0, flush_n * 4));
    cudaEvent_t e0, e1;
    ACP_CUDA_CHECK(cudaEventCreate(&e0));
    ACP_CUDA_CHECK(cudaEventCreate(&e1));
    float total = 0.f;
    for (int it = 0; it < iters + 2; ++it) {
      l2_flush_kernel<<<1184, 256>>>((float*)dflush.p, flush_n);
      ACP_CUDA_CHECK(cudaEventRecord(e0, 0));
      rc = gemm_launch(g, 0);
      if (rc != 0) return rc;
      ACP_CUDA_CHECK(cudaEventRecord(e1, 0));
      ACP_CUDA_CHECK(cudaEventSynchronize(e1));
      float ms = 0.f;
      ACP_CUDA_CHECK(cudaEventElapsedTime(&ms, e0, e1));
      if (it >= 2) total += ms;  // two warm-up launches
    }
    *elapsed_ms = total / iters;
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
  }
  return 0;
}


// mean milliseconds of `iters` launches, L2 flushed before each (two untimed warm-up launches)
template <class F>
static int time_launches(F launch, int iters, float* elapsed_ms) {
  DevBuf dflush;
  const size_t flush_n = (size_t)64 << 20;  // 256 MiB of fp32 > 50 MB L2
  if (dflush.alloc(flush_n * 4)) return -5;
  ACP_CUDA_CHECK(cudaMemset(dflush.p, 0, flush_n * 4));
  cudaEvent_t e0, e1;
  ACP_CUDA_CHECK(cudaEventCreate(&e0));
  ACP_CUDA_CHECK(cudaEventCreate(&e1));
  float total = 0.f;
  int rc = 0;
  for (int it = 0; it < iters + 2 && rc == 0; ++it) {
    l2_flush_kernel<<<1184, 256>>>((float*)dflush.p, flush_n);
    ACP_CUDA_CHECK(cudaEventRecord(e0, 0));
    rc = launch();
    ACP_CUDA_CHECK(cudaEventRecord(e1, 0));
    ACP_CUDA_CHECK(cudaEventSynchronize(e1));
    float ms = 0.f;
    ACP_CUDA_CHECK(cudaEventElapsedTime(&ms, e0, e1));
    if (it >= 2) total += ms;
  }
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  *elapsed_ms = total / iters;
  return rc;
}

// ---------------------------------------------------------------------------------
// Attention hooks.  They share one paged K/V cache builder: the pages of all sequences are a shuffled
// permutation of physical pages 1..num_pages-1 (two of them spare), page 0 is reserved and stays zero like
// the engine's (which never hands it out; the wgmma prefill kernel reads it for a tile's missing second
// page), and every slot no sequence owns (the tail of each sequence's last page, the spare pages) holds the
// bf16 pattern `stale` — what a recycled page keeps from its previous owner.
// ---------------------------------------------------------------------------------
namespace {
struct PagedKv {
  int kv_heads = 0, num_pages = 0;
  std::vector<int> page_off, page_table;   // packed: pages of sequence b are page_table[page_off[b] .. page_off[b+1])
  std::vector<uint16_t> k, v;              // [num_pages][kv_heads][2 dim halves][KV_PAGE][64]
  // element (dim d, kv head h) of position t of sequence b
  size_t at(int b, int t, int h, int d) const {
    const int page = page_table[page_off[b] + t / KV_PAGE];
    return ((size_t)page * kv_heads + h) * (KV_PAGE * HEAD_DIM) + (size_t)(d >> 6) * (KV_PAGE * 64) +
           (size_t)(t % KV_PAGE) * 64 + (d & 63);
  }
};

// sequence b owns positions 0..n_tok[b]-1 (ceil(n_tok[b] / 32) pages)
void paged_kv_build(PagedKv& c, int B, const int* n_tok, int kv_heads, uint16_t stale) {
  c.kv_heads = kv_heads;
  c.page_off.assign(B + 1, 0);
  for (int b = 0; b < B; ++b) c.page_off[b + 1] = c.page_off[b] + (n_tok[b] + KV_PAGE - 1) / KV_PAGE;
  const int n = c.page_off[B];
  c.num_pages = n + 3;
  c.page_table.resize(n);
  for (int i = 0; i < n; ++i) c.page_table[i] = 1 + (int)(((long long)i * 7 + 3) % (c.num_pages - 1));
  {  // make it a permutation (7 may share a factor with num_pages - 1): fall back to reversed order
    std::vector<char> seen(c.num_pages, 0);
    bool ok = true;
    for (int i = 0; i < n; ++i) { if (seen[c.page_table[i]]) ok = false; seen[c.page_table[i]] = 1; }
    if (!ok) for (int i = 0; i < n; ++i) c.page_table[i] = c.num_pages - 1 - i;
  }
  const size_t page_elems = (size_t)kv_heads * KV_PAGE * HEAD_DIM;
  c.k.assign((size_t)c.num_pages * page_elems, stale);
  std::fill(c.k.begin(), c.k.begin() + page_elems, (uint16_t)0);   // page 0
  c.v = c.k;
}

// rows [row0, row0 + count) of a packed [rows][kv_heads][128] K/V array -> positions 0..count-1 of sequence b
void paged_kv_fill(PagedKv& c, int b, const uint16_t* k, const uint16_t* v, size_t row0, int count) {
  for (int t = 0; t < count; ++t)
    for (int h = 0; h < c.kv_heads; ++h)
      for (int d = 0; d < HEAD_DIM; ++d) {
        const size_t src = ((row0 + t) * c.kv_heads + h) * HEAD_DIM + d, dst = c.at(b, t, h, d);
        c.k[dst] = k[src];
        c.v[dst] = v[src];
      }
}

int paged_kv_upload(const PagedKv& c, DevBuf& dk, DevBuf& dv) {
  if (dk.alloc(c.k.size() * 2) || dv.alloc(c.v.size() * 2)) return -5;
  ACP_CUDA_CHECK(cudaMemcpy(dk.p, c.k.data(), c.k.size() * 2, cudaMemcpyHostToDevice));
  ACP_CUDA_CHECK(cudaMemcpy(dv.p, c.v.data(), c.v.size() * 2, cudaMemcpyHostToDevice));
  return 0;
}

// Reads the caches back: the slots (sequence, position) of `written` go to k_out / v_out [n][kv_heads][128];
// every other byte must still be what paged_kv_build / paged_kv_fill put there, else ACP_ERR_GUARD.
int paged_kv_read_back(const PagedKv& c, const DevBuf& dk, const DevBuf& dv, const std::vector<std::pair<int, int>>& written,
                       uint16_t* k_out, uint16_t* v_out) {
  std::vector<uint16_t> k(c.k.size()), v(c.v.size());
  ACP_CUDA_CHECK(cudaMemcpy(k.data(), dk.p, k.size() * 2, cudaMemcpyDeviceToHost));
  ACP_CUDA_CHECK(cudaMemcpy(v.data(), dv.p, v.size() * 2, cudaMemcpyDeviceToHost));
  for (size_t i = 0; i < written.size(); ++i)
    for (int h = 0; h < c.kv_heads; ++h)
      for (int d = 0; d < HEAD_DIM; ++d) {
        const size_t at = c.at(written[i].first, written[i].second, h, d), o = (i * c.kv_heads + h) * HEAD_DIM + d;
        k_out[o] = k[at]; k[at] = c.k[at];
        v_out[o] = v[at]; v[at] = c.v[at];
      }
  if (memcmp(k.data(), c.k.data(), k.size() * 2) || memcmp(v.data(), c.v.data(), v.size() * 2)) {
    fprintf(stderr, "[acp_infer] attention kernel wrote a K/V cache slot it does not own\n");
    return ACP_ERR_GUARD;
  }
  return 0;
}

// A QKV projection result as its consumers read it (GemmOut): bf16 [n_cap][ld] (splits 0) or `splits` fp32
// planes [splits][n_cap][ld].  The caller gives rows 0..rows-1 ([rows][ld], or [splits][rows][ld]); rows
// rows..n_cap-1 are NaN, so a read of a row past the step shows up in the result.
int upload_qkv(DevBuf& d, const void* qkv, int splits, int rows, int n_cap, int ld) {
  const size_t esz = splits ? 4 : 2, planes = splits ? splits : 1;
  const size_t plane_bytes = (size_t)n_cap * ld * esz, given = (size_t)rows * ld * esz;
  if (d.alloc(planes * plane_bytes)) return -5;
  ACP_CUDA_CHECK(cudaMemset(d.p, 0xff, planes * plane_bytes));
  for (size_t s = 0; s < planes; ++s)
    ACP_CUDA_CHECK(cudaMemcpy((uint8_t*)d.p + s * plane_bytes, (const uint8_t*)qkv + s * given, given, cudaMemcpyHostToDevice));
  return 0;
}

int upload_rope_tables(DevBuf& dc, DevBuf& ds, const float* cos_tab, const float* sin_tab, int max_pos) {
  const size_t bytes = (size_t)max_pos * (HEAD_DIM / 2) * 4;
  if (dc.alloc(bytes) || ds.alloc(bytes)) return -5;
  ACP_CUDA_CHECK(cudaMemcpy(dc.p, cos_tab, bytes, cudaMemcpyHostToDevice));
  ACP_CUDA_CHECK(cudaMemcpy(ds.p, sin_tab, bytes, cudaMemcpyHostToDevice));
  return 0;
}

int no_device() {
  if (acp_kernel_device_count() > 0) return 0;
  fprintf(stderr, "[acp_infer] no CUDA device: kernels cannot run (no CPU fallback)\n");
  return -5;
}
}  // namespace

extern "C" int acp_kernel_attn_prefill_batch(const uint16_t* q, const uint16_t* k, const uint16_t* v, int heads,
                                             int kv_heads, int B, const int* q_len, const int* ctx_len, uint16_t stale,
                                             int impl, uint16_t* out, int iters, float* elapsed_ms) {
  if (int rc = no_device()) return rc;
  if (!q || !k || !v || !out || !q_len || !ctx_len || B <= 0 || kv_heads <= 0 || heads % kv_heads) return -1;
  int T = 0;
  for (int b = 0; b < B; ++b) {
    if (q_len[b] <= 0 || ctx_len[b] < q_len[b]) return -1;
    T += q_len[b];
  }
  if (attn_setup_attributes() != 0) return -5;
  PagedKv c;
  paged_kv_build(c, B, ctx_len, kv_heads, stale);
  for (int b = 0, r = 0; b < B; r += ctx_len[b], ++b) paged_kv_fill(c, b, k, v, r, ctx_len[b]);
  // the step's q rows packed one sequence after the other, like the engine's qbuf; rows past T hold `stale`
  const int T_cap = ((T + 255) / 256) * 256;
  const size_t row_elems = (size_t)heads * HEAD_DIM, q_elems = (size_t)T * row_elems;
  DevBuf dq, dk, dv, dout, dints;
  if (dq.alloc((size_t)T_cap * row_elems * 2) || dout.alloc(q_elems * 2 + kGuardBytes)) return -5;
  {
    std::vector<uint16_t> qp((size_t)T_cap * row_elems, stale);
    memcpy(qp.data(), q, q_elems * 2);
    ACP_CUDA_CHECK(cudaMemcpy(dq.p, qp.data(), qp.size() * 2, cudaMemcpyHostToDevice));
  }
  ACP_CUDA_CHECK(cudaMemset(dout.p, 0xff, q_elems * 2 + kGuardBytes));
  if (paged_kv_upload(c, dk, dv)) return -5;
  // query blocks as the engine builds them: per sequence, blk_tokens new tokens each
  const int blk_tokens = impl ? attn_prefill_tc_block_tokens(heads, kv_heads) : (16 / (heads / kv_heads)) * 4;
  std::vector<int> blk_seq, blk_tok0, q_start(B);
  for (int b = 0, row = 0; b < B; row += q_len[b], ++b) {
    q_start[b] = row;
    for (int t0 = 0; t0 < q_len[b]; t0 += blk_tokens) { blk_seq.push_back(b); blk_tok0.push_back(t0); }
  }
  const int n_blocks = (int)blk_seq.size();
  // packed ints: blk_seq[n_blocks] blk_tok0[n_blocks] q_start[B] q_len[B] ctx_len[B] page_off[B+1] page_table[]
  std::vector<int> ints(blk_seq);
  ints.insert(ints.end(), blk_tok0.begin(), blk_tok0.end());
  ints.insert(ints.end(), q_start.begin(), q_start.end());
  ints.insert(ints.end(), q_len, q_len + B);
  ints.insert(ints.end(), ctx_len, ctx_len + B);
  ints.insert(ints.end(), c.page_off.begin(), c.page_off.end());
  ints.insert(ints.end(), c.page_table.begin(), c.page_table.end());
  if (dints.alloc(ints.size() * 4)) return -5;
  ACP_CUDA_CHECK(cudaMemcpy(dints.p, ints.data(), ints.size() * 4, cudaMemcpyHostToDevice));
  const int* di = (const int*)dints.p;
  AttnPrefillArgs pa;
  pa.q = (const __nv_bfloat16*)dq.p; pa.out = (__nv_bfloat16*)dout.p;
  pa.blk_seq = di; pa.blk_tok0 = di + n_blocks; pa.q_start = di + 2 * n_blocks; pa.q_len = pa.q_start + B;
  pa.ctx_len = pa.q_len + B; pa.page_off = pa.ctx_len + B; pa.page_table = pa.page_off + B + 1;
  pa.heads = heads; pa.kv_heads = kv_heads; pa.scale = 1.0f / sqrtf((float)HEAD_DIM);
  CUtensorMap tq, tk, tv;
  if (impl) {
    if (attn_make_q_map(&tq, dq.p, (uint64_t)T_cap, heads, kv_heads) != 0) return -5;
    if (attn_make_kv_half_map(&tk, dk.p, c.num_pages, kv_heads) != 0 || attn_make_kv_half_map(&tv, dv.p, c.num_pages, kv_heads) != 0) return -5;
  } else {
    if (attn_make_kv_map(&tk, dk.p, c.num_pages, kv_heads) != 0 || attn_make_kv_map(&tv, dv.p, c.num_pages, kv_heads) != 0) return -5;
  }
  auto launch = [&]() { return impl ? launch_attn_prefill_tc(tq, tk, tv, pa, n_blocks, 0) : launch_attn_prefill(tk, tv, pa, n_blocks, 0); };
  int rc = launch();
  if (rc != 0) return rc;
  ACP_CUDA_CHECK(cudaDeviceSynchronize());
  if ((rc = check_guard(dout, q_elems * 2)) != 0) return rc;
  ACP_CUDA_CHECK(cudaMemcpy(out, dout.p, q_elems * 2, cudaMemcpyDeviceToHost));
  std::vector<uint16_t> none;
  if ((rc = paged_kv_read_back(c, dk, dv, {}, none.data(), none.data())) != 0) return rc;
  if (iters > 0 && elapsed_ms != nullptr) return time_launches(launch, iters, elapsed_ms);
  return 0;
}

extern "C" int acp_kernel_attn_prefill(const uint16_t* q, const uint16_t* k, const uint16_t* v, int heads, int kv_heads,
                                       int q_len, int ctx, int impl, uint16_t* out, int iters, float* elapsed_ms) {
  return acp_kernel_attn_prefill_batch(q, k, v, heads, kv_heads, 1, &q_len, &ctx, 0, impl, out, iters, elapsed_ms);
}

extern "C" int acp_kernel_attn_decode(const uint16_t* k, const uint16_t* v, const void* qkv, int splits, int n_cap,
                                      const float* cos_tab, const float* sin_tab, int max_pos, int B, const int* ctx_len,
                                      int heads, int kv_heads, int mode, uint16_t stale, uint16_t* out, uint16_t* k_new,
                                      uint16_t* v_new) {
  if (int rc = no_device()) return rc;
  if (!k || !v || !qkv || !cos_tab || !sin_tab || !ctx_len || !out || !k_new || !v_new || B <= 0 || n_cap < B ||
      splits < 0 || kv_heads <= 0 || heads % kv_heads || heads / kv_heads > 16 || mode < 0 || mode > 2)
    return -1;
  int max_pages = 0;
  std::vector<int> chunk_cum(B + 1, 0);
  for (int b = 0; b < B; ++b) {
    if (ctx_len[b] < 1 || ctx_len[b] > max_pos) return -1;
    max_pages = std::max(max_pages, (ctx_len[b] + KV_PAGE - 1) / KV_PAGE);
    chunk_cum[b + 1] = chunk_cum[b] + attn_decode_chunks(ctx_len[b]);   // as the engine's tile_cum
  }
  const int total_chunks = chunk_cum[B];
  if (mode == 1 && total_chunks != B) return -1;   // the per-item kernel takes one chunk per sequence
  if (attn_setup_attributes() != 0) return -5;
  // positions 0..ctx-2 are cached; ctx-1 (the new token) is appended by the kernel
  PagedKv c;
  paged_kv_build(c, B, ctx_len, kv_heads, stale);
  for (int b = 0, r = 0; b < B; r += ctx_len[b] - 1, ++b) paged_kv_fill(c, b, k, v, r, ctx_len[b] - 1);
  const int ld = (heads + 2 * kv_heads) * HEAD_DIM;
  const int max_chunks = attn_decode_chunks(max_pages * KV_PAGE);   // workspace stride, as the model sizes it
  const size_t out_bytes = (size_t)B * heads * HEAD_DIM * 2;
  const size_t ws_bytes = attn_decode_ws_floats(B, heads, kv_heads, max_chunks) * 4;
  DevBuf dqkv, dk, dv, dcos, dsin, dout, dws, dints;
  if (upload_qkv(dqkv, qkv, splits, B, n_cap, ld) || upload_rope_tables(dcos, dsin, cos_tab, sin_tab, max_pos) ||
      paged_kv_upload(c, dk, dv) || dout.alloc(out_bytes + kGuardBytes) || dws.alloc(ws_bytes + kGuardBytes))
    return -5;
  ACP_CUDA_CHECK(cudaMemset(dout.p, 0xff, out_bytes + kGuardBytes));
  ACP_CUDA_CHECK(cudaMemset(dws.p, 0xff, ws_bytes + kGuardBytes));
  // packed ints: ctx_len[B] chunk_cum[B+1] page_off[B+1] page_table[]
  std::vector<int> ints(ctx_len, ctx_len + B);
  ints.insert(ints.end(), chunk_cum.begin(), chunk_cum.end());
  ints.insert(ints.end(), c.page_off.begin(), c.page_off.end());
  ints.insert(ints.end(), c.page_table.begin(), c.page_table.end());
  if (dints.alloc(ints.size() * 4)) return -5;
  ACP_CUDA_CHECK(cudaMemcpy(dints.p, ints.data(), ints.size() * 4, cudaMemcpyHostToDevice));
  const int* di = (const int*)dints.p;
  AttnDecodeArgs a;
  a.q = nullptr; a.out = (__nv_bfloat16*)dout.p;
  a.ctx_len = di; a.chunk_cum = di + B; a.page_off = di + 2 * B + 1; a.page_table = a.page_off + B + 1;
  a.heads = heads; a.kv_heads = kv_heads; a.num_seqs = B;
  a.total_chunks = total_chunks; a.max_chunks = max_chunks;
  a.per_item = mode == 2 ? 0 : (total_chunks == B ? 1 : 0);   // mode 0 picks like the model
  a.scale = 1.0f / sqrtf((float)HEAD_DIM); a.ws = (float*)dws.p;
  a.qkv_ptr = dqkv.p; a.qkv_splits = splits; a.qkv_n_cap = n_cap; a.qkv_ld = ld;
  a.cos_tab = (const float*)dcos.p; a.sin_tab = (const float*)dsin.p;
  a.k_cache = (__nv_bfloat16*)dk.p; a.v_cache = (__nv_bfloat16*)dv.p;
  CUtensorMap tk, tv;
  if (attn_make_kv_map(&tk, dk.p, c.num_pages, kv_heads) != 0 || attn_make_kv_map(&tv, dv.p, c.num_pages, kv_heads) != 0) return -5;
  int rc = launch_attn_decode(tk, tv, a, 0);
  if (rc == 0 && !a.per_item) rc = launch_attn_merge(a, 0);
  if (rc != 0) return rc;
  ACP_CUDA_CHECK(cudaDeviceSynchronize());
  if ((rc = check_guard(dout, out_bytes)) != 0 || (rc = check_guard(dws, ws_bytes)) != 0) return rc;
  ACP_CUDA_CHECK(cudaMemcpy(out, dout.p, out_bytes, cudaMemcpyDeviceToHost));
  std::vector<std::pair<int, int>> written;
  for (int b = 0; b < B; ++b) written.emplace_back(b, ctx_len[b] - 1);
  return paged_kv_read_back(c, dk, dv, written, k_new, v_new);
}

extern "C" int acp_kernel_rope_kv(const void* qkv, int splits, int n_cap, int T, const int* seq_of_row, const int* pos,
                                  int B, const float* cos_tab, const float* sin_tab, int max_pos, int heads, int kv_heads,
                                  uint16_t stale, uint16_t* q_out, uint16_t* k_out, uint16_t* v_out) {
  if (int rc = no_device()) return rc;
  if (!qkv || !seq_of_row || !pos || !cos_tab || !sin_tab || !q_out || !k_out || !v_out || T <= 0 || B <= 0 ||
      n_cap < T || splits < 0 || kv_heads <= 0 || heads % kv_heads)
    return -1;
  // sequence b owns positions 0..(its largest row position); each (sequence, position) is written once
  std::vector<int> n_tok(B, 1);
  std::vector<std::pair<int, int>> written;
  for (int t = 0; t < T; ++t) {
    if (seq_of_row[t] < 0 || seq_of_row[t] >= B || pos[t] < 0 || pos[t] >= max_pos) return -1;
    n_tok[seq_of_row[t]] = std::max(n_tok[seq_of_row[t]], pos[t] + 1);
    written.emplace_back(seq_of_row[t], pos[t]);
  }
  {
    std::vector<std::pair<int, int>> u(written);
    std::sort(u.begin(), u.end());
    if (std::adjacent_find(u.begin(), u.end()) != u.end()) return -1;
  }
  PagedKv c;
  paged_kv_build(c, B, n_tok.data(), kv_heads, stale);
  const int ld = (heads + 2 * kv_heads) * HEAD_DIM;
  const size_t q_bytes = (size_t)T * heads * HEAD_DIM * 2;
  DevBuf dqkv, dk, dv, dcos, dsin, dq, dints;
  if (upload_qkv(dqkv, qkv, splits, T, n_cap, ld) || upload_rope_tables(dcos, dsin, cos_tab, sin_tab, max_pos) ||
      paged_kv_upload(c, dk, dv) || dq.alloc(q_bytes + kGuardBytes))
    return -5;
  ACP_CUDA_CHECK(cudaMemset(dq.p, 0xff, q_bytes + kGuardBytes));
  // packed ints: pos[T] seq_of_row[T] page_off[B+1] page_table[]
  std::vector<int> ints(pos, pos + T);
  ints.insert(ints.end(), seq_of_row, seq_of_row + T);
  ints.insert(ints.end(), c.page_off.begin(), c.page_off.end());
  ints.insert(ints.end(), c.page_table.begin(), c.page_table.end());
  if (dints.alloc(ints.size() * 4)) return -5;
  ACP_CUDA_CHECK(cudaMemcpy(dints.p, ints.data(), ints.size() * 4, cudaMemcpyHostToDevice));
  const int* di = (const int*)dints.p;
  RopeKvArgs ra;
  ra.qkv.ptr = dqkv.p; ra.qkv.splits = splits; ra.qkv.n_cap = n_cap; ra.qkv.ld = ld;
  ra.pos = di; ra.seq_of_row = di + T; ra.page_off = di + 2 * T; ra.page_table = ra.page_off + B + 1;
  ra.cos_tab = (const float*)dcos.p; ra.sin_tab = (const float*)dsin.p; ra.qbuf = (__nv_bfloat16*)dq.p;
  ra.k_cache = (__nv_bfloat16*)dk.p; ra.v_cache = (__nv_bfloat16*)dv.p;
  ra.T = T; ra.heads = heads; ra.kv_heads = kv_heads;
  int rc = launch_rope_kv(ra, 0);
  if (rc != 0) return rc;
  ACP_CUDA_CHECK(cudaDeviceSynchronize());
  if ((rc = check_guard(dq, q_bytes)) != 0) return rc;
  ACP_CUDA_CHECK(cudaMemcpy(q_out, dq.p, q_bytes, cudaMemcpyDeviceToHost));
  return paged_kv_read_back(c, dk, dv, written, k_out, v_out);
}

extern "C" int acp_kernel_gemm_fp8(const uint8_t* w, const float* w_scale, const uint8_t* x, const float* x_scale, int M,
                                   int N, int K, int splits, int epi, int bn, void* out, int iters, float* elapsed_ms) {
  if (acp_kernel_device_count() <= 0) {
    fprintf(stderr, "[acp_infer] no CUDA device: kernels cannot run (no CPU fallback)\n");
    return -5;
  }
  if (!w || !w_scale || !x || !x_scale || !out || M <= 0 || N <= 0 || K <= 0 || epi == EPI_ARGMAX) return -1;
  if (gemm_setup_attributes() != 0) return -5;
  DevBuf dw, dx, dsw, dsx, dout;
  const int n_pad = ((N + 255) / 256) * 256;
  // zero codes pad M and K to (128, 128) multiples; weights go into the engine's tiled e4m3 layout
  const int Mp = ((M + GEMM_BM - 1) / GEMM_BM) * GEMM_BM, Kp = ((K + GEMM_BK_E4M3 - 1) / GEMM_BK_E4M3) * GEMM_BK_E4M3;
  const int nkb_p = Kp / GEMM_BK_E4M3;
  std::vector<uint8_t> wt((size_t)Mp * Kp, 0), xp((size_t)n_pad * Kp, 0);
  for (int r = 0; r < M; ++r)
    for (int c = 0; c < K; ++c)
      wt[((size_t)(r / GEMM_BM) * nkb_p + c / GEMM_BK_E4M3) * (GEMM_BM * GEMM_BK_E4M3) + (size_t)(r % GEMM_BM) * GEMM_BK_E4M3 +
         c % GEMM_BK_E4M3] = w[(size_t)r * K + c];
  for (int r = 0; r < N; ++r) memcpy(&xp[(size_t)r * Kp], &x[(size_t)r * K], (size_t)K);
  if (dw.alloc(wt.size()) || dx.alloc(xp.size()) || dsw.alloc((size_t)Mp * 4) || dsx.alloc((size_t)n_pad * 4)) return -5;
  ACP_CUDA_CHECK(cudaMemcpy(dw.p, wt.data(), wt.size(), cudaMemcpyHostToDevice));
  ACP_CUDA_CHECK(cudaMemcpy(dx.p, xp.data(), xp.size(), cudaMemcpyHostToDevice));
  ACP_CUDA_CHECK(cudaMemcpy(dsw.p, w_scale, (size_t)M * 4, cudaMemcpyHostToDevice));
  ACP_CUDA_CHECK(cudaMemcpy(dsx.p, x_scale, (size_t)N * 4, cudaMemcpyHostToDevice));
  size_t out_bytes = 0;
  if (epi == EPI_BF16) out_bytes = (size_t)N * M * 2;
  else if (epi == EPI_F32) out_bytes = (size_t)splits * N * M * 4;
  else if (epi == EPI_SWIGLU) out_bytes = (size_t)N * (M / 2) * 2;
  else return -1;
  if (dout.alloc(out_bytes + kGuardBytes)) return -5;
  ACP_CUDA_CHECK(cudaMemset(dout.p, 0xff, out_bytes + kGuardBytes));
  TmaMaps mw, mx;
  if (tma_make_weight_e4m3(&mw, dw.p, Mp, Kp) != 0) return -5;
  if (tma_make_act_e4m3(&mx, dx.p, n_pad, Kp) != 0) return -5;
  GemmLaunch g;
  g.w = &mw.w; g.x = &mx; g.M = M; g.N = N; g.K = Kp; g.splits = splits; g.epi = epi;
  g.ld = (epi == EPI_SWIGLU) ? M / 2 : M; g.n_cap = N; g.out = dout.p; g.bn_override = bn;
  g.fp8 = true; g.w_scale = (const float*)dsw.p; g.x_scale = (const float*)dsx.p;
  int rc = gemm_launch(g, 0);
  if (rc != 0) return rc;
  ACP_CUDA_CHECK(cudaDeviceSynchronize());
  if ((rc = check_guard(dout, out_bytes)) != 0) return rc;
  ACP_CUDA_CHECK(cudaMemcpy(out, dout.p, out_bytes, cudaMemcpyDeviceToHost));
  if (iters > 0 && elapsed_ms != nullptr) return time_launches([&] { return gemm_launch(g, 0); }, iters, elapsed_ms);
  return 0;
}

// ---------------------------------------------------------------------------------
// Mixture-of-experts block: the launch sequence of Model::moe_mlp on buffers sized and laid out as alloc_all and
// load_weights make them.  xe / he / ye start as NaN, so a GEMM that reads a row the step does not own turns a
// result NaN, and one that stores past its group leaves a changed row behind.
// ---------------------------------------------------------------------------------
namespace {
// [e_local][rows][cols] row-major -> the engine's tiled layout of the concatenated experts (128 x 64 tiles,
// [m_tile][kb]); `interleave` puts gate row j at 2j and up row j (row rows/2 + j) at 2j + 1 (gu_e_map_)
std::vector<uint16_t> tile_experts(const uint16_t* w, int e_local, int rows, int cols, bool interleave) {
  const int nkb = cols / GEMM_BK;
  std::vector<uint16_t> t((size_t)e_local * rows * cols);
  for (int e = 0; e < e_local; ++e)
    for (int r = 0; r < rows; ++r) {
      const int src = interleave ? (r & 1) * (rows / 2) + (r >> 1) : r;
      const size_t g = (size_t)e * rows + r;   // row of the concatenated tensor
      const uint16_t* s = w + ((size_t)e * rows + src) * cols;
      for (int c = 0; c < cols; c += GEMM_BK)
        memcpy(&t[((g / GEMM_BM) * nkb + c / GEMM_BK) * (GEMM_BM * GEMM_BK) + (g % GEMM_BM) * GEMM_BK], s + c, GEMM_BK * 2);
    }
  return t;
}

// rows [from, rows) of a [rows][cols] bf16 device buffer still hold the 0xffff fill
int check_nan_rows(const DevBuf& d, size_t rows, size_t cols, size_t from, const char* what) {
  std::vector<uint16_t> h((rows - from) * cols);
  ACP_CUDA_CHECK(cudaMemcpy(h.data(), (const uint16_t*)d.p + from * cols, h.size() * 2, cudaMemcpyDeviceToHost));
  for (size_t i = 0; i < h.size(); ++i)
    if (h[i] != 0xffff) {
      fprintf(stderr, "[acp_infer] moe: %s row %zu (past the step's %zu rows) was written\n", what, from + i / cols, from);
      return ACP_ERR_GUARD;
    }
  return 0;
}
}  // namespace

extern "C" int acp_kernel_moe(const uint16_t* xn, const uint16_t* wr, const uint16_t* wgu, const uint16_t* wdown, int T,
                              int hidden, int ffn, int E, int e_first, int e_local, int bn, int t_cap, int partial_f32,
                              const int32_t* topk_in, const float* topk_w_in, int32_t* topk_idx, float* topk_w,
                              int32_t* row_of, int32_t* ranges, int32_t* tiles, int32_t* info, uint16_t* he, uint16_t* ye,
                              void* out) {
  if (int rc = no_device()) return rc;
  if (!xn || !wgu || !wdown || !topk_idx || !topk_w || !row_of || !ranges || !tiles || !info || !he || !ye || !out) return -1;
  if (T < 1 || t_cap < T || 2 * t_cap > 65535 || hidden <= 0 || ffn <= 0 || hidden % GEMM_BM || ffn % GEMM_BK) return -1;
  if (E < 2 || E > GEMM_GROUP_MAX || e_local < 1 || e_first < 0 || e_first + e_local > E) return -1;
  if (bn != 0 && bn != 16 && bn != 32 && bn != 64 && bn != 128 && bn != 256) return -1;
  if ((topk_in == nullptr) != (topk_w_in == nullptr) || (topk_in == nullptr && wr == nullptr)) return -1;
  if (topk_in)
    for (int i = 0; i < 2 * T; ++i)
      if (topk_in[i] < 0 || topk_in[i] >= E) return -1;
  if (gemm_setup_attributes() != 0) return -5;
  if (bn == 0) bn = gemm_pick_bn((2 * T + E - 1) / E);   // as Model::moe_mlp
  const int cap = moe_tile_cap(T, bn, e_local);
  // buffers as Model::alloc_all sizes them for max_tokens_per_step = t_cap
  const int Tp = ((t_cap + 255) / 256) * 256;
  const size_t rows = (size_t)2 * Tp + 256, n_ranges = (size_t)moe_ranges_ints(Tp);
  const size_t out_bytes = (size_t)T * hidden * (partial_f32 ? 4 : 2), tk = (size_t)2 * T * 4;
  DevBuf dxn, dwr, dgu, ddown, dxe, dhe, dye, didx, dw, drow, dranges, dout;
  if (dxn.alloc((size_t)T * hidden * 2) || dgu.alloc((size_t)e_local * 2 * ffn * hidden * 2) ||
      ddown.alloc((size_t)e_local * hidden * ffn * 2) || dxe.alloc(rows * hidden * 2) || dhe.alloc(rows * ffn * 2) ||
      dye.alloc(rows * hidden * 2) || didx.alloc(tk + kGuardBytes) || dw.alloc(tk + kGuardBytes) ||
      drow.alloc(tk + kGuardBytes) || dranges.alloc(n_ranges * 4) || dout.alloc(out_bytes + kGuardBytes))
    return -5;
  ACP_CUDA_CHECK(cudaMemcpy(dxn.p, xn, (size_t)T * hidden * 2, cudaMemcpyHostToDevice));
  {
    const std::vector<uint16_t> t = tile_experts(wgu, e_local, 2 * ffn, hidden, true);
    ACP_CUDA_CHECK(cudaMemcpy(dgu.p, t.data(), t.size() * 2, cudaMemcpyHostToDevice));
  }
  {
    const std::vector<uint16_t> t = tile_experts(wdown, e_local, hidden, ffn, false);
    ACP_CUDA_CHECK(cudaMemcpy(ddown.p, t.data(), t.size() * 2, cudaMemcpyHostToDevice));
  }
  for (DevBuf* d : {&dxe, &dhe, &dye}) ACP_CUDA_CHECK(cudaMemset(d->p, 0xff, (d == &dhe ? rows * ffn : rows * hidden) * 2));
  for (DevBuf* d : {&didx, &dw, &drow}) ACP_CUDA_CHECK(cudaMemset(d->p, 0xff, tk + kGuardBytes));
  ACP_CUDA_CHECK(cudaMemset(dranges.p, 0xff, n_ranges * 4));
  ACP_CUDA_CHECK(cudaMemset(dout.p, 0xff, out_bytes + kGuardBytes));
  TmaMaps mgu, mdown, mxe, mhe;
  if (tma_make_weight(&mgu, dgu.p, (uint64_t)e_local * 2 * ffn, hidden) || tma_make_weight(&mdown, ddown.p, (uint64_t)e_local * hidden, ffn) ||
      tma_make_act(&mxe, dxe.p, rows, hidden) || tma_make_act(&mhe, dhe.p, rows, ffn))
    return -5;
  int* d_idx = (int*)didx.p;
  float* d_w = (float*)dw.p;
  int* d_ranges = (int*)dranges.p;
  int rc = 0;
  if (topk_in) {
    ACP_CUDA_CHECK(cudaMemcpy(d_idx, topk_in, tk, cudaMemcpyHostToDevice));
    ACP_CUDA_CHECK(cudaMemcpy(d_w, topk_w_in, tk, cudaMemcpyHostToDevice));
  } else {
    if (dwr.alloc((size_t)E * hidden * 2)) return -5;
    ACP_CUDA_CHECK(cudaMemcpy(dwr.p, wr, (size_t)E * hidden * 2, cudaMemcpyHostToDevice));
    if ((rc = launch_moe_router((const __nv_bfloat16*)dxn.p, (const __nv_bfloat16*)dwr.p, hidden, E, T, d_idx, d_w, 0))) return rc;
  }
  if ((rc = launch_moe_dispatch(d_idx, T, e_first, e_local, bn, d_ranges, (int*)drow.p, 0)) ||
      (rc = launch_moe_gather((const __nv_bfloat16*)dxn.p, (const int*)drow.p, hidden, T, (__nv_bfloat16*)dxe.p, 0)))
    return rc;
  GemmLaunch g;
  g.groups = e_local; g.group_ranges = d_ranges; g.splits = 1;
  g.bn_override = bn;
  g.N = cap * bn;
  g.w = &mgu.w; g.x = &mxe; g.M = 2 * ffn; g.K = hidden; g.epi = EPI_SWIGLU; g.out = dhe.p; g.ld = ffn; g.n_cap = T;
  if ((rc = gemm_launch(g, 0))) return rc;
  g.w = &mdown.w; g.x = &mhe; g.M = hidden; g.K = ffn; g.epi = EPI_BF16; g.out = dye.p; g.ld = hidden;
  if ((rc = gemm_launch(g, 0))) return rc;
  if ((rc = launch_moe_combine((const __nv_bfloat16*)dye.p, (const int*)drow.p, d_w, hidden, T, dout.p, partial_f32 != 0, 0))) return rc;
  ACP_CUDA_CHECK(cudaDeviceSynchronize());
  for (const DevBuf* d : {&didx, &dw, &drow})
    if ((rc = check_guard(*d, tk))) return rc;
  if ((rc = check_guard(dout, out_bytes))) return rc;
  std::vector<int> rg(n_ranges);
  ACP_CUDA_CHECK(cudaMemcpy(rg.data(), d_ranges, n_ranges * 4, cudaMemcpyDeviceToHost));
  const int n_tiles = rg[GEMM_GROUP_TILES];
  if (n_tiles < 0 || n_tiles > cap) {
    fprintf(stderr, "[acp_infer] moe: %d tiles, capacity %d\n", n_tiles, cap);
    return ACP_ERR_GUARD;
  }
  // every int of `ranges` but the local groups, the tile count and the tile list keeps the -1 fill
  for (size_t i = 0; i < n_ranges; ++i) {
    const bool owned = i < (size_t)2 * e_local || i == (size_t)GEMM_GROUP_TILES ||
                       (i >= (size_t)GEMM_GROUP_TILES + 2 && i < (size_t)GEMM_GROUP_TILES + 2 + 2 * n_tiles);
    if (!owned && rg[i] != -1) {
      fprintf(stderr, "[acp_infer] moe: ranges[%zu] past the tile list was written\n", i);
      return ACP_ERR_GUARD;
    }
  }
  int n_local = 0;
  for (int e = 0; e < e_local; ++e) n_local += rg[2 * e + 1];
  if (n_local < 0 || n_local > 2 * T) return ACP_ERR_GUARD;
  if ((rc = check_nan_rows(dxe, rows, hidden, n_local, "xe")) || (rc = check_nan_rows(dhe, rows, ffn, n_local, "he")) ||
      (rc = check_nan_rows(dye, rows, hidden, n_local, "ye")))
    return rc;
  ACP_CUDA_CHECK(cudaMemcpy(topk_idx, d_idx, tk, cudaMemcpyDeviceToHost));
  ACP_CUDA_CHECK(cudaMemcpy(topk_w, d_w, tk, cudaMemcpyDeviceToHost));
  ACP_CUDA_CHECK(cudaMemcpy(row_of, drow.p, tk, cudaMemcpyDeviceToHost));
  memcpy(ranges, rg.data(), (size_t)2 * e_local * 4);
  memcpy(tiles, rg.data() + GEMM_GROUP_TILES + 2, (size_t)2 * n_tiles * 4);
  info[0] = bn; info[1] = n_tiles; info[2] = n_local; info[3] = cap;
  ACP_CUDA_CHECK(cudaMemcpy(he, dhe.p, (size_t)n_local * ffn * 2, cudaMemcpyDeviceToHost));
  ACP_CUDA_CHECK(cudaMemcpy(ye, dye.p, (size_t)n_local * hidden * 2, cudaMemcpyDeviceToHost));
  ACP_CUDA_CHECK(cudaMemcpy(out, dout.p, out_bytes, cudaMemcpyDeviceToHost));
  return 0;
}

extern "C" int acp_kernel_quantize_fp8(const uint16_t* x, int rows, int cols, uint8_t* codes, float* scales) {
  if (acp_kernel_device_count() <= 0) {
    fprintf(stderr, "[acp_infer] no CUDA device: kernels cannot run (no CPU fallback)\n");
    return -5;
  }
  if (!x || !codes || !scales || rows <= 0 || cols <= 0 || cols % 8) return -1;
  DevBuf dx, dc, ds;
  if (dx.alloc((size_t)rows * cols * 2) || dc.alloc((size_t)rows * cols) || ds.alloc((size_t)rows * 4)) return -5;
  ACP_CUDA_CHECK(cudaMemcpy(dx.p, x, (size_t)rows * cols * 2, cudaMemcpyHostToDevice));
  int rc = launch_quantize_rows_e4m3((const __nv_bfloat16*)dx.p, rows, cols, (uint8_t*)dc.p, (float*)ds.p, 0);
  if (rc != 0) return rc;
  ACP_CUDA_CHECK(cudaDeviceSynchronize());
  ACP_CUDA_CHECK(cudaMemcpy(codes, dc.p, (size_t)rows * cols, cudaMemcpyDeviceToHost));
  ACP_CUDA_CHECK(cudaMemcpy(scales, ds.p, (size_t)rows * 4, cudaMemcpyDeviceToHost));
  return 0;
}
