// kernel_tests.cu — C-ABI per-kernel test hooks (include/acp_infer_kernels.h).
// Host buffers in, host buffers out; used only by tests/ to compare each kernel with oracle/.
#include "acp_infer_kernels.h"
#include "common.cuh"
#include "gemm.h"
#include "gemm_wgmma.cuh"
#include "attention.h"
#include <string.h>
#include <vector>

using namespace acp;

namespace {
struct DevBuf {
  void* p = nullptr;
  ~DevBuf() { if (p) cudaFree(p); }
  int alloc(size_t bytes) { return cudaMalloc(&p, bytes ? bytes : 1) == cudaSuccess ? 0 : -5; }
};
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
  if (dout.alloc(out_bytes)) return -5;
  ACP_CUDA_CHECK(cudaMemset(dout.p, 0xff, out_bytes ? out_bytes : 1));
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


extern "C" int acp_kernel_attn_prefill(const uint16_t* q, const uint16_t* k, const uint16_t* v, int heads, int kv_heads,
                                       int q_len, int ctx, int impl, uint16_t* out, int iters, float* elapsed_ms) {
  if (acp_kernel_device_count() <= 0) {
    fprintf(stderr, "[acp_infer] no CUDA device: kernels cannot run (no CPU fallback)\n");
    return -5;
  }
  if (!q || !k || !v || !out || q_len <= 0 || ctx < q_len || heads % kv_heads) return -1;
  if (attn_setup_attributes() != 0) return -5;
  const int n_pages_seq = (ctx + KV_PAGE - 1) / KV_PAGE;
  const int num_pages = n_pages_seq + 3;     // page 0 reserved (all zero), two spare
  const int max_pages = n_pages_seq + 2;
  // shuffled page table: page i of the sequence -> physical page perm[i] in 1..num_pages-1
  std::vector<int> pt(max_pages, 0);
  for (int i = 0; i < n_pages_seq; ++i) pt[i] = 1 + (int)(((long long)i * 7 + 3) % (num_pages - 1));
  {  // make it a permutation (7 may share a factor with num_pages - 1): fall back to reversed order
    std::vector<char> seen(num_pages, 0);
    bool ok = true;
    for (int i = 0; i < n_pages_seq; ++i) { if (seen[pt[i]]) ok = false; seen[pt[i]] = 1; }
    if (!ok) for (int i = 0; i < n_pages_seq; ++i) pt[i] = num_pages - 1 - i;
  }
  const size_t blk_elems = (size_t)KV_PAGE * HEAD_DIM;   // one (page, kv head) block
  std::vector<uint16_t> kc((size_t)num_pages * kv_heads * blk_elems, 0), vc(kc.size(), 0);
  for (int t = 0; t < ctx; ++t)
    for (int h = 0; h < kv_heads; ++h)
      for (int d = 0; d < HEAD_DIM; ++d) {
        const size_t dst = ((size_t)pt[t / KV_PAGE] * kv_heads + h) * blk_elems + (size_t)(d >> 6) * (KV_PAGE * 64) +
                           (size_t)(t % KV_PAGE) * 64 + (d & 63);
        kc[dst] = k[((size_t)t * kv_heads + h) * HEAD_DIM + d];
        vc[dst] = v[((size_t)t * kv_heads + h) * HEAD_DIM + d];
      }
  const int T_cap = ((q_len + 255) / 256) * 256;
  DevBuf dq, dk, dv, dout, dints, dflush;
  const size_t q_elems = (size_t)q_len * heads * HEAD_DIM;
  if (dq.alloc((size_t)T_cap * heads * HEAD_DIM * 2) || dk.alloc(kc.size() * 2) || dv.alloc(vc.size() * 2) ||
      dout.alloc((size_t)T_cap * heads * HEAD_DIM * 2))
    return -5;
  ACP_CUDA_CHECK(cudaMemset(dq.p, 0, (size_t)T_cap * heads * HEAD_DIM * 2));
  ACP_CUDA_CHECK(cudaMemset(dout.p, 0xff, (size_t)T_cap * heads * HEAD_DIM * 2));
  ACP_CUDA_CHECK(cudaMemcpy(dq.p, q, q_elems * 2, cudaMemcpyHostToDevice));
  ACP_CUDA_CHECK(cudaMemcpy(dk.p, kc.data(), kc.size() * 2, cudaMemcpyHostToDevice));
  ACP_CUDA_CHECK(cudaMemcpy(dv.p, vc.data(), vc.size() * 2, cudaMemcpyHostToDevice));
  const int blk_tokens = impl ? attn_prefill_tc_block_tokens(heads, kv_heads) : (16 / (heads / kv_heads)) * 4;
  const int n_blocks = (q_len + blk_tokens - 1) / blk_tokens;
  // packed ints: blk_seq[n_blocks] blk_tok0[n_blocks] q_start[1] q_len[1] ctx_len[1] page_table[max_pages]
  std::vector<int> ints;
  for (int i = 0; i < n_blocks; ++i) ints.push_back(0);
  for (int i = 0; i < n_blocks; ++i) ints.push_back(i * blk_tokens);
  ints.push_back(0); ints.push_back(q_len); ints.push_back(ctx);
  for (int p : pt) ints.push_back(p);
  if (dints.alloc(ints.size() * 4)) return -5;
  ACP_CUDA_CHECK(cudaMemcpy(dints.p, ints.data(), ints.size() * 4, cudaMemcpyHostToDevice));
  const int* di = (const int*)dints.p;
  AttnPrefillArgs pa;
  pa.q = (const __nv_bfloat16*)dq.p; pa.out = (__nv_bfloat16*)dout.p;
  pa.blk_seq = di; pa.blk_tok0 = di + n_blocks; pa.q_start = di + 2 * n_blocks; pa.q_len = di + 2 * n_blocks + 1;
  pa.ctx_len = di + 2 * n_blocks + 2; pa.page_table = di + 2 * n_blocks + 3; pa.max_pages = max_pages;
  pa.heads = heads; pa.kv_heads = kv_heads; pa.scale = 1.0f / sqrtf((float)HEAD_DIM);
  CUtensorMap tq, tk, tv;
  if (impl) {
    if (attn_make_q_map(&tq, dq.p, (uint64_t)T_cap, heads, kv_heads) != 0) return -5;
    if (attn_make_kv_half_map(&tk, dk.p, num_pages, kv_heads) != 0 || attn_make_kv_half_map(&tv, dv.p, num_pages, kv_heads) != 0) return -5;
  } else {
    if (attn_make_kv_map(&tk, dk.p, num_pages, kv_heads) != 0 || attn_make_kv_map(&tv, dv.p, num_pages, kv_heads) != 0) return -5;
  }
  auto launch = [&]() { return impl ? launch_attn_prefill_tc(tq, tk, tv, pa, n_blocks, 0) : launch_attn_prefill(tk, tv, pa, n_blocks, 0); };
  int rc = launch();
  if (rc != 0) return rc;
  ACP_CUDA_CHECK(cudaDeviceSynchronize());
  ACP_CUDA_CHECK(cudaMemcpy(out, dout.p, q_elems * 2, cudaMemcpyDeviceToHost));
  if (iters > 0 && elapsed_ms != nullptr) {
    const size_t flush_n = (size_t)64 << 20;
    if (dflush.alloc(flush_n * 4)) return -5;
    ACP_CUDA_CHECK(cudaMemset(dflush.p, 0, flush_n * 4));
    cudaEvent_t e0, e1;
    ACP_CUDA_CHECK(cudaEventCreate(&e0));
    ACP_CUDA_CHECK(cudaEventCreate(&e1));
    float total = 0.f;
    for (int it = 0; it < iters + 2; ++it) {
      l2_flush_kernel<<<1184, 256>>>((float*)dflush.p, flush_n);
      ACP_CUDA_CHECK(cudaEventRecord(e0, 0));
      rc = launch();
      if (rc != 0) return rc;
      ACP_CUDA_CHECK(cudaEventRecord(e1, 0));
      ACP_CUDA_CHECK(cudaEventSynchronize(e1));
      float ms = 0.f;
      ACP_CUDA_CHECK(cudaEventElapsedTime(&ms, e0, e1));
      if (it >= 2) total += ms;
    }
    *elapsed_ms = total / iters;
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
  }
  return 0;
}
