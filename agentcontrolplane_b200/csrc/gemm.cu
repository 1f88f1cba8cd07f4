// gemm.cu — host side of the wgmma GEMM: TMA descriptor construction and launch dispatch.
#include "gemm.h"
#include "gemm_wgmma.cuh"
#include <cudaTypedefs.h>
#include <mutex>
#include <stdlib.h>

namespace acp {

static PFN_cuTensorMapEncodeTiled_v12000 g_encode = nullptr;

int tma_init() {
  static std::once_flag once;
  static int rc = 0;
  std::call_once(once, [] {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
    if (e != cudaSuccess || fn == nullptr || qres != cudaDriverEntryPointSuccess) {
      fprintf(stderr, "[acp_infer] cuTensorMapEncodeTiled unavailable: %s\n",
              cudaGetErrorString(e));
      rc = -5;
      return;
    }
    g_encode = (PFN_cuTensorMapEncodeTiled_v12000)fn;
  });
  return rc;
}

int tma_encode_2d_bf16(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols,
                       uint32_t box_rows) {
  if (tma_init() != 0) return -5;
  // innermost dimension first
  cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t gstride[1] = {(cuuint64_t)cols * 2};  // bytes, dims 1..rank-1
  cuuint32_t box[2] = {(cuuint32_t)GEMM_BK, (cuuint32_t)box_rows};
  cuuint32_t estride[2] = {1, 1};
  CUresult r = g_encode(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), gdim,
                        gstride, box, estride, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    fprintf(stderr, "[acp_infer] cuTensorMapEncodeTiled failed (%d) rows=%llu cols=%llu box=%u\n",
            (int)r, (unsigned long long)rows, (unsigned long long)cols, box_rows);
    return -5;
  }
  return 0;
}

int tma_encode_3d_bf16(CUtensorMap* out, const void* base, uint64_t d0, uint64_t d1, uint64_t d2,
                       uint32_t box0, uint32_t box1, uint32_t box2) {
  if (tma_init() != 0) return -5;
  cuuint64_t gdim[3] = {(cuuint64_t)d0, (cuuint64_t)d1, (cuuint64_t)d2};
  cuuint64_t gstride[2] = {(cuuint64_t)d0 * 2, (cuuint64_t)d0 * d1 * 2};
  cuuint32_t box[3] = {box0, box1, box2};
  cuuint32_t estride[3] = {1, 1, 1};
  CUresult r = g_encode(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), gdim, gstride, box, estride,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    fprintf(stderr, "[acp_infer] cuTensorMapEncodeTiled(3d) failed (%d) dims=%llu x %llu x %llu box=%u x %u x %u\n", (int)r,
            (unsigned long long)d0, (unsigned long long)d1, (unsigned long long)d2, box0, box1, box2);
    return -5;
  }
  return 0;
}

// Weights are stored TILED in HBM: tile (m_tile, kb) = 128 rows x 64 bf16 = 16 KiB CONTIGUOUS,
// tiles ordered [m_tile][kb].  One TMA box is then one contiguous 16 KiB read (DRAM-page friendly)
// instead of 128 segments of 128 B strided by a whole weight row.  Seen by TMA as a 2-D tensor
// [(M/128)*(K/64)*128 rows][64 cols].
int tma_make_weight(TmaMaps* m, const void* base, uint64_t rows, uint64_t cols) {
  if (rows % GEMM_BM != 0 || cols % GEMM_BK != 0) {
    fprintf(stderr, "[acp_infer] tiled weight needs M %% 128 == 0 and K %% 64 == 0 (got %llu x %llu)\n",
            (unsigned long long)rows, (unsigned long long)cols);
    return -1;
  }
  const uint64_t tiles = (rows / GEMM_BM) * (cols / GEMM_BK);
  int rc = tma_encode_2d_bf16(&m->w, base, tiles * GEMM_BM, GEMM_BK, GEMM_BM);
  m->has_w = (rc == 0);
  return rc;
}
int tma_make_act(TmaMaps* m, const void* base, uint64_t rows, uint64_t cols) {
  for (int i = 0; i < 5; ++i) {
    // NOTE: the box is never clamped to the tensor: the producer always expects the full
    // BN x 128 bytes per stage and TMA zero-fills rows past the end of the tensor.
    const uint32_t box = 16u << i;
    int rc = tma_encode_2d_bf16(&m->x[i], base, rows, cols, box);
    if (rc != 0) return rc;
  }
  m->has_x = true;
  return 0;
}

int gemm_pick_bn(int N) {
  if (N <= 16) return 16;
  if (N <= 32) return 32;
  if (N <= 64) return 64;
  if (N <= 128) return 128;
  return 256;
}

template <int BN, int EPI>
static int launch_one(const GemmLaunch& g, const CUtensorMap& tx, cudaStream_t stream) {
  GemmArgs a;
  a.M = g.M; a.N = g.N; a.K = g.K; a.splits = g.splits; a.ld = g.ld; a.n_cap = g.n_cap;
  a.out = g.out; a.amax_val = g.amax_val; a.amax_idx = g.amax_idx; a.n_dev = g.n_dev;
  a.group_ranges = g.groups > 0 ? g.group_ranges : nullptr;
  // grouped: g.N = the tile-list capacity in ROWS (moe_tile_cap * BN), grid.x walks the flat tile list
  dim3 grid((g.N + BN - 1) / BN, (g.M + GEMM_BM - 1) / GEMM_BM, g.groups > 0 ? 1 : g.splits);
  cudaError_t e = acp_launch(gemm_wx_kernel<BN, EPI>, grid, dim3(GEMM_THREADS), GemmCfg<BN>::kSmemBytes,
                             stream, *g.w, tx, a);
  if (e != cudaSuccess) {
    fprintf(stderr, "[acp_infer] gemm launch failed BN=%d EPI=%d: %s\n", BN, EPI,
            cudaGetErrorString(e));
    return -5;
  }
  return 0;
}

template <int BN>
static int launch_bn(const GemmLaunch& g, const CUtensorMap& tx, cudaStream_t stream) {
  switch (g.epi) {
    case EPI_BF16: return launch_one<BN, EPI_BF16>(g, tx, stream);
    case EPI_F32: return launch_one<BN, EPI_F32>(g, tx, stream);
    case EPI_ARGMAX: return launch_one<BN, EPI_ARGMAX>(g, tx, stream);
    case EPI_SWIGLU: return launch_one<BN, EPI_SWIGLU>(g, tx, stream);
  }
  return -1;
}

static bool persistent_enabled() {
  static int v = -1;
  if (v < 0) { const char* e = getenv("ACP_GEMM_PERSISTENT"); v = (e && *e == '0') ? 0 : 1; }
  return v == 1;
}

// Which kernel gemm_launch picks (pure host logic: tests/test_abi_cpu.py pins the defaults without a GPU):
// prefill-sized problems (N > 256; bf16, fused-SwiGLU or ONE fp32 plane out; not grouped) run the persistent
// kernel, everything else the tiled one.  bn_override < 0 forces the persistent kernel (test hook).
// Tensor-parallel shards keep the fp32 plane of the row-parallel projections on the tiled kernel unless
// ACP_TP_GEMM_PERSISTENT_F32=1.
int gemm_path(const GemmLaunch& g) {
  static const bool tp_f32 = [] { const char* e = getenv("ACP_TP_GEMM_PERSISTENT_F32"); return e && *e == '1'; }();
  const bool f32_ok = g.epi == EPI_F32 && g.splits == 1 && (!g.tp_shard || tp_f32);
  if (g.N > 256 && g.bn_override <= 0 && g.groups == 0 && (persistent_enabled() || g.bn_override < 0) &&
      (g.epi == EPI_BF16 || g.epi == EPI_SWIGLU || f32_ok))
    return GEMM_PATH_PERSISTENT;
  return GEMM_PATH_TILED;
}

template <int EPI>
static int launch_persistent(const GemmLaunch& g, cudaStream_t stream) {
  GemmArgs a;
  a.M = g.M; a.N = g.N; a.K = g.K; a.splits = 1; a.ld = g.ld; a.n_cap = g.n_cap;
  a.out = g.out; a.amax_val = nullptr; a.amax_idx = nullptr; a.n_dev = g.n_dev;
  a.group_ranges = nullptr;
  const int m_tiles = (g.M + GEMM_BM - 1) / GEMM_BM, n_tiles = (g.N + PGEMM_BN - 1) / PGEMM_BN;
  int grid = m_tiles * n_tiles;
  if (grid > GEMM_SMS) grid = GEMM_SMS;  // one persistent CTA per SM
  cudaError_t e = acp_launch(gemm_wx_persistent_kernel<EPI>, dim3(grid), dim3(GEMM_THREADS), PGemmCfg::kSmemBytes, stream,
                             *g.w, g.x->x[4], a, m_tiles, n_tiles);
  if (e != cudaSuccess) {
    fprintf(stderr, "[acp_infer] persistent gemm launch failed EPI=%d: %s\n", EPI, cudaGetErrorString(e));
    return -5;
  }
  return 0;
}

int gemm_launch(const GemmLaunch& g, cudaStream_t stream) {
  if (g.N <= 0 || g.M <= 0) return 0;
  if (g.epi != EPI_F32 && g.splits != 1) return -1;
  if (g.groups > 0 && (g.splits != 1 || g.group_ranges == nullptr || (g.epi != EPI_BF16 && g.epi != EPI_SWIGLU))) return -1;
  switch (gemm_path(g)) {
    case GEMM_PATH_PERSISTENT:
      return g.epi == EPI_BF16 ? launch_persistent<EPI_BF16>(g, stream)
             : g.epi == EPI_F32 ? launch_persistent<EPI_F32>(g, stream) : launch_persistent<EPI_SWIGLU>(g, stream);
    default: break;
  }
  const int bn = g.bn_override > 0 ? g.bn_override : gemm_pick_bn(g.N);
  switch (bn) {
    case 16: return launch_bn<16>(g, g.x->x[0], stream);
    case 32: return launch_bn<32>(g, g.x->x[1], stream);
    case 64: return launch_bn<64>(g, g.x->x[2], stream);
    case 128: return launch_bn<128>(g, g.x->x[3], stream);
    case 256: return launch_bn<256>(g, g.x->x[4], stream);
  }
  return -1;
}

template <int BN, int EPI>
static int set_attr() {
  return cudaFuncSetAttribute(gemm_wx_kernel<BN, EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                              GemmCfg<BN>::kSmemBytes) == cudaSuccess ? 0 : -5;
}
template <int BN>
static int set_attr_bn() {
  return set_attr<BN, EPI_BF16>() | set_attr<BN, EPI_F32>() | set_attr<BN, EPI_ARGMAX>() |
         set_attr<BN, EPI_SWIGLU>();
}
int gemm_setup_attributes() {
  int rc = set_attr_bn<16>() | set_attr_bn<32>() | set_attr_bn<64>() | set_attr_bn<128>() |
           set_attr_bn<256>();
  if (cudaFuncSetAttribute(gemm_wx_persistent_kernel<EPI_F32>, cudaFuncAttributeMaxDynamicSharedMemorySize, PGemmCfg::kSmemBytes) != cudaSuccess ||
      cudaFuncSetAttribute(gemm_wx_persistent_kernel<EPI_BF16>, cudaFuncAttributeMaxDynamicSharedMemorySize, PGemmCfg::kSmemBytes) != cudaSuccess ||
      cudaFuncSetAttribute(gemm_wx_persistent_kernel<EPI_SWIGLU>, cudaFuncAttributeMaxDynamicSharedMemorySize, PGemmCfg::kSmemBytes) != cudaSuccess)
    rc = -5;
  if (rc != 0) fprintf(stderr, "[acp_infer] cudaFuncSetAttribute(max dyn smem) failed\n");
  return rc;
}

}  // namespace acp
