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

// [rows][cols] row-major, box = one 128-byte swizzle row (64 bf16 or 128 e4m3) x box_rows
static int tma_encode_2d(CUtensorMap* out, bool e4m3, const void* base, uint64_t rows, uint64_t cols, uint32_t box_rows) {
  if (tma_init() != 0) return -5;
  const uint64_t esize = e4m3 ? 1 : 2;
  // innermost dimension first
  cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t gstride[1] = {(cuuint64_t)(cols * esize)};  // bytes, dims 1..rank-1
  cuuint32_t box[2] = {(cuuint32_t)(e4m3 ? GEMM_BK_E4M3 : GEMM_BK), (cuuint32_t)box_rows};
  cuuint32_t estride[2] = {1, 1};
  CUresult r = g_encode(out, e4m3 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), gdim,
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
int tma_encode_2d_bf16(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint32_t box_rows) {
  return tma_encode_2d(out, false, base, rows, cols, box_rows);
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
// FP8 weights use the same tiling with 128 e4m3 per tile row: tile (m_tile, kb) = 128 rows x 128 B.
static int make_weight(TmaMaps* m, bool e4m3, const void* base, uint64_t rows, uint64_t cols) {
  const uint64_t bk = e4m3 ? GEMM_BK_E4M3 : GEMM_BK;
  if (rows % GEMM_BM != 0 || cols % bk != 0) {
    fprintf(stderr, "[acp_infer] tiled weight needs M %% 128 == 0 and K %% %llu == 0 (got %llu x %llu)\n",
            (unsigned long long)bk, (unsigned long long)rows, (unsigned long long)cols);
    return -1;
  }
  const uint64_t tiles = (rows / GEMM_BM) * (cols / bk);
  int rc = tma_encode_2d(&m->w, e4m3, base, tiles * GEMM_BM, bk, GEMM_BM);
  m->has_w = (rc == 0);
  return rc;
}
static int make_act(TmaMaps* m, bool e4m3, const void* base, uint64_t rows, uint64_t cols) {
  for (int i = 0; i < 5; ++i) {
    // NOTE: the box is never clamped to the tensor: the producer always expects the full
    // BN x 128 bytes per stage and TMA zero-fills rows past the end of the tensor.
    const uint32_t box = 16u << i;
    int rc = tma_encode_2d(&m->x[i], e4m3, base, rows, cols, box);
    if (rc != 0) return rc;
  }
  m->has_x = true;
  return 0;
}
int tma_make_weight(TmaMaps* m, const void* base, uint64_t rows, uint64_t cols) { return make_weight(m, false, base, rows, cols); }
int tma_make_act(TmaMaps* m, const void* base, uint64_t rows, uint64_t cols) { return make_act(m, false, base, rows, cols); }
int tma_make_weight_e4m3(TmaMaps* m, const void* base, uint64_t rows, uint64_t cols) { return make_weight(m, true, base, rows, cols); }
int tma_make_act_e4m3(TmaMaps* m, const void* base, uint64_t rows, uint64_t cols) { return make_act(m, true, base, rows, cols); }

int gemm_pick_bn_e4m3(int N) { return N <= 128 ? gemm_pick_bn(N) : 128; }
int gemm_pick_bn(int N) {
  if (N <= 16) return 16;
  if (N <= 32) return 32;
  if (N <= 64) return 64;
  if (N <= 128) return 128;
  return 256;
}

template <int BN, int EPI, bool FP8 = false>
static int launch_one(const GemmLaunch& g, const CUtensorMap& tx, cudaStream_t stream) {
  GemmArgs a;
  a.M = g.M; a.N = g.N; a.K = g.K; a.splits = g.splits; a.ld = g.ld; a.n_cap = g.n_cap;
  a.out = g.out; a.amax_val = g.amax_val; a.amax_idx = g.amax_idx; a.n_dev = g.n_dev;
  a.group_ranges = g.groups > 0 ? g.group_ranges : nullptr;
  a.w_scale = g.w_scale; a.x_scale = g.x_scale;
  // grouped: g.N = the tile-list capacity in ROWS (moe_tile_cap * BN), grid.x walks the flat tile list
  dim3 grid((g.N + BN - 1) / BN, (g.M + GEMM_BM - 1) / GEMM_BM, g.groups > 0 ? 1 : g.splits);
  cudaError_t e = acp_launch(gemm_wx_kernel<BN, EPI, FP8>, grid, dim3(GEMM_THREADS), GemmCfg<BN>::kSmemBytes,
                             stream, *g.w, tx, a);
  if (e != cudaSuccess) {
    fprintf(stderr, "[acp_infer] gemm launch failed BN=%d EPI=%d FP8=%d: %s\n", BN, EPI, (int)FP8,
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
template <int BN>
static int launch_bn_e4m3(const GemmLaunch& g, const CUtensorMap& tx, cudaStream_t stream) {
  switch (g.epi) {
    case EPI_BF16: return launch_one<BN, EPI_BF16, true>(g, tx, stream);
    case EPI_F32: return launch_one<BN, EPI_F32, true>(g, tx, stream);
    case EPI_SWIGLU: return launch_one<BN, EPI_SWIGLU, true>(g, tx, stream);
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

// Co-resident 2-CTA clusters of each persistent instantiation ([FP8][EPI]), from cudaOccupancyMaxActiveClusters
// in gemm_setup_attributes (0 until then).
static int g_pgemm_clusters[2][4] = {};

template <int EPI, bool FP8 = false>
static int launch_persistent(const GemmLaunch& g, cudaStream_t stream) {
  constexpr int BN = FP8 ? PGEMM_BN_E4M3 : PGEMM_BN;
  GemmArgs a;
  a.M = g.M; a.N = g.N; a.K = g.K; a.splits = 1; a.ld = g.ld; a.n_cap = g.n_cap;
  a.out = g.out; a.amax_val = nullptr; a.amax_idx = nullptr; a.n_dev = g.n_dev;
  a.group_ranges = nullptr;
  a.w_scale = g.w_scale; a.x_scale = g.x_scale;
  const int m_tiles = (g.M + GEMM_BM - 1) / GEMM_BM, n_tiles = (g.N + BN - 1) / BN;
  const int max_clusters = g_pgemm_clusters[FP8][EPI];
  if (max_clusters <= 0) {
    fprintf(stderr, "[acp_infer] persistent gemm: no co-resident cluster count (gemm_setup_attributes not run)\n");
    return -5;
  }
  int clusters = ((m_tiles + 1) / 2) * n_tiles;   // one cluster per pair of m-tiles of an n-tile
  if (clusters > max_clusters) clusters = max_clusters;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(2 * clusters);
  cfg.blockDim = dim3(GEMM_THREADS);
  cfg.dynamicSmemBytes = PGemmSmem<EPI, FP8>;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 2; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
  attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[1].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = acp_pdl_enabled() ? 2 : 1;
  // X in halves of BN / 2 token rows, one per CTA of the cluster (box 128 rows for bf16, 64 for FP8)
  cudaError_t e = cudaLaunchKernelEx(&cfg, gemm_wx_persistent_kernel<EPI, FP8>, *g.w, g.x->x[FP8 ? 2 : 3], a, m_tiles, n_tiles);
  if (e != cudaSuccess) {
    fprintf(stderr, "[acp_infer] persistent gemm launch failed EPI=%d: %s\n", EPI, cudaGetErrorString(e));
    return -5;
  }
  return 0;
}

static int gemm_launch_e4m3(const GemmLaunch& g, cudaStream_t stream) {
  if (g.groups > 0 || g.epi == EPI_ARGMAX || g.w_scale == nullptr || g.x_scale == nullptr || g.bn_override > 128) return -1;
  if (gemm_path(g) == GEMM_PATH_PERSISTENT)
    return g.epi == EPI_BF16 ? launch_persistent<EPI_BF16, true>(g, stream)
           : g.epi == EPI_F32 ? launch_persistent<EPI_F32, true>(g, stream) : launch_persistent<EPI_SWIGLU, true>(g, stream);
  const int bn = g.bn_override > 0 ? g.bn_override : gemm_pick_bn_e4m3(g.N);
  switch (bn) {
    case 16: return launch_bn_e4m3<16>(g, g.x->x[0], stream);
    case 32: return launch_bn_e4m3<32>(g, g.x->x[1], stream);
    case 64: return launch_bn_e4m3<64>(g, g.x->x[2], stream);
    case 128: return launch_bn_e4m3<128>(g, g.x->x[3], stream);
  }
  return -1;
}

int gemm_launch(const GemmLaunch& g, cudaStream_t stream) {
  if (g.N <= 0 || g.M <= 0) return 0;
  if (g.epi != EPI_F32 && g.splits != 1) return -1;
  if (g.fp8) return gemm_launch_e4m3(g, stream);
  // grouped: group g's weights are whole m-tiles g * M / 128 .. of the concatenated tensor, so M % 128 == 0
  if (g.groups > 0 && (g.splits != 1 || g.group_ranges == nullptr || (g.epi != EPI_BF16 && g.epi != EPI_SWIGLU) ||
                       g.groups > GEMM_GROUP_MAX || g.M % GEMM_BM || g.K % GEMM_BK))
    return -1;
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

template <int BN, int EPI, bool FP8 = false>
static int set_attr() {
  return cudaFuncSetAttribute(gemm_wx_kernel<BN, EPI, FP8>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                              GemmCfg<BN>::kSmemBytes) == cudaSuccess ? 0 : -5;
}
template <int BN>
static int set_attr_bn() {
  int rc = set_attr<BN, EPI_BF16>() | set_attr<BN, EPI_F32>() | set_attr<BN, EPI_ARGMAX>() | set_attr<BN, EPI_SWIGLU>();
  if constexpr (BN <= 128) rc |= set_attr<BN, EPI_BF16, true>() | set_attr<BN, EPI_F32, true>() | set_attr<BN, EPI_SWIGLU, true>();
  return rc;
}
template <int EPI, bool FP8>
static int set_attr_persistent() {
  constexpr int bytes = PGemmSmem<EPI, FP8>;
  if (cudaFuncSetAttribute(gemm_wx_persistent_kernel<EPI, FP8>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes) != cudaSuccess)
    return -5;
  // how many 2-CTA clusters of this kernel fit on the device at once (the persistent grid)
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(2 * GEMM_SMS);
  cfg.blockDim = dim3(GEMM_THREADS);
  cfg.dynamicSmemBytes = bytes;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 2; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  int clusters = 0;
  cudaError_t e = cudaOccupancyMaxActiveClusters(&clusters, gemm_wx_persistent_kernel<EPI, FP8>, &cfg);
  if (e != cudaSuccess || clusters <= 0) {
    fprintf(stderr, "[acp_infer] cudaOccupancyMaxActiveClusters(persistent gemm EPI=%d FP8=%d) = %d: %s\n", EPI, (int)FP8, clusters,
            cudaGetErrorString(e));
    return -5;
  }
  g_pgemm_clusters[FP8][EPI] = clusters;
  return 0;
}
int gemm_persistent_clusters(bool fp8, int epi) { return (epi >= 0 && epi < 4) ? g_pgemm_clusters[fp8][epi] : 0; }
int gemm_setup_attributes() {
  int rc = set_attr_bn<16>() | set_attr_bn<32>() | set_attr_bn<64>() | set_attr_bn<128>() |
           set_attr_bn<256>();
  rc |= set_attr_persistent<EPI_F32, false>() | set_attr_persistent<EPI_BF16, false>() | set_attr_persistent<EPI_SWIGLU, false>() |
        set_attr_persistent<EPI_F32, true>() | set_attr_persistent<EPI_BF16, true>() | set_attr_persistent<EPI_SWIGLU, true>();
  if (rc != 0) fprintf(stderr, "[acp_infer] cudaFuncSetAttribute(max dyn smem) failed\n");
  return rc;
}

}  // namespace acp
