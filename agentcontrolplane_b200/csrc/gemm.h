// gemm.h — host interface of the wgmma GEMM (see gemm_wgmma.cuh for the kernels).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace acp {

// TMA descriptors of one bf16 [rows][cols] row-major matrix, one per supported N-tile.
// idx 0..4 <-> box rows 16, 32, 64, 128, 256; `w` is the 128-row box used for weights.
struct TmaMaps {
  CUtensorMap w;       // box {64, 128}
  CUtensorMap x[5];    // box {64, 16 << i}
  bool has_w = false, has_x = false;
};

int tma_init();  // resolves cuTensorMapEncodeTiled through cudart; 0 on success
int tma_encode_2d_bf16(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols,
                       uint32_t box_rows);
// 3-D bf16 tensor {d0 (contiguous), d1, d2} with byte strides {d0*2 for d1, d0*d1*2 for d2}, 128-byte swizzle
int tma_encode_3d_bf16(CUtensorMap* out, const void* base, uint64_t d0, uint64_t d1, uint64_t d2,
                       uint32_t box0, uint32_t box1, uint32_t box2);
int tma_make_weight(TmaMaps* m, const void* base, uint64_t rows, uint64_t cols);
int tma_make_act(TmaMaps* m, const void* base, uint64_t rows, uint64_t cols);

struct GemmLaunch {
  const CUtensorMap* w = nullptr;  // weight map (box 128 rows)
  const TmaMaps* x = nullptr;      // activation maps
  int M = 0, N = 0, K = 0;
  int splits = 1;
  int epi = 0;          // GemmEpi
  int ld = 0;           // output leading dim
  int n_cap = 0;        // partial-plane row capacity
  void* out = nullptr;
  float* amax_val = nullptr;
  int* amax_idx = nullptr;
  const int* n_dev = nullptr;
  int bn_override = 0;  // 0 = pick from N; < 0 = force the persistent kernel (N > 256)
  // a tensor-parallel shard's GEMM: the fp32 plane of the row-parallel projections stays on the tiled kernel
  // unless ACP_TP_GEMM_PERSISTENT_F32=1 — see gemm.cu gemm_path
  bool tp_shard = false;
  // grouped mode (mixture of experts): `groups` weight tensors of M rows each, concatenated in `w`;
  // group g works on rows [ranges[2g], ranges[2g] + ranges[2g+1]) of x / out (device array, layout of
  // moe_dispatch_kernel incl. its flat tile list).  bn_override = the tile height the list was built for,
  // N = tile capacity * bn_override (grid.x = capacity).
  int groups = 0;
  const int* group_ranges = nullptr;
};
int gemm_pick_bn(int N);
int gemm_launch(const GemmLaunch& g, cudaStream_t stream);
enum { GEMM_PATH_TILED = 0, GEMM_PATH_PERSISTENT = 1 };
int gemm_path(const GemmLaunch& g);   // the kernel gemm_launch would pick for this problem
int gemm_setup_attributes();  // cudaFuncSetAttribute for every instantiation (once per device)

}  // namespace acp
