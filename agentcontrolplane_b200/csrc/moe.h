// moe.h — host launchers of the mixture-of-experts kernels (moe.cu).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>

namespace acp {

// topk_idx[T][2] expert ids (largest logit first), topk_w[T][2] renormalised softmax weights
int launch_moe_router(const __nv_bfloat16* xn, const __nv_bfloat16* wr, int hidden, int E, int T, int* topk_idx,
                      float* topk_w, cudaStream_t s);
// ranges[e_local][2] = {first row, rows} of each local expert in the expert-sorted buffers,
// row_of[T][2] = row of each assignment (-1: the expert lives on another rank)
// Also writes the flat tile list of the grouped GEMMs for N tiles of `bn` rows (layout: GEMM_GROUP_TILES in
// gemm_wgmma.cuh; at most moe_tile_cap(T, bn, e_local) entries).
int launch_moe_dispatch(const int* topk_idx, int T, int e_first, int e_local, int bn, int* ranges, int* row_of, cudaStream_t s);
int moe_ranges_ints(int T);                       // size of the `ranges` array for steps of up to T rows
int moe_tile_cap(int T, int bn, int e_local);     // upper bound of the tile count (grid.x of the grouped GEMMs)
int launch_moe_gather(const __nv_bfloat16* xn, const int* row_of, int hidden, int T, __nv_bfloat16* xe, cudaStream_t s);
// out = bf16 [T][hidden] (one rounding) or, partial_f32, the fp32 sum over this rank's experts
int launch_moe_combine(const __nv_bfloat16* ye, const int* row_of, const float* topk_w, int hidden, int T, void* out,
                       bool partial_f32, cudaStream_t s);

}  // namespace acp
