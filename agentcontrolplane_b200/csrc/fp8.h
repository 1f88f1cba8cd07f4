// fp8.h — the row quantiser of the FP8 (e4m3) presets on the device (DESIGN.md §5):
//   amax = max|x|,  s = fp32(amax / 448) (1 when amax == 0),  code = e4m3_rne(clamp(fp32(x / s), -448, 448))
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>

namespace acp {

// Activations: rows [0, rows) of a row-major bf16 [.][cols] matrix -> e4m3 codes [.][cols] + scales [rows].
int launch_quantize_rows_e4m3(const __nv_bfloat16* x, int rows, int cols, uint8_t* codes, float* scales,
                              cudaStream_t stream);
// Weights: a tiled bf16 [M][K] matrix (128 x 64 tiles, gemm.cu) -> tiled e4m3 codes (128 x 128 tiles) + s_w [M].
int launch_quantize_weight_e4m3(const __nv_bfloat16* w_tiled, int M, int K, uint8_t* codes_tiled, float* scales,
                                cudaStream_t stream);

}  // namespace acp
