// nccl_dyn.h — NCCL resolved with dlopen at run time (only engines with "tp" > 1 need it), so
// libacp_infer.so has no link-time dependency on libnccl.  Single-process / one-comm-per-GPU use
// (ncclCommInitAll); collectives run over NVLink / NVSwitch.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

namespace acp {

typedef struct ncclComm* NcclComm;
struct NcclApi {
  bool ok = false;
  int (*CommInitAll)(NcclComm*, int, const int*) = nullptr;
  int (*CommDestroy)(NcclComm) = nullptr;
  int (*AllReduce)(const void*, void*, size_t, int, int, NcclComm, cudaStream_t) = nullptr;
  int (*AllGather)(const void*, void*, size_t, int, NcclComm, cudaStream_t) = nullptr;
  int (*GroupStart)() = nullptr;
  int (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
};
constexpr int kNcclFloat32 = 7;  // ncclFloat32
constexpr int kNcclInt8 = 0;     // ncclInt8 / ncclChar (byte-wise all-gather)
constexpr int kNcclSum = 0;      // ncclSum

const NcclApi& nccl_api();  // loads libnccl.so.2 on first use; ok == false if unavailable

}  // namespace acp
