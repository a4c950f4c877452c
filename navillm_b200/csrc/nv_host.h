// navillm_b200 — host-side helpers shared by the C-ABI translation units (internal).
#pragma once

#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#define NV_OK 0
#define NV_ERR_BAD_ARG (-1)
#define NV_ERR_NO_DEVICE (-2)
#define NV_ERR_UNSUPPORTED (-3)

extern "C" const char* nv_last_error(void);

namespace nv {

void set_error(const char* fmt, ...);

// Returns the positive cudaError_t after recording its string.
int cuda_fail(cudaError_t e, const char* what, const char* file, int line);

#define NV_CUDA(call)                                                          \
  do {                                                                         \
    cudaError_t _e = (call);                                                   \
    if (_e != cudaSuccess) return ::nv::cuda_fail(_e, #call, __FILE__, __LINE__); \
  } while (0)

#define NV_REQUIRE(cond, ...)        \
  do {                               \
    if (!(cond)) {                   \
      ::nv::set_error(__VA_ARGS__);  \
      return NV_ERR_BAD_ARG;         \
    }                                \
  } while (0)

#define NV_LAUNCH_CHECK() NV_CUDA(cudaGetLastError())

int sm_count();

// Programmatic dependent launch switch (nv_set_pdl): when on, the kernels of the decode chain are launched with
// cudaLaunchAttributeProgrammaticStreamSerialization (see griddep_wait / griddep_launch in nv_common.cuh).
extern int g_pdl;

// Batch-invariant split-K (nv_set_fixed_splits): when on, the panorama encoder GEMMs (nv_sgemm, nv_gemm_tf32) take a K split
// count that depends on K alone, not on the tile count (the batch) or sm_count().
extern int g_fixed_splits;

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute at[1];
  if (g_pdl) {
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at;
    cfg.numAttrs = 1;
  }
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

// 2-D tiled tensor map of bf16 (elem_bytes 2), fp32 (4) or raw bytes such as e4m3 (1). `inner` is the contiguous dimension.
// swizzle128: 128-byte swizzle, the box row must be exactly 128 bytes; otherwise unswizzled, box rows a multiple of 16 bytes.
// Out-of-bounds box elements read as zero (and are clipped on store).
int make_tmap_2d(CUtensorMap* out, const void* base, int elem_bytes, uint64_t inner, uint64_t outer,
                 uint64_t outer_stride_bytes, uint32_t box_inner, uint32_t box_outer, bool swizzle128 = true);

}  // namespace nv
