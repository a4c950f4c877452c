// navillm_b200 — C-ABI runtime: error reporting, device query, TMA tensor-map encoding.
//
// The library allocates no device memory of its own: every buffer (inputs, outputs, workspaces) is
// owned by the caller (the PyTorch caching allocator in the Python host).  There is deliberately NO
// CPU fallback anywhere in this library: with no sm_90 device every compute entry point fails with
// NV_ERR_NO_DEVICE (north star: "no CPU fallback").
#include "nv_host.h"

#include <stdarg.h>
#include <string.h>

#include <mutex>

namespace nv {

static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int cuda_fail(cudaError_t e, const char* what, const char* file, int line) {
  set_error("CUDA error %d (%s) at %s:%d in `%s`", (int)e, cudaGetErrorString(e), file, line, what);
  return (int)e;
}

int g_pdl = 0;

int sm_count() {
  static int n = -1;
  if (n < 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 0;
    cudaDeviceProp p;
    if (cudaGetDeviceProperties(&p, dev) != cudaSuccess) return 0;
    n = p.multiProcessorCount;
  }
  return n;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    // Resolved at run time so the shared library has no link-time dependency on libcuda.so.1 and can
    // be dlopen()ed on a GPU-less build machine (symbol-export test).
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

int make_tmap_2d(CUtensorMap* out, const void* base, int elem_bytes, uint64_t inner, uint64_t outer,
                 uint64_t outer_stride_bytes, uint32_t box_inner, uint32_t box_outer, bool swizzle128) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) {
    set_error("cuTensorMapEncodeTiled unavailable (no CUDA driver / no GPU)");
    return NV_ERR_NO_DEVICE;
  }
  NV_REQUIRE((reinterpret_cast<uintptr_t>(base) & 15) == 0, "TMA base pointer %p not 16-byte aligned", base);
  NV_REQUIRE((outer_stride_bytes & 15) == 0, "TMA row stride %llu B not a multiple of 16",
             (unsigned long long)outer_stride_bytes);
  NV_REQUIRE(elem_bytes == 1 || elem_bytes == 2 || elem_bytes == 4, "TMA element size %d not supported", elem_bytes);
  if (swizzle128)
    NV_REQUIRE(box_inner * elem_bytes == 128, "TMA box inner extent must be 128 bytes (got %u)", box_inner * elem_bytes);
  else
    NV_REQUIRE((box_inner * elem_bytes) % 16 == 0 && box_inner <= 256, "TMA box inner extent %u B not a multiple of 16",
               box_inner * elem_bytes);
  NV_REQUIRE(box_outer >= 1 && box_outer <= 256, "TMA box outer extent %u out of range", box_outer);
  const CUtensorMapDataType dt = elem_bytes == 1   ? CU_TENSOR_MAP_DATA_TYPE_UINT8
                                 : elem_bytes == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                                                   : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {outer_stride_bytes};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(out, dt, 2, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed: CUresult %d (inner=%llu outer=%llu stride=%llu box=%ux%u)", (int)r,
              (unsigned long long)inner, (unsigned long long)outer, (unsigned long long)outer_stride_bytes,
              box_inner, box_outer);
    return NV_ERR_BAD_ARG;
  }
  return NV_OK;
}

}  // namespace nv

extern "C" {

const char* nv_last_error(void) { return nv::g_err; }

int nv_abi_version(void) { return 1; }

int nv_set_pdl(int on) {
  const int prev = nv::g_pdl;
  nv::g_pdl = on ? 1 : 0;
  return prev;
}

// 0 when an sm_90 (Hopper) device is current, NV_ERR_NO_DEVICE otherwise.
int nv_device_check(void) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) {
    cudaGetLastError();
    nv::set_error("no CUDA device: %s", cudaGetErrorString(e));
    return NV_ERR_NO_DEVICE;
  }
  cudaDeviceProp p;
  e = cudaGetDeviceProperties(&p, dev);
  if (e != cudaSuccess) {
    cudaGetLastError();
    nv::set_error("cudaGetDeviceProperties: %s", cudaGetErrorString(e));
    return NV_ERR_NO_DEVICE;
  }
  if (p.major != 9 || p.minor != 0) {
    nv::set_error("device %d is sm_%d%d; this library is built for sm_90a only", dev, p.major, p.minor);
    return NV_ERR_NO_DEVICE;
  }
  return NV_OK;
}

int nv_sm_count(void) { return nv::sm_count(); }

}  // extern "C"
