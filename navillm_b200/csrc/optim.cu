// navillm_b200 — fused gradient-norm clip + AdamW over the flat parameter / gradient buffers ("next" row n3 of
// SURVEY.md §8f).  Replaces train.py:86-89 of the reference:
//     torch.nn.utils.clip_grad_norm_(model.parameters(), 40.); optimizer.step()   (AdamW, tools/optims.py:43)
// which walks ~700 tensors with several elementwise passes each.  Here: one sum-of-squares pass per flat
// buffer, a one-thread kernel that turns the partial sums into the clip coefficient ON THE DEVICE (no host
// sync), and one update pass per buffer that reads p,g,m,v and writes p,m,v once (7 x bytes(p) of HBM traffic).
// Math in fp32; parameters and moments are stored in the parameter dtype (bf16 for the LM, like torch AdamW on
// bf16 parameters; fp32 for the encoder).
// Opt-in for the bf16 buffer: the error-compensated update keeps a bf16 residual r next to each weight p, so the pair
// stands for the master value p + r (about 16 significant bits) and updates far below half a bf16 ulp of p still land.
// It reads p,r,g,m,v and writes p,r,m,v (9 x bytes(p)).
#include "nv_common.cuh"
#include "nv_host.h"

namespace nv {

template <typename T> __device__ __forceinline__ float ldf(const T* p);
template <> __device__ __forceinline__ float ldf<float>(const float* p) { return *p; }
template <> __device__ __forceinline__ float ldf<__nv_bfloat16>(const __nv_bfloat16* p) { return __bfloat162float(*p); }
template <typename T> __device__ __forceinline__ void stf(T* p, float v);
template <> __device__ __forceinline__ void stf<float>(float* p, float v) { *p = v; }
template <> __device__ __forceinline__ void stf<__nv_bfloat16>(__nv_bfloat16* p, float v) { *p = __float2bfloat16_rn(v); }

template <typename T>
__global__ void __launch_bounds__(256) sumsq_kernel(const T* __restrict__ g, int64_t n, float* __restrict__ partial) {
  __shared__ float red[8];
  float s = 0.f;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float v = ldf(g + i);
    s += v * v;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < 8; ++i) t += red[i];
    partial[blockIdx.x] = t;
  }
}

// state[0] = total grad norm, state[1] = clip coefficient = min(1, max_norm / (norm + 1e-6))  (torch semantics)
__global__ void clip_coef_kernel(const float* __restrict__ partial, int n_partial, float max_norm, float* __restrict__ state) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  double t = 0.0;
  for (int i = 0; i < n_partial; ++i) t += (double)partial[i];
  const float norm = (float)sqrt(t);
  state[0] = norm;
  const float c = max_norm / (norm + 1e-6f);
  state[1] = c < 1.f ? c : 1.f;
}

// One element of torch.optim.AdamW in fp32: advances m and v by the (clipped) gradient gi and returns the updated weight x.
// Both update kernels call it, so they round the same way.
__device__ __forceinline__ float adamw_update(float x, float gi, float& mi, float& vi, float lr, float b1, float b2, float eps,
                                              float wd, float bc1, float bc2_sqrt) {
  x *= (1.f - lr * wd);                        // decoupled weight decay
  mi = mi + (1.f - b1) * (gi - mi);            // lerp, like torch
  vi = b2 * vi + (1.f - b2) * gi * gi;
  const float denom = sqrtf(vi) / bc2_sqrt + eps;
  return x - (lr / bc1) * (mi / denom);
}

template <typename T>
__global__ void __launch_bounds__(256) adamw_kernel(T* __restrict__ p, T* __restrict__ g, T* __restrict__ m,
                                                    T* __restrict__ v, int64_t n, float lr, float b1, float b2, float eps,
                                                    float wd, float bc1, float bc2_sqrt, const float* __restrict__ state,
                                                    int write_clipped_grad) {
  const float coef = state ? state[1] : 1.f;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float gi = ldf(g + i) * coef;
    float pi = ldf(p + i);
    float mi = ldf(m + i), vi = ldf(v + i);
    pi = adamw_update(pi, gi, mi, vi, lr, b1, b2, eps, wd, bc1, bc2_sqrt);
    stf(p + i, pi); stf(m + i, mi); stf(v + i, vi);
    if (write_clipped_grad) stf(g + i, gi);      // leave the clipped gradient behind, like clip_grad_norm_
  }
}

// The compensated update of one bf16 element: x = p + r is the master value; p' = bf16_rn(x') and r' = bf16_rn(x' - p')
// (the difference is exact in fp32).  Where x' - p' lies a hair under half an ulp of p', rounding lifts r' onto the tie
// and p' + r' would round to p's neighbour; there r' is rounded toward zero instead, so bf16_rn(p' + r') == p' always.
__device__ __forceinline__ void adamw_compensated_elem(__nv_bfloat16& p, __nv_bfloat16& r, __nv_bfloat16& g, __nv_bfloat16& m,
                                                       __nv_bfloat16& v, float coef, float lr, float b1, float b2, float eps,
                                                       float wd, float bc1, float bc2_sqrt) {
  const float gi = __bfloat162float(g) * coef;
  const float pf = __bfloat162float(p), rf = __bfloat162float(r);
  float mi = __bfloat162float(m), vi = __bfloat162float(v);
  // r == 0 passes p through untouched (no -0 + 0 = +0, no flush of a subnormal p), so the step equals adamw_kernel's bit for bit
  const float x = adamw_update(rf != 0.f ? pf + rf : pf, gi, mi, vi, lr, b1, b2, eps, wd, bc1, bc2_sqrt);
  p = __float2bfloat16_rn(x);
  const float pf2 = __bfloat162float(p), d = x - pf2;
  r = __float2bfloat16_rn(d);
  if (__bfloat16_as_ushort(__float2bfloat16_rn(pf2 + __bfloat162float(r))) != __bfloat16_as_ushort(p)) r = __float2bfloat16_rz(d);
  m = __float2bfloat16_rn(mi);
  v = __float2bfloat16_rn(vi);
  g = __float2bfloat16_rn(gi);
}

union Bf16x8 {
  uint4 u;
  __nv_bfloat16 h[8];
};

// 16-byte accesses: 8 elements per thread per iteration, then a scalar tail of n % 8 elements.  All operands 16-byte aligned.
__global__ void __launch_bounds__(256) adamw_compensated_kernel(__nv_bfloat16* __restrict__ p, __nv_bfloat16* __restrict__ r,
                                                                __nv_bfloat16* __restrict__ g, __nv_bfloat16* __restrict__ m,
                                                                __nv_bfloat16* __restrict__ v, int64_t n, float lr, float b1,
                                                                float b2, float eps, float wd, float bc1, float bc2_sqrt,
                                                                const float* __restrict__ state, int write_clipped_grad) {
  const float coef = state ? state[1] : 1.f;
  const int64_t tid = blockIdx.x * (int64_t)blockDim.x + threadIdx.x, stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t n8 = n / 8;
  for (int64_t i = tid; i < n8; i += stride) {
    Bf16x8 P, R, G, M, V;
    P.u = reinterpret_cast<const uint4*>(p)[i];
    R.u = reinterpret_cast<const uint4*>(r)[i];
    G.u = reinterpret_cast<const uint4*>(g)[i];
    M.u = reinterpret_cast<const uint4*>(m)[i];
    V.u = reinterpret_cast<const uint4*>(v)[i];
#pragma unroll
    for (int j = 0; j < 8; ++j)
      adamw_compensated_elem(P.h[j], R.h[j], G.h[j], M.h[j], V.h[j], coef, lr, b1, b2, eps, wd, bc1, bc2_sqrt);
    reinterpret_cast<uint4*>(p)[i] = P.u;
    reinterpret_cast<uint4*>(r)[i] = R.u;
    reinterpret_cast<uint4*>(m)[i] = M.u;
    reinterpret_cast<uint4*>(v)[i] = V.u;
    if (write_clipped_grad) reinterpret_cast<uint4*>(g)[i] = G.u;
  }
  for (int64_t i = n8 * 8 + tid; i < n; i += stride) {
    __nv_bfloat16 gi = g[i];
    adamw_compensated_elem(p[i], r[i], gi, m[i], v[i], coef, lr, b1, b2, eps, wd, bc1, bc2_sqrt);
    if (write_clipped_grad) g[i] = gi;
  }
}

}  // namespace nv

using namespace nv;
#define S_(x) reinterpret_cast<cudaStream_t>(x)

extern "C" {

int nv_optim_partials(void) { return sm_count() * 8; }

// partial: fp32 [nv_optim_partials()] slice for this buffer (caller concatenates the slices of all buffers)
int nv_grad_sumsq(const void* g, int64_t n, int is_bf16, float* partial, void* stream) {
  const int blocks = sm_count() * 8;
  if (is_bf16) sumsq_kernel<__nv_bfloat16><<<blocks, 256, 0, S_(stream)>>>(reinterpret_cast<const __nv_bfloat16*>(g), n, partial);
  else sumsq_kernel<float><<<blocks, 256, 0, S_(stream)>>>(reinterpret_cast<const float*>(g), n, partial);
  NV_LAUNCH_CHECK();
  return NV_OK;
}

int nv_clip_coef(const float* partial, int n_partial, float max_norm, float* state, void* stream) {
  clip_coef_kernel<<<1, 32, 0, S_(stream)>>>(partial, n_partial, max_norm, state);
  NV_LAUNCH_CHECK();
  return NV_OK;
}

int nv_adamw_flat(void* p, void* g, void* m, void* v, int64_t n, int is_bf16, float lr, float beta1, float beta2, float eps,
                  float weight_decay, int step, const float* clip_state, int write_clipped_grad, void* stream) {
  NV_REQUIRE(step >= 1, "nv_adamw_flat: step must be >= 1");
  const float bc1 = 1.f - powf(beta1, (float)step);
  const float bc2s = sqrtf(1.f - powf(beta2, (float)step));
  const int blocks = sm_count() * 8;
  if (is_bf16)
    adamw_kernel<__nv_bfloat16><<<blocks, 256, 0, S_(stream)>>>(
        reinterpret_cast<__nv_bfloat16*>(p), reinterpret_cast<__nv_bfloat16*>(g), reinterpret_cast<__nv_bfloat16*>(m),
        reinterpret_cast<__nv_bfloat16*>(v), n, lr, beta1, beta2, eps, weight_decay, bc1, bc2s, clip_state, write_clipped_grad);
  else
    adamw_kernel<float><<<blocks, 256, 0, S_(stream)>>>(reinterpret_cast<float*>(p), reinterpret_cast<float*>(g),
                                                        reinterpret_cast<float*>(m), reinterpret_cast<float*>(v), n, lr, beta1,
                                                        beta2, eps, weight_decay, bc1, bc2s, clip_state, write_clipped_grad);
  NV_LAUNCH_CHECK();
  return NV_OK;
}

int nv_adamw_flat_compensated(void* p, void* r, void* g, void* m, void* v, int64_t n, float lr, float beta1, float beta2, float eps,
                              float weight_decay, int step, const float* clip_state, int write_clipped_grad, void* stream) {
  NV_REQUIRE(step >= 1, "nv_adamw_flat_compensated: step must be >= 1");
  NV_REQUIRE(n >= 0, "nv_adamw_flat_compensated: n must be >= 0");
  NV_REQUIRE(((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(r) | reinterpret_cast<uintptr_t>(g) |
               reinterpret_cast<uintptr_t>(m) | reinterpret_cast<uintptr_t>(v)) & 15) == 0,
             "nv_adamw_flat_compensated: p, r, g, m and v must be 16-byte aligned");
  const float bc1 = 1.f - powf(beta1, (float)step);
  const float bc2s = sqrtf(1.f - powf(beta2, (float)step));
  const int blocks = sm_count() * 8;
  using B = __nv_bfloat16;
  adamw_compensated_kernel<<<blocks, 256, 0, S_(stream)>>>(reinterpret_cast<B*>(p), reinterpret_cast<B*>(r), reinterpret_cast<B*>(g),
                                                           reinterpret_cast<B*>(m), reinterpret_cast<B*>(v), n, lr, beta1, beta2,
                                                           eps, weight_decay, bc1, bc2s, clip_state, write_clipped_grad);
  NV_LAUNCH_CHECK();
  return NV_OK;
}

}  // extern "C"
