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
// Opt-in for the bf16 buffer: block-wise 8-bit moments (1 byte per element of m and of v, plus one fp32 absmax per 64
// elements each), with or without the residual: it reads p,g,codes,absmax and writes p,codes,absmax, 10.25 bytes per
// element against 14 (14.25 against 18 with the residual).
#include <algorithm>

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
// pf and rf are p and r as read, gi is the clipped gradient; the moments come in and go out as fp32, so each kernel stores
// them in its own format.
__device__ __forceinline__ void adamw_compensated_elem(__nv_bfloat16& p, __nv_bfloat16& r, float pf, float rf, float gi,
                                                       float& mi, float& vi, float lr, float b1, float b2, float eps, float wd,
                                                       float bc1, float bc2_sqrt) {
  // r == 0 passes p through untouched (no -0 + 0 = +0, no flush of a subnormal p), so the step equals adamw_kernel's bit for bit
  const float x = adamw_update(rf != 0.f ? pf + rf : pf, gi, mi, vi, lr, b1, b2, eps, wd, bc1, bc2_sqrt);
  p = __float2bfloat16_rn(x);
  const float pf2 = __bfloat162float(p), d = x - pf2;
  r = __float2bfloat16_rn(d);
  if (__bfloat16_as_ushort(__float2bfloat16_rn(pf2 + __bfloat162float(r))) != __bfloat16_as_ushort(p)) r = __float2bfloat16_rz(d);
}

// ... with bf16 moments, for adamw_compensated_kernel
__device__ __forceinline__ void adamw_compensated_elem(__nv_bfloat16& p, __nv_bfloat16& r, __nv_bfloat16& g, __nv_bfloat16& m,
                                                       __nv_bfloat16& v, float coef, float lr, float b1, float b2, float eps,
                                                       float wd, float bc1, float bc2_sqrt) {
  const float gi = __bfloat162float(g) * coef;
  const float pf = __bfloat162float(p), rf = __bfloat162float(r);
  float mi = __bfloat162float(m), vi = __bfloat162float(v);
  adamw_compensated_elem(p, r, pf, rf, gi, mi, vi, lr, b1, b2, eps, wd, bc1, bc2_sqrt);
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

// ---- block-wise 8-bit moments (Dettmers et al., "8-bit Optimizers via Block-wise Quantization", ICLR 2022) ------------
// Each 64-element block of a moment is one fp32 absmax and 64 uint8 codes; the value of a code is map[code] * absmax.
// navillm_b200/optim.py builds the two sorted 256-entry maps (signed for m, unsigned for v) and owns the format; the
// kernels read them.  The signed map is symmetric: map[127 - k] == -map[128 + k], 128 is the code of 0 and 127 a spare
// duplicate of 0 that is never produced.  The unsigned map starts with 0 and ends with 1.  A block's absmax element
// quantizes to +-1, so it is stored exactly.
constexpr int QBLK = 64;
constexpr int M_ZERO = 128;

// Shared-memory copy of the maps plus each searched range in Eytzinger (breadth-first) order, so that the probes of one
// binary-search level sit side by side in the banks: the magnitude half of the signed map (map[128 .. 255]) and the
// unsigned map.
struct QMaps {
  float map[512];        // signed (m) then unsigned (v), sorted
  float eyt_m[128];      // eyt[node], node in [1, 128): probe of that node of the search over map[128 .. 255]
  float eyt_v[256];
};

template <int LEN>
__device__ __forceinline__ void build_eytzinger(float* eyt, const float* tab) {
  for (int node = 1 + threadIdx.x; node < LEN; node += blockDim.x) {
    const int k = 31 - __clz(node), j = node - (1 << k), s = LEN >> (k + 1);
    eyt[node] = tab[(2 * j + 1) * s];
  }
}

__device__ __forceinline__ void load_qmaps(QMaps& q, const float* __restrict__ maps) {
  for (int i = threadIdx.x; i < 512; i += blockDim.x) q.map[i] = maps[i];
  build_eytzinger<128>(q.eyt_m, maps + M_ZERO);
  build_eytzinger<256>(q.eyt_v, maps + 256);
  __syncthreads();
}

// Index of the entry of tab[0 .. LEN) (ascending, tab[0] = 0) nearest to y >= 0; a tie goes to the smaller entry.
template <int LEN>
__device__ __forceinline__ int nearest_entry(const float* tab, const float* eyt, float y) {
  int node = 1;
#pragma unroll
  for (int s = LEN / 2; s > 0; s >>= 1) node = 2 * node + (eyt[node] <= y ? 1 : 0);
  const int i = node - LEN;                                   // the largest i with tab[i] <= y
  return (i + 1 < LEN && tab[i + 1] - y < y - tab[i]) ? i + 1 : i;
}

// y = x / absmax with an IEEE division (the build uses --use_fast_math); a block whose absmax is 0 stores code 0
__device__ __forceinline__ uint8_t quantize_m(const QMaps& q, float x, float amax) {
  if (amax == 0.f) return 0;
  const float y = __fdiv_rn(x, amax);
  const int k = nearest_entry<128>(q.map + M_ZERO, q.eyt_m, fabsf(y));
  return (uint8_t)(y < 0.f && k > 0 ? M_ZERO - 1 - k : M_ZERO + k);
}

__device__ __forceinline__ uint8_t quantize_v(const QMaps& q, float x, float amax) {
  if (amax == 0.f) return 0;
  return (uint8_t)nearest_entry<256>(q.map + 256, q.eyt_v, __fdiv_rn(x, amax));
}

// One bf16 weight's update with fp32 moments: adamw_kernel's arithmetic, or the compensated one with residual r
template <bool COMP>
__device__ __forceinline__ void adamw_elem(__nv_bfloat16& p, __nv_bfloat16& r, float gi, float& mi, float& vi, float lr,
                                           float b1, float b2, float eps, float wd, float bc1, float bc2_sqrt) {
  if constexpr (COMP)
    adamw_compensated_elem(p, r, __bfloat162float(p), __bfloat162float(r), gi, mi, vi, lr, b1, b2, eps, wd, bc1, bc2_sqrt);
  else
    p = __float2bfloat16_rn(adamw_update(__bfloat162float(p), gi, mi, vi, lr, b1, b2, eps, wd, bc1, bc2_sqrt));
}

union U8x8 {
  uint2 u;
  uint8_t b[8];
};

// One thread owns 8 consecutive elements (16-byte p / r / g, 8-byte codes), a group of 8 lanes one 64-element block: the
// block's new absmax of m and v is reduced with 3 shuffles in the group before requantizing.  Warp 0 of CTA 0 then takes
// the partial last block (n % 64 elements), two elements per lane.
template <bool COMP>
__global__ void __launch_bounds__(256) adamw_8bit_kernel(__nv_bfloat16* __restrict__ p, __nv_bfloat16* __restrict__ r,
                                                         __nv_bfloat16* __restrict__ g, uint8_t* __restrict__ mc,
                                                         float* __restrict__ ma, uint8_t* __restrict__ vc,
                                                         float* __restrict__ va, const float* __restrict__ maps, int64_t n,
                                                         float lr, float b1, float b2, float eps, float wd, float bc1,
                                                         float bc2_sqrt, const float* __restrict__ state,
                                                         int write_clipped_grad) {
  __shared__ QMaps q;
  load_qmaps(q, maps);
  const float coef = state ? state[1] : 1.f;
  const int lane = threadIdx.x & 31;
  const int64_t n8 = n / QBLK * (QBLK / 8), stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i - lane < n8; i += stride) {   // warp-uniform trips
    const bool act = i < n8;                   // n8 is a multiple of 8, so a group of 8 lanes is active or idle as one
    Bf16x8 P, R, G;
    U8x8 MC, VC;
    float mab = 0.f, vab = 0.f;
    P.u = R.u = G.u = make_uint4(0, 0, 0, 0);
    MC.u = VC.u = make_uint2(0, 0);
    if (act) {
      P.u = reinterpret_cast<const uint4*>(p)[i];
      if constexpr (COMP) R.u = reinterpret_cast<const uint4*>(r)[i];
      G.u = reinterpret_cast<const uint4*>(g)[i];
      MC.u = reinterpret_cast<const uint2*>(mc)[i];
      VC.u = reinterpret_cast<const uint2*>(vc)[i];
      mab = ma[i >> 3];
      vab = va[i >> 3];
    }
    float mf[8], vf[8], am = 0.f, av = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      mf[j] = q.map[MC.b[j]] * mab;
      vf[j] = q.map[256 + VC.b[j]] * vab;
      const float gi = __bfloat162float(G.h[j]) * coef;
      adamw_elem<COMP>(P.h[j], R.h[j], gi, mf[j], vf[j], lr, b1, b2, eps, wd, bc1, bc2_sqrt);
      G.h[j] = __float2bfloat16_rn(gi);
      am = fmaxf(am, fabsf(mf[j]));
      av = fmaxf(av, vf[j]);
    }
#pragma unroll
    for (int o = 1; o < 8; o <<= 1) {
      am = fmaxf(am, __shfl_xor_sync(0xffffffffu, am, o));
      av = fmaxf(av, __shfl_xor_sync(0xffffffffu, av, o));
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      MC.b[j] = quantize_m(q, mf[j], am);
      VC.b[j] = quantize_v(q, vf[j], av);
    }
    if (act) {
      reinterpret_cast<uint4*>(p)[i] = P.u;
      if constexpr (COMP) reinterpret_cast<uint4*>(r)[i] = R.u;
      reinterpret_cast<uint2*>(mc)[i] = MC.u;
      reinterpret_cast<uint2*>(vc)[i] = VC.u;
      if (write_clipped_grad) reinterpret_cast<uint4*>(g)[i] = G.u;
      if ((lane & 7) == 0) {
        ma[i >> 3] = am;
        va[i >> 3] = av;
      }
    }
  }
  const int64_t t0 = n / QBLK * QBLK;
  if (t0 < n && blockIdx.x == 0 && threadIdx.x < 32) {
    const float mab = ma[t0 / QBLK], vab = va[t0 / QBLK];
    float mf[2], vf[2], am = 0.f, av = 0.f;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int64_t e = t0 + lane + 32 * j;
      mf[j] = vf[j] = 0.f;
      if (e < n) {
        mf[j] = q.map[mc[e]] * mab;
        vf[j] = q.map[256 + vc[e]] * vab;
        __nv_bfloat16 pe = p[e], re = COMP ? r[e] : __float2bfloat16_rn(0.f);
        const float gi = __bfloat162float(g[e]) * coef;
        adamw_elem<COMP>(pe, re, gi, mf[j], vf[j], lr, b1, b2, eps, wd, bc1, bc2_sqrt);
        p[e] = pe;
        if constexpr (COMP) r[e] = re;
        if (write_clipped_grad) g[e] = __float2bfloat16_rn(gi);
        am = fmaxf(am, fabsf(mf[j]));
        av = fmaxf(av, vf[j]);
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      am = fmaxf(am, __shfl_xor_sync(0xffffffffu, am, o));
      av = fmaxf(av, __shfl_xor_sync(0xffffffffu, av, o));
    }
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int64_t e = t0 + lane + 32 * j;
      if (e < n) {
        mc[e] = quantize_m(q, mf[j], am);
        vc[e] = quantize_v(q, vf[j], av);
      }
    }
    if (lane == 0) {
      ma[t0 / QBLK] = am;
      va[t0 / QBLK] = av;
    }
  }
}

// One moment (bf16 or fp32, n elements) to codes [n] + absmax [ceil(n / 64)]: one warp per block, two elements per lane.
template <typename T>
__global__ void __launch_bounds__(256) moments_quantize_kernel(const T* __restrict__ src, uint8_t* __restrict__ code,
                                                               float* __restrict__ absmax, const float* __restrict__ maps,
                                                               int64_t n, int is_signed) {
  __shared__ QMaps q;
  load_qmaps(q, maps);
  const int lane = threadIdx.x & 31;
  const int64_t nblk = (n + QBLK - 1) / QBLK, wstride = (int64_t)gridDim.x * blockDim.x / 32;
  for (int64_t b = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) / 32; b < nblk; b += wstride) {
    const int64_t e0 = b * QBLK + lane, e1 = e0 + 32;
    const float x0 = e0 < n ? ldf(src + e0) : 0.f, x1 = e1 < n ? ldf(src + e1) : 0.f;
    float am = fmaxf(fabsf(x0), fabsf(x1));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) am = fmaxf(am, __shfl_xor_sync(0xffffffffu, am, o));
    if (e0 < n) code[e0] = is_signed ? quantize_m(q, x0, am) : quantize_v(q, x0, am);
    if (e1 < n) code[e1] = is_signed ? quantize_m(q, x1, am) : quantize_v(q, x1, am);
    if (lane == 0) absmax[b] = am;
  }
}

template <typename T>
__global__ void __launch_bounds__(256) moments_dequantize_kernel(const uint8_t* __restrict__ code,
                                                                 const float* __restrict__ absmax, T* __restrict__ dst,
                                                                 const float* __restrict__ maps, int64_t n, int is_signed) {
  const float* map = maps + (is_signed ? 0 : 256);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    stf(dst + i, __ldg(map + code[i]) * absmax[i / QBLK]);
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

// Block-wise 8-bit moments; all arrays as in adamw_8bit_kernel, r null for the plain update.
int nv_adamw_flat_8bit(void* p, void* r, void* g, void* m_code, float* m_absmax, void* v_code, float* v_absmax,
                       const float* maps, int64_t n, float lr, float beta1, float beta2, float eps, float weight_decay, int step,
                       const float* clip_state, int write_clipped_grad, void* stream) {
  NV_REQUIRE(step >= 1, "nv_adamw_flat_8bit: step must be >= 1");
  NV_REQUIRE(n >= 0, "nv_adamw_flat_8bit: n must be >= 0");
  NV_REQUIRE(((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(r) | reinterpret_cast<uintptr_t>(g)) & 15) == 0,
             "nv_adamw_flat_8bit: p, r and g must be 16-byte aligned");
  NV_REQUIRE(((reinterpret_cast<uintptr_t>(m_code) | reinterpret_cast<uintptr_t>(v_code)) & 7) == 0,
             "nv_adamw_flat_8bit: the code arrays must be 8-byte aligned");
  const float bc1 = 1.f - powf(beta1, (float)step);
  const float bc2s = sqrtf(1.f - powf(beta2, (float)step));
  const int blocks = sm_count() * 8;
  using B = __nv_bfloat16;
  auto kern = r ? adamw_8bit_kernel<true> : adamw_8bit_kernel<false>;
  kern<<<blocks, 256, 0, S_(stream)>>>(reinterpret_cast<B*>(p), reinterpret_cast<B*>(r), reinterpret_cast<B*>(g),
                                       reinterpret_cast<uint8_t*>(m_code), m_absmax, reinterpret_cast<uint8_t*>(v_code), v_absmax,
                                       maps, n, lr, beta1, beta2, eps, weight_decay, bc1, bc2s, clip_state, write_clipped_grad);
  NV_LAUNCH_CHECK();
  return NV_OK;
}

int nv_moments_quantize_8bit(const void* src, int is_bf16, void* code, float* absmax, int64_t n, int is_signed,
                             const float* maps, void* stream) {
  NV_REQUIRE(n >= 0, "nv_moments_quantize_8bit: n must be >= 0");
  if (n == 0) return NV_OK;
  const int64_t warps = (n + QBLK - 1) / QBLK;
  const int blocks = (int)std::min<int64_t>((warps + 7) / 8, (int64_t)sm_count() * 8);
  if (is_bf16)
    moments_quantize_kernel<__nv_bfloat16><<<blocks, 256, 0, S_(stream)>>>(
        reinterpret_cast<const __nv_bfloat16*>(src), reinterpret_cast<uint8_t*>(code), absmax, maps, n, is_signed);
  else
    moments_quantize_kernel<float><<<blocks, 256, 0, S_(stream)>>>(reinterpret_cast<const float*>(src),
                                                                   reinterpret_cast<uint8_t*>(code), absmax, maps, n, is_signed);
  NV_LAUNCH_CHECK();
  return NV_OK;
}

int nv_moments_dequantize_8bit(const void* code, const float* absmax, void* dst, int is_bf16, int64_t n, int is_signed,
                               const float* maps, void* stream) {
  NV_REQUIRE(n >= 0, "nv_moments_dequantize_8bit: n must be >= 0");
  if (n == 0) return NV_OK;
  const int blocks = (int)std::min<int64_t>((n + 255) / 256, (int64_t)sm_count() * 8);
  if (is_bf16)
    moments_dequantize_kernel<__nv_bfloat16><<<blocks, 256, 0, S_(stream)>>>(
        reinterpret_cast<const uint8_t*>(code), absmax, reinterpret_cast<__nv_bfloat16*>(dst), maps, n, is_signed);
  else
    moments_dequantize_kernel<float><<<blocks, 256, 0, S_(stream)>>>(reinterpret_cast<const uint8_t*>(code), absmax,
                                                                     reinterpret_cast<float*>(dst), maps, n, is_signed);
  NV_LAUNCH_CHECK();
  return NV_OK;
}

}  // extern "C"
