// navillm_b200 — decode-phase kernels for greedy / sampled generation (HBM-bound regime).
//
// Replaces what the reference reaches through HF GenerationMixin.generate after the prefill
// (models/nav_model.py:324-338,388-399; models/modified_lm.py:184-199): a tuple-of-tensors KV cache grown by
// torch.cat every token and eager attention over it.  Here the cache is pre-allocated and contiguous
// ([B, Smax, H*128] per layer for K and for V, bf16, real tokens only), one new token per sequence attends
// over it with 128-bit coalesced loads, and the step has static shapes so the host can replay it as a CUDA
// graph (sequence lengths live in device memory).
//
// Opt-in fp8 cache (nv_kv_store_prefill_fp8, nv_decode_attn_rope_fp8, nv_kv_store_suffix_fp8): the same layout in e4m3 bytes
// plus one int8 exponent per (sequence, position, head) row of 128 elements, quantized with the weight format of nv_fp8.cuh as
// rows are stored.
#include <type_traits>

#include "nv_common.cuh"
#include "nv_fp8.cuh"
#include "nv_host.h"

namespace nv {

__device__ __forceinline__ void unpack8d(const uint4& u, float (&f)[8]) {
  f[0] = bf16_lo(u.x); f[1] = bf16_hi(u.x); f[2] = bf16_lo(u.y); f[3] = bf16_hi(u.y);
  f[4] = bf16_lo(u.z); f[5] = bf16_hi(u.z); f[6] = bf16_lo(u.w); f[7] = bf16_hi(u.w);
}

// eight e4m3 bytes of a cache row with exponent e -> the fp32 values unpack8d gives for the same row rounded to bf16 (K', V')
__device__ __forceinline__ void unpack8q(const uint2& u, int e, float (&f)[8]) {
  const float s = fp8_pow2(e);
  fp8x4_to_f32x4(u.x, s, f);
  fp8x4_to_f32x4(u.y, s, f + 4);
}

// fp8 twin of kv_store_prefill_kernel: a half-warp owns one (token, head) row of K and of V; 16 lanes x 8 elements.
// Same packing (offs: rows already cached per sequence, or null) and the same drop of rows at p >= Smax.  Each row's amax,
// exponent and bytes follow quantize_fp8_rows_kernel.
__global__ void __launch_bounds__(256) kv_store_prefill_fp8_kernel(const __nv_bfloat16* __restrict__ qkv, int64_t ld,
                                                                   const int* __restrict__ cu, const int* __restrict__ offs,
                                                                   uint8_t* __restrict__ kq,
                                                                   uint8_t* __restrict__ vq, int8_t* __restrict__ ke,
                                                                   int8_t* __restrict__ ve, int B, int Smax, int H) {
  const int HD = H * 128;
  const int hl = threadIdx.x & 15, half = (threadIdx.x >> 4) & 1;
  const int64_t rows = (int64_t)cu[B] * H;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  // the loop bound is uniform over the warp, so both halves reach every shuffle
  for (int64_t r0 = 2 * ((int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)); r0 < rows; r0 += 2 * warps) {
    const int64_t r = r0 + half;
    const bool live = r < rows;
    const int t = live ? (int)(r / H) : 0, h = live ? (int)(r % H) : 0;
    int b = 0;
    while (b + 1 < B && cu[b + 1] <= t) ++b;
    const int p = t - cu[b] + (offs && live ? offs[b] : 0);
    uint4 k = make_uint4(0, 0, 0, 0), v = k;
    if (live) {
      k = *reinterpret_cast<const uint4*>(qkv + (int64_t)t * ld + HD + h * 128 + hl * 8);
      v = *reinterpret_cast<const uint4*>(qkv + (int64_t)t * ld + 2 * HD + h * 128 + hl * 8);
    }
    uint32_t mk = bf16x8_amax_bits(k), mv = bf16x8_amax_bits(v);
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) {                             // reduce inside the half-warp
      mk = max(mk, __shfl_xor_sync(0xffffffffu, mk, o));
      mv = max(mv, __shfl_xor_sync(0xffffffffu, mv, o));
    }
    if (live && p < Smax) {
      const int ek = fp8_row_exponent(__uint_as_float(mk << 16)), ev = fp8_row_exponent(__uint_as_float(mv << 16));
      const int64_t row = (int64_t)b * Smax + p;
      *reinterpret_cast<uint2*>(kq + row * HD + h * 128 + hl * 8) = fp8x8_from_bf16x8(k, fp8_pow2(-ek));
      *reinterpret_cast<uint2*>(vq + row * HD + h * 128 + hl * 8) = fp8x8_from_bf16x8(v, fp8_pow2(-ev));
      if (hl == 0) {
        ke[row * H + h] = (int8_t)ek;
        ve[row * H + h] = (int8_t)ev;
      }
    }
  }
}

// Copy the K and V column blocks of packed prefill rows into the cache: row t of sequence b at local
// position p goes to cache[b, p, :].
__global__ void kv_store_prefill_kernel(const __nv_bfloat16* __restrict__ qkv, int64_t ld, const int* __restrict__ cu,
                                        const int* __restrict__ offs, __nv_bfloat16* __restrict__ kc,
                                        __nv_bfloat16* __restrict__ vc, int B, int Smax, int HD) {
  const int vecs = HD >> 3;
  const int T = cu[B];
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < (int64_t)T * vecs;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int v = idx % vecs, t = idx / vecs;
    int b = 0;
    while (b + 1 < B && cu[b + 1] <= t) ++b;
    const int p = t - cu[b] + (offs ? offs[b] : 0);          // offs: rows already cached for this sequence
    if (p >= Smax) continue;
    const int64_t dst = ((int64_t)b * Smax + p) * HD + v * 8;
    *reinterpret_cast<uint4*>(kc + dst) = *reinterpret_cast<const uint4*>(qkv + (int64_t)t * ld + HD + v * 8);
    *reinterpret_cast<uint4*>(vc + dst) = *reinterpret_cast<const uint4*>(qkv + (int64_t)t * ld + 2 * HD + v * 8);
  }
}

// Append the new token's K,V (row b of qkv [B, 3*HD]) at position lens[b].
__global__ void kv_append_kernel(const __nv_bfloat16* __restrict__ qkv, int64_t ld, const int* __restrict__ lens,
                                 __nv_bfloat16* __restrict__ kc, __nv_bfloat16* __restrict__ vc, int B, int Smax, int HD) {
  const int vecs = HD >> 3;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < B * vecs; idx += gridDim.x * blockDim.x) {
    const int v = idx % vecs, b = idx / vecs;
    const int p = lens[b];
    if (p >= Smax) continue;
    const int64_t dst = ((int64_t)b * Smax + p) * HD + v * 8;
    *reinterpret_cast<uint4*>(kc + dst) = *reinterpret_cast<const uint4*>(qkv + (int64_t)b * ld + HD + v * 8);
    *reinterpret_cast<uint4*>(vc + dst) = *reinterpret_cast<const uint4*>(qkv + (int64_t)b * ld + 2 * HD + v * 8);
  }
}

// Decode step: rotary embedding of the new token's q and k heads (in place, rounding points of rope_kernel) fused with
// the append of its rotated K and its V to the cache at position lens[b] (= the token's rotary position).
// Work items: [0, B*2H*8) rotate one 8-element chunk pair (d, d + 64) of a q or k head; [.., + B*HD/8) copy one V chunk.
__global__ void decode_rope_kv_kernel(__nv_bfloat16* __restrict__ qkv, int64_t ld, const int* __restrict__ lens,
                                      const __nv_bfloat16* __restrict__ cos_t, const __nv_bfloat16* __restrict__ sin_t,
                                      __nv_bfloat16* __restrict__ kc, __nv_bfloat16* __restrict__ vc, int B, int Smax, int H) {
  griddep_launch();
  griddep_wait();
  const int HD = H * 128;
  const int n_rot = B * 2 * H * 8, n_v = B * (HD >> 3);
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < n_rot + n_v; idx += gridDim.x * blockDim.x) {
    if (idx < n_rot) {
      const int c = idx & 7, h = (idx >> 3) % (2 * H), b = idx / (16 * H);
      const int p = lens[b];
      __nv_bfloat16* base = qkv + (int64_t)b * ld + h * 128;
      float x1[8], x2[8], c1[8], s1[8], c2[8], s2[8];
      unpack8d(*reinterpret_cast<const uint4*>(base + c * 8), x1);
      unpack8d(*reinterpret_cast<const uint4*>(base + 64 + c * 8), x2);
      unpack8d(*reinterpret_cast<const uint4*>(cos_t + (int64_t)p * 128 + c * 8), c1);
      unpack8d(*reinterpret_cast<const uint4*>(sin_t + (int64_t)p * 128 + c * 8), s1);
      unpack8d(*reinterpret_cast<const uint4*>(cos_t + (int64_t)p * 128 + 64 + c * 8), c2);
      unpack8d(*reinterpret_cast<const uint4*>(sin_t + (int64_t)p * 128 + 64 + c * 8), s2);
      uint4 o1, o2;
      uint32_t* q1 = &o1.x; uint32_t* q2 = &o2.x;
#pragma unroll
      for (int j = 0; j < 8; j += 2) {
        const float a0 = bf16_round(x1[j] * c1[j]) + bf16_round(-x2[j] * s1[j]);
        const float a1 = bf16_round(x1[j + 1] * c1[j + 1]) + bf16_round(-x2[j + 1] * s1[j + 1]);
        const float b0 = bf16_round(x2[j] * c2[j]) + bf16_round(x1[j] * s2[j]);
        const float b1 = bf16_round(x2[j + 1] * c2[j + 1]) + bf16_round(x1[j + 1] * s2[j + 1]);
        q1[j >> 1] = pack_bf16x2(a0, a1);
        q2[j >> 1] = pack_bf16x2(b0, b1);
      }
      *reinterpret_cast<uint4*>(base + c * 8) = o1;
      *reinterpret_cast<uint4*>(base + 64 + c * 8) = o2;
      if (h >= H && p < Smax) {                               // a k head: rotated K goes to the cache
        __nv_bfloat16* dst = kc + ((int64_t)b * Smax + p) * HD + (h - H) * 128;
        *reinterpret_cast<uint4*>(dst + c * 8) = o1;
        *reinterpret_cast<uint4*>(dst + 64 + c * 8) = o2;
      }
    } else {
      const int j = idx - n_rot;
      const int v = j % (HD >> 3), b = j / (HD >> 3);
      const int p = lens[b];
      if (p < Smax)
        *reinterpret_cast<uint4*>(vc + ((int64_t)b * Smax + p) * HD + v * 8) =
            *reinterpret_cast<const uint4*>(qkv + (int64_t)b * ld + 2 * HD + v * 8);
    }
  }
}

// One new query per sequence over its cache (keys 0..lens[b], the new token included: call after append).
// CTA = (b, h), DA_WARPS warps; half-warps stream keys with 16-byte loads; per-warp online softmax, merged in smem.
// (8 warps: 256 (b, h) CTAs of 4 warps kept too few loads in flight for a 50 MB cache read; all CTAs are co-resident.)
constexpr int DA_WARPS = 8;
// ROPE = true fuses decode_rope_kv_kernel: q points at the PRE-RoPE fused qkv row block [B, 3*H*128]; warp 0 rotates this
// head's q and k at position lens[b] (same rounding points as rope_kernel), appends the rotated k and the v to the caches
// and hands the rotated q to the CTA through shared memory - one launch less per decoder layer and token.
// FP8 = true reads an fp8 cache (kc / vc e4m3 bytes, ke / ve the row exponents [B, Smax, H]; with ROPE the new k and v rows are
// quantized as they are appended).  Keys are expanded to the fp32 values of the bf16-rounded rows K' / V', and the key
// assignment and every reduction order are those of the bf16 kernel, so the output is bit for bit the bf16 kernel's on K' / V'.
template <bool FP8>
using kv_elem_t = typename std::conditional<FP8, uint8_t, __nv_bfloat16>::type;

template <bool ROPE, bool FP8 = false>
__global__ void __launch_bounds__(DA_WARPS * 32) decode_attn_kernel(const __nv_bfloat16* __restrict__ q, int64_t ldq,
                                                          kv_elem_t<FP8>* __restrict__ kc, kv_elem_t<FP8>* __restrict__ vc,
                                                          const int* __restrict__ lens, __nv_bfloat16* __restrict__ out,
                                                          int64_t ldo, int Smax, int H, float scale,
                                                          const __nv_bfloat16* __restrict__ cos_t,
                                                          const __nv_bfloat16* __restrict__ sin_t,
                                                          int8_t* __restrict__ ke, int8_t* __restrict__ ve) {
  __shared__ float s_m[DA_WARPS], s_l[DA_WARPS];
  __shared__ float s_acc[DA_WARPS][128];
  __shared__ uint4 s_q[16];                            // rotated q of this head (bf16 x 128)
  griddep_launch();
  griddep_wait();
  const int b = blockIdx.x / H, h = blockIdx.x % H;
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int half = lane >> 4, hl = lane & 15;          // half-warp id, lane within the half (8 dims each)
  const int n = lens[b] + 1;                            // keys visible to the new token
  const int HD = H * 128;
  if (ROPE) {
    const int p = n - 1;
    if (w == 0) {
      uint4 r0 = make_uint4(0, 0, 0, 0), r1 = r0;       // FP8: this lane's chunks of the new k row (lanes 8..15) or v row (16..31)
      if (lane < 16) {                                  // lanes 0..7: q chunk c, lanes 8..15: k chunk c
        const int c = lane & 7, is_k = lane >> 3;
        const __nv_bfloat16* base = q + (int64_t)b * ldq + (is_k ? HD : 0) + h * 128;
        float x1[8], x2[8], c1[8], s1[8], c2[8], s2[8];
        unpack8d(*reinterpret_cast<const uint4*>(base + c * 8), x1);
        unpack8d(*reinterpret_cast<const uint4*>(base + 64 + c * 8), x2);
        unpack8d(*reinterpret_cast<const uint4*>(cos_t + (int64_t)p * 128 + c * 8), c1);
        unpack8d(*reinterpret_cast<const uint4*>(sin_t + (int64_t)p * 128 + c * 8), s1);
        unpack8d(*reinterpret_cast<const uint4*>(cos_t + (int64_t)p * 128 + 64 + c * 8), c2);
        unpack8d(*reinterpret_cast<const uint4*>(sin_t + (int64_t)p * 128 + 64 + c * 8), s2);
        uint4 o1, o2;
        uint32_t* q1 = &o1.x; uint32_t* q2 = &o2.x;
#pragma unroll
        for (int j = 0; j < 8; j += 2) {
          const float a0 = bf16_round(x1[j] * c1[j]) + bf16_round(-x2[j] * s1[j]);
          const float a1 = bf16_round(x1[j + 1] * c1[j + 1]) + bf16_round(-x2[j + 1] * s1[j + 1]);
          const float b0 = bf16_round(x2[j] * c2[j]) + bf16_round(x1[j] * s2[j]);
          const float b1 = bf16_round(x2[j + 1] * c2[j + 1]) + bf16_round(x1[j + 1] * s2[j + 1]);
          q1[j >> 1] = pack_bf16x2(a0, a1);
          q2[j >> 1] = pack_bf16x2(b0, b1);
        }
        if (!is_k) {
          s_q[c] = o1; s_q[8 + c] = o2;
        } else if constexpr (FP8) {
          r0 = o1; r1 = o2;
        } else if (p < Smax) {
          __nv_bfloat16* dst = kc + ((int64_t)b * Smax + p) * HD + h * 128;
          *reinterpret_cast<uint4*>(dst + c * 8) = o1;
          *reinterpret_cast<uint4*>(dst + 64 + c * 8) = o2;
        }
      } else if constexpr (FP8) {
        r0 = *reinterpret_cast<const uint4*>(q + (int64_t)b * ldq + 2 * HD + h * 128 + (lane - 16) * 8);
      } else if (p < Smax) {                            // lanes 16..31: this head's v (16 x 16 bytes)
        const int v = lane - 16;
        *reinterpret_cast<uint4*>(vc + ((int64_t)b * Smax + p) * HD + h * 128 + v * 8) =
            *reinterpret_cast<const uint4*>(q + (int64_t)b * ldq + 2 * HD + h * 128 + v * 8);
      }
      if constexpr (FP8) {
        // row amax: the k row over lanes 8..15 (xor 1, 2, 4), the v row over lanes 16..31 (and xor 8); lanes 0..7 reduce
        // a value nobody uses
        uint32_t m = max(bf16x8_amax_bits(r0), bf16x8_amax_bits(r1));
#pragma unroll
        for (int o = 1; o < 8; o <<= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
        const uint32_t m8 = __shfl_xor_sync(0xffffffffu, m, 8);
        if (lane >= 16) m = max(m, m8);
        const int e = fp8_row_exponent(__uint_as_float(m << 16));
        const float inv = fp8_pow2(-e);
        if (lane >= 8 && p < Smax) {
          const int64_t row = (int64_t)b * Smax + p;
          if (lane < 16) {
            uint8_t* dst = kc + row * HD + h * 128 + (lane & 7) * 8;
            *reinterpret_cast<uint2*>(dst) = fp8x8_from_bf16x8(r0, inv);
            *reinterpret_cast<uint2*>(dst + 64) = fp8x8_from_bf16x8(r1, inv);
            if (lane == 8) ke[row * H + h] = (int8_t)e;
          } else {
            *reinterpret_cast<uint2*>(vc + row * HD + h * 128 + (lane - 16) * 8) = fp8x8_from_bf16x8(r0, inv);
            if (lane == 16) ve[row * H + h] = (int8_t)e;
          }
        }
      }
    }
    __syncthreads();                                    // rotated q in smem, new k / v rows visible to the whole CTA
  }
  float qf[8];
  unpack8d(ROPE ? s_q[hl] : *reinterpret_cast<const uint4*>(q + (int64_t)b * ldq + h * 128 + hl * 8), qf);
  const float sl2 = scale * 1.4426950408889634f;
  float m = -INFINITY, l = 0.f, acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  // A warp takes 8 consecutive keys per iteration (4 per half-warp): eight 16-byte loads per lane are in flight
  // before the first use, which is what a latency-bound streaming loop needs (one key per half-warp and
  // iteration kept ~1 MB in flight chip-wide and ran at 35 us for 52 MB of cache).
  constexpr int KPI = 4;
  // one key's 8 elements of this lane: 16 bytes of bf16, or 8 e4m3 bytes and (ke / ve) the row's exponent
  using raw_t = typename std::conditional<FP8, uint2, uint4>::type;
  auto load_keys = [&](int jb, raw_t (&kr)[KPI], raw_t (&vr)[KPI], int (&kx)[KPI], int (&vx)[KPI]) {
#pragma unroll
    for (int u = 0; u < KPI; ++u) {
      if (jb + u < n) {
        const int64_t off = ((int64_t)b * Smax + jb + u) * HD + h * 128 + hl * 8;
        kr[u] = *reinterpret_cast<const raw_t*>(kc + off);
        vr[u] = *reinterpret_cast<const raw_t*>(vc + off);
        if constexpr (FP8) {
          const int64_t row = ((int64_t)b * Smax + jb + u) * H + h;
          kx[u] = ke[row];
          vx[u] = ve[row];
        }
      } else {
        if constexpr (FP8) {
          kr[u] = make_uint2(0, 0);
          vr[u] = make_uint2(0, 0);
          kx[u] = vx[u] = 0;
        } else {
          kr[u] = make_uint4(0, 0, 0, 0);
          vr[u] = make_uint4(0, 0, 0, 0);
        }
      }
    }
  };
  auto unpack = [&](const raw_t& r, int x, float (&f)[8]) {
    if constexpr (FP8) unpack8q(r, x, f);
    else unpack8d(r, f);
  };
  // software pipeline: the loads of the NEXT 8 keys are in flight while the current ones are reduced (the loop is a chain
  // of DRAM-latency-long iterations otherwise)
  raw_t knext[KPI], vnext[KPI];
  int kxnext[KPI], vxnext[KPI];
  load_keys(w * 2 * KPI + half * KPI, knext, vnext, kxnext, vxnext);
  for (int j0 = w * 2 * KPI; j0 < n; j0 += DA_WARPS * 2 * KPI) {
    const int jb = j0 + half * KPI;
    raw_t kraw[KPI], vraw[KPI];
    int kx[KPI], vx[KPI];
#pragma unroll
    for (int u = 0; u < KPI; ++u) { kraw[u] = knext[u]; vraw[u] = vnext[u]; kx[u] = kxnext[u]; vx[u] = vxnext[u]; }
    if (j0 + DA_WARPS * 2 * KPI < n) load_keys(jb + DA_WARPS * 2 * KPI, knext, vnext, kxnext, vxnext);
    float sc[KPI];
#pragma unroll
    for (int u = 0; u < KPI; ++u) {
      float kf[8];
      unpack(kraw[u], kx[u], kf);
      float s = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) s += qf[i] * kf[i];
      sc[u] = s;
    }
#pragma unroll
    for (int o = 8; o > 0; o >>= 1)
#pragma unroll
      for (int u = 0; u < KPI; ++u) sc[u] += __shfl_xor_sync(0xffffffffu, sc[u], o);   // reduce inside the half-warp
    float mn = m;
#pragma unroll
    for (int u = 0; u < KPI; ++u)
      if (jb + u < n) mn = fmaxf(mn, sc[u]);
    if (mn != -INFINITY) {
      const float a = exp2f((m - mn) * sl2);
      l *= a;
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] *= a;
#pragma unroll
      for (int u = 0; u < KPI; ++u) {
        if (jb + u < n) {
          const float p = exp2f((sc[u] - mn) * sl2);
          float vf[8];
          unpack(vraw[u], vx[u], vf);
          l += p;
#pragma unroll
          for (int i = 0; i < 8; ++i) acc[i] += p * vf[i];
        }
      }
      m = mn;
    }
  }
  // merge the two half-warps
  {
    const float mo = __shfl_xor_sync(0xffffffffu, m, 16), lo = __shfl_xor_sync(0xffffffffu, l, 16);
    const float mn = fmaxf(m, mo);
    const float a = (m == -INFINITY) ? 0.f : exp2f((m - mn) * sl2), ao = (mo == -INFINITY) ? 0.f : exp2f((mo - mn) * sl2);
    l = l * a + lo * ao;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float other = __shfl_xor_sync(0xffffffffu, acc[i], 16);
      acc[i] = acc[i] * a + other * ao;
    }
    m = mn;
  }
  if (lane < 16) {
    if (lane == 0) { s_m[w] = m; s_l[w] = l; }
#pragma unroll
    for (int i = 0; i < 8; ++i) s_acc[w][hl * 8 + i] = acc[i];
  }
  __syncthreads();
  if (threadIdx.x < 128) {
    const int d = threadIdx.x;
    float mm = s_m[0];
#pragma unroll
    for (int k = 1; k < DA_WARPS; ++k) mm = fmaxf(mm, s_m[k]);
    float num = 0.f, den = 0.f;
#pragma unroll
    for (int k = 0; k < DA_WARPS; ++k) {
      const float a = (s_m[k] == -INFINITY) ? 0.f : exp2f((s_m[k] - mm) * sl2);
      num += s_acc[k][d] * a;
      den += s_l[k] * a;
    }
    out[(int64_t)b * ldo + h * 128 + d] = __float2bfloat16_rn(num / den);
  }
}

// Special ids masked by argmax_kernel and sample_topk_kernel: they are staged in shared memory, so the host entry points
// reject longer lists.
constexpr int MAX_SPECIAL = 64;

// next[b] = finished[b] ? pad_id : argmax_c logits[b,c] over non-special columns (first index wins ties, like
// torch.argmax); finished[b] |= next == eos (when stop_on_eos).  One CTA per row.
__global__ void __launch_bounds__(1024) argmax_kernel(const __nv_bfloat16* __restrict__ logits, int64_t ld, int V,
                                                      const int* __restrict__ special, int n_special,
                                                      int* __restrict__ finished, int eos_id, int pad_id, int stop_on_eos,
                                                      int* __restrict__ next) {
  __shared__ float sv[32];
  __shared__ int si[32];
  __shared__ int s_special[MAX_SPECIAL];
  griddep_launch();
  griddep_wait();
  const int b = blockIdx.x;
  const int ns = n_special;
  if (threadIdx.x < ns) s_special[threadIdx.x] = special[threadIdx.x];
  __syncthreads();
  float best = -INFINITY;
  int bi = V;
  const __nv_bfloat16* row = logits + (int64_t)b * ld;
  const bool vec_ok = (ld & 7) == 0;                       // 16-byte aligned rows
  const int nvec = vec_ok ? (V >> 3) : 0;
  for (int v = threadIdx.x; v < nvec; v += blockDim.x) {
    float f[8];
    unpack8d(*reinterpret_cast<const uint4*>(row + v * 8), f);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int c = v * 8 + i;
      bool sp = false;
      for (int s = 0; s < ns; ++s) sp |= (s_special[s] == c);
      if (!sp && f[i] > best) { best = f[i]; bi = c; }     // ascending scan keeps the smallest index per thread on ties
    }
  }
  for (int c = nvec * 8 + threadIdx.x; c < V; c += blockDim.x) {
    bool sp = false;
    for (int s = 0; s < ns; ++s) sp |= (s_special[s] == c);
    const float v = __bfloat162float(row[c]);
    if (!sp && (v > best || (v == best && c < bi))) { best = v; bi = c; }
  }
  // warp then CTA reduction; ties -> smallest index (torch.argmax returns the first maximal element)
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float v2 = __shfl_xor_sync(0xffffffffu, best, o);
    const int i2 = __shfl_xor_sync(0xffffffffu, bi, o);
    if (v2 > best || (v2 == best && i2 < bi)) { best = v2; bi = i2; }
  }
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) { sv[w] = best; si[w] = bi; }
  __syncthreads();
  if (w == 0) {
    const int nw = blockDim.x >> 5;
    best = lane < nw ? sv[lane] : -INFINITY;
    bi = lane < nw ? si[lane] : V;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float v2 = __shfl_xor_sync(0xffffffffu, best, o);
      const int i2 = __shfl_xor_sync(0xffffffffu, bi, o);
      if (v2 > best || (v2 == best && i2 < bi)) { best = v2; bi = i2; }
    }
    if (lane == 0) {
      int tok = bi;
      if (finished[b]) tok = pad_id;
      else if (stop_on_eos && tok == eos_id) finished[b] = 1;
      next[b] = tok;
    }
  }
}

// ---- trie-constrained decoding (TrieLogitsProcessor, models/modified_lm.py:10-30; caller tasks/agents/mp3d_agent.py:545-584)
// The trie is in CSR form: the children of node n are edges node_ptr[n] .. node_ptr[n+1], with child_tok ascending and
// child_node the node each edge leads to; node 0 is the root and node n_nodes an extra childless "dead" node.  One CTA per
// row: (1) advance state[b] by last[b] with the semantics of tools/trie.py (a node without children stays; otherwise move to
// the child, and a token that is not a child sets *miss and moves to the dead node); (2) out[b, :] = -inf except the allowed
// tokens (the node's children, or leaf_tok when it has none), which carry their logit; (3) a row whose allowed non-special
// values are all -inf, or with an allowed NaN, sets *miss and gets 0.0 at its first allowed non-special token (else at its
// first non-special column), so the argmax / draw that follows stays inside [0, V).
constexpr int TM_THREADS = 512;

__device__ __forceinline__ bool tm_is_special(const int* s_special, int ns, int c) {
  bool sp = false;
  for (int s = 0; s < ns; ++s) sp |= (s_special[s] == c);
  return sp;
}

__global__ void __launch_bounds__(TM_THREADS) trie_mask_kernel(const __nv_bfloat16* __restrict__ logits, int64_t ld,
                                                               __nv_bfloat16* __restrict__ out, int64_t ldo, int V,
                                                               const int* __restrict__ node_ptr, const int* __restrict__ child_tok,
                                                               const int* __restrict__ child_node, int n_nodes, int leaf_tok,
                                                               const int* __restrict__ special, int n_special,
                                                               int* __restrict__ state, const int* __restrict__ last,
                                                               int* __restrict__ miss) {
  __shared__ int s_special[MAX_SPECIAL];
  __shared__ int s_node;
  griddep_launch();
  griddep_wait();
  const int b = blockIdx.x, tid = threadIdx.x;
  const int ns = n_special;
  if (tid < ns) s_special[tid] = special[tid];
  if (tid == 0) {
    int node = state[b];
    const int e0 = node_ptr[node], e1 = node_ptr[node + 1];
    if (last != nullptr && e1 > e0) {
      const int tok = last[b];
      int lo = e0, hi = e1;                                   // first edge with child_tok >= tok
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (child_tok[mid] < tok) lo = mid + 1;
        else hi = mid;
      }
      if (lo < e1 && child_tok[lo] == tok) {
        node = child_node[lo];
      } else {
        node = n_nodes;
        *miss = 1;
      }
      state[b] = node;
    }
    s_node = node;
  }
  __nv_bfloat16* orow = out + (int64_t)b * ldo;
  const uint4 ninf = make_uint4(0xFF80FF80u, 0xFF80FF80u, 0xFF80FF80u, 0xFF80FF80u);   // bf16 -inf x 8
  const int nvec = V >> 3;
  for (int v = tid; v < nvec; v += TM_THREADS) reinterpret_cast<uint4*>(orow)[v] = ninf;
  for (int c = nvec * 8 + tid; c < V; c += TM_THREADS) orow[c] = __ushort_as_bfloat16((unsigned short)0xFF80u);
  __syncthreads();
  const int node = s_node;
  const int e0 = node_ptr[node], e1 = node_ptr[node + 1];
  const bool leaf = e1 == e0;
  const int n_allowed = leaf ? 1 : e1 - e0;
  const __nv_bfloat16* lrow = logits + (int64_t)b * ld;
  int live = 0, nan = 0;
  for (int i = tid; i < n_allowed; i += TM_THREADS) {       // fan-outs of any size: looped, not capped
    const int c = leaf ? leaf_tok : child_tok[e0 + i];
    const __nv_bfloat16 x = lrow[c];
    orow[c] = x;
    const float f = __bfloat162float(x);
    nan |= (f != f);
    live |= (f > -INFINITY && !tm_is_special(s_special, ns, c));
  }
  const int any_nan = __syncthreads_or(nan), any_live = __syncthreads_or(live);
  if (tid == 0 && (any_nan || !any_live)) {
    *miss = 1;
    int c = -1;
    for (int i = 0; i < n_allowed && c < 0; ++i) {           // children are distinct: at most ns + 1 iterations
      const int t = leaf ? leaf_tok : child_tok[e0 + i];
      if (!tm_is_special(s_special, ns, t)) c = t;
    }
    if (c < 0)
      for (c = 0; c < V && tm_is_special(s_special, ns, c); ++c) {
      }
    if (c < V) orow[c] = __float2bfloat16_rn(0.f);
  }
}

__global__ void add_int_kernel(int* __restrict__ x, int n, int delta) {
  griddep_launch();
  griddep_wait();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) x[i] += delta;
}

// ---- sampled decoding (HF GenerationMixin.sample as the reference reaches it with do_sample=True, tasks/agents/llava.py:58-62
// -> models/nav_model.py:388-396): next-token scores -> TemperatureLogitsWarper (scores / T, in the logits' dtype: bf16) ->
// TopKLogitsWarper (transformers' generation default top_k = 50: every score strictly below the k-th largest becomes -inf,
// ties at the k-th value stay) -> softmax (fp32 inside, rounded to bf16) -> one multinomial draw.  One CTA per row: the
// row's scores live in shared memory, the k-th largest is found exactly with two 8-bit radix passes over the 16 significant
// bits of a bf16 value, and the draw is the inverse CDF (token order) of the bf16 probabilities at the uniform number u[b]
// the host supplies (torch.rand: the torch CUDA generator stays the seed authority, like torch.multinomial in the reference).
// finished / eos / pad handling as argmax_kernel.  probs_out (optional, fp32 [B, V]) receives the sampling distribution.
constexpr int SMP_THREADS = 1024;

__device__ __forceinline__ uint32_t smp_key16(float v) {          // monotone: larger float -> larger key; -inf lowest
  uint32_t u = __float_as_uint(v);
  u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  return u >> 16;
}

// threads cooperatively find, scanning bins from the top, the bin that holds the `want`-th largest element (1-based);
// returns that bin and how many elements sit in higher bins.  hist: 256 counters in shared memory.
__device__ __forceinline__ void smp_pick_bin(const int* hist, int want, int& bin, int& above) {
  __shared__ int s_bin, s_above;
  if (threadIdx.x == 0) {
    int acc = 0, b = 255;
    for (; b > 0; --b) {
      if (acc + hist[b] >= want) break;
      acc += hist[b];
    }
    s_bin = b;
    s_above = acc;
  }
  __syncthreads();
  bin = s_bin;
  above = s_above;
  __syncthreads();
}

__global__ void __launch_bounds__(SMP_THREADS) sample_topk_kernel(const __nv_bfloat16* __restrict__ logits, int64_t ld, int V,
                                                                  const int* __restrict__ special, int n_special,
                                                                  int* __restrict__ finished, int eos_id, int pad_id, int stop_on_eos,
                                                                  float temperature, int top_k, const float* __restrict__ u,
                                                                  int* __restrict__ next, float* __restrict__ probs_out) {
  extern __shared__ float sc[];                              // [V] scores, then probabilities
  __shared__ int hist[256];
  __shared__ float red[32];
  __shared__ int s_special[MAX_SPECIAL];
  __shared__ int s_idx, s_last;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int ns = n_special;
  if (tid < ns) s_special[tid] = special[tid];
  if (tid < 256) hist[tid] = 0;
  if (tid == 0) { s_idx = V; s_last = -1; }
  __syncthreads();
  const __nv_bfloat16* row = logits + (int64_t)b * ld;
  // 1. scores = bf16(logit / T), special tokens -inf (models/modified_lm.py:122-124); histogram of the high key byte
  float mx = -INFINITY;
  for (int c = tid; c < V; c += SMP_THREADS) {
    bool sp = false;
    for (int s = 0; s < ns; ++s) sp |= (s_special[s] == c);
    float v = sp ? -INFINITY : bf16_round(__bfloat162float(row[c]) / temperature);
    if (v != v) v = -INFINITY;                               // NaN scores cannot be drawn
    sc[c] = v;
    mx = fmaxf(mx, v);
    atomicAdd(&hist[smp_key16(v) >> 8], 1);
  }
  __syncthreads();
  // 2. the k-th largest score, exactly
  const int k = max(1, min(top_k > 0 ? top_k : V, V));
  int hi_bin, above;
  smp_pick_bin(hist, k, hi_bin, above);
  if (tid < 256) hist[tid] = 0;
  __syncthreads();
  for (int c = tid; c < V; c += SMP_THREADS) {
    const uint32_t key = smp_key16(sc[c]);
    if ((int)(key >> 8) == hi_bin) atomicAdd(&hist[key & 255u], 1);
  }
  __syncthreads();
  int lo_bin, above2;
  smp_pick_bin(hist, k - above, lo_bin, above2);
  const uint32_t thr_key = ((uint32_t)hi_bin << 8) | (uint32_t)lo_bin;      // keep score >= k-th largest (ties stay)
  // 3. softmax over the kept scores (fp32), rounded to bf16 like the reference's bf16 softmax output
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if (lane == 0) red[w] = mx;
  __syncthreads();
  mx = red[lane];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  __syncthreads();
  float part = 0.f;
  for (int c = tid; c < V; c += SMP_THREADS) {
    const float v = sc[c];
    const float e = (smp_key16(v) >= thr_key && v > -INFINITY) ? expf(v - mx) : 0.f;
    sc[c] = e;
    part += e;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
  if (lane == 0) red[w] = part;
  __syncthreads();
  float denom = red[lane];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) denom += __shfl_xor_sync(0xffffffffu, denom, o);
  __syncthreads();
  // 4. probabilities + inverse CDF in token order: thread t owns the contiguous chunk [t*CH, (t+1)*CH)
  const int CH = (V + SMP_THREADS - 1) / SMP_THREADS;
  const int c0 = min(tid * CH, V), c1 = min(c0 + CH, V);
  float local = 0.f;
  int last_kept = -1;
  for (int c = c0; c < c1; ++c) {
    const float p = bf16_round(sc[c] / denom);
    sc[c] = p;
    local += p;
    if (p > 0.f) last_kept = c;
    if (probs_out) probs_out[(int64_t)b * V + c] = p;
  }
  if (last_kept >= 0) atomicMax(&s_last, last_kept);
  float incl = local;                                        // inclusive scan of the chunk sums over the CTA
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  if (lane == 31) red[w] = incl;
  __syncthreads();
  float wsum = red[lane];
  float wincl = wsum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float t = __shfl_up_sync(0xffffffffu, wincl, o);
    if (lane >= o) wincl += t;
  }
  const float total = __shfl_sync(0xffffffffu, wincl, 31);
  const float wprefix = __shfl_sync(0xffffffffu, wincl - wsum, w);   // sum of the warps before this one
  const float prefix = wprefix + incl - local;
  const float target = u[b] * total;
  if (prefix + local > target) {
    float run = prefix;
    for (int c = c0; c < c1; ++c) {
      run += sc[c];
      if (run > target && sc[c] > 0.f) { atomicMin(&s_idx, c); break; }
    }
  }
  __syncthreads();
  if (tid == 0) {
    int tok = s_idx < V ? s_idx : s_last;                    // rounding pushed the target to the total: last kept token
    if (tok < 0) tok = pad_id;                               // every score -inf (cannot happen with a live row)
    if (finished[b]) tok = pad_id;
    else if (stop_on_eos && tok == eos_id) finished[b] = 1;
    next[b] = tok;
  }
}

}  // namespace nv

using namespace nv;
#define S_(x) reinterpret_cast<cudaStream_t>(x)
#define BF(x) reinterpret_cast<__nv_bfloat16*>(x)
#define CBF(x) reinterpret_cast<const __nv_bfloat16*>(x)

extern "C" {

int nv_kv_store_prefill(const void* qkv, int64_t ld, const int* cu_seqlens, void* kcache, void* vcache, int B, int T,
                        int Smax, int HD, void* stream) {
  if (T == 0) return NV_OK;
  NV_REQUIRE((HD & 7) == 0 && (ld & 7) == 0, "nv_kv_store_prefill: alignment");
  const int64_t work = (int64_t)T * (HD >> 3);
  int grid = (int)((work + 255) / 256);
  const int cap = sm_count() * 16;
  if (grid > cap) grid = cap;
  kv_store_prefill_kernel<<<grid, 256, 0, S_(stream)>>>(CBF(qkv), ld, cu_seqlens, nullptr, BF(kcache), BF(vcache), B, Smax, HD);
  NV_LAUNCH_CHECK();
  return NV_OK;
}

// Same, appending after `cached[b]` rows that the cache already holds for sequence b (cross-step prefix reuse).
int nv_kv_store_suffix(const void* qkv, int64_t ld, const int* cu_seqlens, const int* cached, void* kcache, void* vcache,
                       int B, int T, int Smax, int HD, void* stream) {
  if (T == 0) return NV_OK;
  NV_REQUIRE((HD & 7) == 0 && (ld & 7) == 0 && cached, "nv_kv_store_suffix: alignment / null offsets");
  const int64_t work = (int64_t)T * (HD >> 3);
  int grid = (int)((work + 255) / 256);
  const int cap = sm_count() * 16;
  if (grid > cap) grid = cap;
  kv_store_prefill_kernel<<<grid, 256, 0, S_(stream)>>>(CBF(qkv), ld, cu_seqlens, cached, BF(kcache), BF(vcache), B, Smax, HD);
  NV_LAUNCH_CHECK();
  return NV_OK;
}

int nv_kv_append(const void* qkv, int64_t ld, const int* lens, void* kcache, void* vcache, int B, int Smax, int HD,
                 void* stream) {
  if (B == 0) return NV_OK;
  kv_append_kernel<<<(B * (HD >> 3) + 255) / 256, 256, 0, S_(stream)>>>(CBF(qkv), ld, lens, BF(kcache), BF(vcache), B, Smax, HD);
  NV_LAUNCH_CHECK();
  return NV_OK;
}

int nv_decode_rope_kv(void* qkv, int64_t ld, const int* lens, const void* cos_t, const void* sin_t, void* kcache, void* vcache,
                      int B, int Smax, int H, int head_dim, void* stream) {
  NV_REQUIRE(head_dim == 128 && (ld & 7) == 0, "nv_decode_rope_kv: head_dim must be 128, ld %% 8 == 0");
  if (B == 0) return NV_OK;
  const int work = B * 2 * H * 8 + B * (H * 128 / 8);
  NV_CUDA(launch_pdl(decode_rope_kv_kernel, dim3((work + 255) / 256), dim3(256), 0, S_(stream), BF(qkv), ld, lens, CBF(cos_t),
                     CBF(sin_t), BF(kcache), BF(vcache), B, Smax, H));
  return NV_OK;
}

int nv_decode_attn(const void* q, int64_t ldq, const void* kcache, const void* vcache, const int* lens, void* out,
                   int64_t ldo, int B, int Smax, int H, int head_dim, float scale, void* stream) {
  NV_REQUIRE(head_dim == 128, "nv_decode_attn: head_dim must be 128");
  if (B == 0) return NV_OK;
  NV_CUDA(launch_pdl(decode_attn_kernel<false>, dim3(B * H), dim3(DA_WARPS * 32), 0, S_(stream), CBF(q), ldq,
                     const_cast<__nv_bfloat16*>(CBF(kcache)), const_cast<__nv_bfloat16*>(CBF(vcache)), lens, BF(out), ldo, Smax, H, scale,
                     (const __nv_bfloat16*)nullptr, (const __nv_bfloat16*)nullptr, (int8_t*)nullptr, (int8_t*)nullptr));
  return NV_OK;
}

// Fused form of nv_decode_rope_kv + nv_decode_attn for one new token per sequence: qkv [B, 3*H*128] PRE-RoPE (q | k | v
// column blocks); rotates q and k at position lens[b], appends k / v to the caches at row lens[b] and attends over rows
// 0..lens[b].  qkv is not modified.
int nv_decode_attn_rope(const void* qkv, int64_t ld, const int* lens, const void* cos_t, const void* sin_t, void* kcache,
                        void* vcache, void* out, int64_t ldo, int B, int Smax, int H, int head_dim, float scale, void* stream) {
  NV_REQUIRE(head_dim == 128 && (ld & 7) == 0, "nv_decode_attn_rope: head_dim must be 128, ld %% 8 == 0");
  if (B == 0) return NV_OK;
  NV_CUDA(launch_pdl(decode_attn_kernel<true>, dim3(B * H), dim3(DA_WARPS * 32), 0, S_(stream), CBF(qkv), ld, BF(kcache), BF(vcache), lens,
                     BF(out), ldo, Smax, H, scale, CBF(cos_t), CBF(sin_t), (int8_t*)nullptr, (int8_t*)nullptr));
  return NV_OK;
}

// fp8 cache (format: include/navillm_b200.h): nv_kv_store_prefill with every stored (token, head) row quantized.
int nv_kv_store_prefill_fp8(const void* qkv, int64_t ld, const int* cu_seqlens, void* kq, void* vq, void* kexp, void* vexp, int B,
                            int T, int Smax, int H, void* stream) {
  NV_REQUIRE(B >= 0 && T >= 0 && Smax > 0 && H > 0, "nv_kv_store_prefill_fp8: bad sizes (B=%d T=%d Smax=%d H=%d)", B, T, Smax, H);
  if (T == 0 || B == 0) return NV_OK;
  NV_REQUIRE(qkv && cu_seqlens && kq && vq && kexp && vexp, "nv_kv_store_prefill_fp8: null argument");
  NV_REQUIRE((ld & 7) == 0 && ((uintptr_t)qkv & 15) == 0 && ((uintptr_t)kq & 7) == 0 && ((uintptr_t)vq & 7) == 0,
             "nv_kv_store_prefill_fp8: alignment (ld %% 8 == 0, 16-byte qkv, 8-byte caches)");
  const int64_t warps = ((int64_t)T * H + 1) / 2;
  int grid = (int)((warps + 7) / 8);
  const int cap = sm_count() * 16;
  if (grid > cap) grid = cap;
  kv_store_prefill_fp8_kernel<<<grid, 256, 0, S_(stream)>>>(CBF(qkv), ld, cu_seqlens, nullptr, reinterpret_cast<uint8_t*>(kq),
                                                            reinterpret_cast<uint8_t*>(vq), reinterpret_cast<int8_t*>(kexp),
                                                            reinterpret_cast<int8_t*>(vexp), B, Smax, H);
  NV_LAUNCH_CHECK();
  return NV_OK;
}

// nv_kv_store_suffix into an fp8 cache: the new rows of sequence b go after its cached[b] rows, each stored (token, head) row
// quantized as nv_kv_store_prefill_fp8 quantizes it.
int nv_kv_store_suffix_fp8(const void* qkv, int64_t ld, const int* cu_seqlens, const int* cached, void* kq, void* vq, void* kexp,
                           void* vexp, int B, int T, int Smax, int H, void* stream) {
  NV_REQUIRE(B >= 0 && T >= 0 && Smax > 0 && H > 0, "nv_kv_store_suffix_fp8: bad sizes (B=%d T=%d Smax=%d H=%d)", B, T, Smax, H);
  if (T == 0 || B == 0) return NV_OK;
  NV_REQUIRE(qkv && cu_seqlens && cached && kq && vq && kexp && vexp, "nv_kv_store_suffix_fp8: null argument");
  NV_REQUIRE((ld & 7) == 0 && ((uintptr_t)qkv & 15) == 0 && ((uintptr_t)kq & 7) == 0 && ((uintptr_t)vq & 7) == 0,
             "nv_kv_store_suffix_fp8: alignment (ld %% 8 == 0, 16-byte qkv, 8-byte caches)");
  const int64_t warps = ((int64_t)T * H + 1) / 2;
  int grid = (int)((warps + 7) / 8);
  const int cap = sm_count() * 16;
  if (grid > cap) grid = cap;
  kv_store_prefill_fp8_kernel<<<grid, 256, 0, S_(stream)>>>(CBF(qkv), ld, cu_seqlens, cached, reinterpret_cast<uint8_t*>(kq),
                                                            reinterpret_cast<uint8_t*>(vq), reinterpret_cast<int8_t*>(kexp),
                                                            reinterpret_cast<int8_t*>(vexp), B, Smax, H);
  NV_LAUNCH_CHECK();
  return NV_OK;
}

// nv_decode_attn_rope over an fp8 cache: the new k / v rows are quantized as they are appended.
int nv_decode_attn_rope_fp8(const void* qkv, int64_t ld, const int* lens, const void* cos_t, const void* sin_t, void* kq, void* vq,
                            void* kexp, void* vexp, void* out, int64_t ldo, int B, int Smax, int H, int head_dim, float scale,
                            void* stream) {
  NV_REQUIRE(head_dim == 128 && (ld & 7) == 0, "nv_decode_attn_rope_fp8: head_dim must be 128, ld %% 8 == 0");
  NV_REQUIRE(B >= 0 && Smax > 0 && H > 0, "nv_decode_attn_rope_fp8: bad sizes (B=%d Smax=%d H=%d)", B, Smax, H);
  if (B == 0) return NV_OK;
  NV_REQUIRE(qkv && lens && cos_t && sin_t && kq && vq && kexp && vexp && out, "nv_decode_attn_rope_fp8: null argument");
  NV_REQUIRE(((uintptr_t)qkv & 15) == 0 && ((uintptr_t)kq & 7) == 0 && ((uintptr_t)vq & 7) == 0,
             "nv_decode_attn_rope_fp8: alignment (16-byte qkv, 8-byte caches)");
  NV_CUDA(launch_pdl(decode_attn_kernel<true, true>, dim3(B * H), dim3(DA_WARPS * 32), 0, S_(stream), CBF(qkv), ld,
                     reinterpret_cast<uint8_t*>(kq), reinterpret_cast<uint8_t*>(vq), lens, BF(out), ldo, Smax, H, scale, CBF(cos_t),
                     CBF(sin_t), reinterpret_cast<int8_t*>(kexp), reinterpret_cast<int8_t*>(vexp)));
  return NV_OK;
}

int nv_argmax_masked(const void* logits, int64_t ld, int V, const int* special, int n_special, int* finished, int eos_id,
                     int pad_id, int stop_on_eos, int* next, int B, void* stream) {
  NV_REQUIRE(n_special >= 0 && n_special <= MAX_SPECIAL, "nv_argmax_masked: n_special=%d out of range (max %d)", n_special,
             MAX_SPECIAL);
  if (B == 0) return NV_OK;
  NV_CUDA(launch_pdl(argmax_kernel, dim3(B), dim3(1024), 0, S_(stream), CBF(logits), ld, V, special, n_special, finished, eos_id, pad_id,
                     stop_on_eos, next));
  return NV_OK;
}

// Sampled next token (HF sample: temperature -> top-k -> softmax -> multinomial); see sample_topk_kernel.  logits [B, V] bf16,
// u [B] uniform numbers in [0, 1), probs_out: optional fp32 [B, V] copy of the sampling distribution (tests).
int nv_sample_topk(const void* logits, int64_t ld, int V, const int* special, int n_special, int* finished, int eos_id, int pad_id,
                   int stop_on_eos, float temperature, int top_k, const float* u, int* next, float* probs_out, int B, void* stream) {
  NV_REQUIRE(logits && u && next && finished && V > 0 && temperature > 0.f, "nv_sample_topk: bad arguments (temperature must be > 0)");
  NV_REQUIRE(n_special >= 0 && n_special <= MAX_SPECIAL, "nv_sample_topk: n_special=%d out of range (max %d)", n_special,
             MAX_SPECIAL);
  NV_REQUIRE((int64_t)V * 4 <= 200 * 1024, "nv_sample_topk: vocabulary of %d does not fit the shared-memory score row", V);
  if (B == 0) return NV_OK;
  static bool attr_set = false;
  if (!attr_set) {
    NV_CUDA(cudaFuncSetAttribute(sample_topk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr_set = true;
  }
  sample_topk_kernel<<<B, SMP_THREADS, (size_t)V * 4, S_(stream)>>>(CBF(logits), ld, V, special, n_special, finished, eos_id, pad_id,
                                                                     stop_on_eos, temperature, top_k, u, next, probs_out);
  NV_LAUNCH_CHECK();
  return NV_OK;
}

// Trie mask of the next-token logits (see trie_mask_kernel).  logits [B, V] bf16 (ld), out [B, V] bf16 (ldo % 8 == 0, 16-byte
// aligned base), state int32 [B] node per row, last int32 [B] or null (no advance), miss int32 [1] (set, never cleared).
int nv_trie_mask(const void* logits, int64_t ld, void* out, int64_t ldo, int V, const int* node_ptr, const int* child_tok,
                 const int* child_node, int n_nodes, int leaf_tok, const int* special, int n_special, int* state, const int* last,
                 int* miss, int B, void* stream) {
  NV_REQUIRE(logits && out && node_ptr && child_tok && child_node && state && miss && B >= 0, "nv_trie_mask: null argument");
  NV_REQUIRE(V > 0 && n_nodes >= 1 && ld >= V && ldo >= V && (ldo & 7) == 0 && ((uintptr_t)out & 15) == 0,
             "nv_trie_mask: bad shape (V=%d, n_nodes=%d, ld=%lld, ldo=%lld; ldo %% 8 == 0 and a 16-byte aligned out needed)", V,
             n_nodes, (long long)ld, (long long)ldo);
  NV_REQUIRE(leaf_tok >= 0 && leaf_tok < V, "nv_trie_mask: leaf_tok=%d outside [0, %d)", leaf_tok, V);
  NV_REQUIRE(n_special >= 0 && n_special <= MAX_SPECIAL && (n_special == 0 || special),
             "nv_trie_mask: n_special=%d out of range (max %d)", n_special, MAX_SPECIAL);
  if (B == 0) return NV_OK;
  NV_CUDA(launch_pdl(trie_mask_kernel, dim3(B), dim3(TM_THREADS), 0, S_(stream), CBF(logits), ld, BF(out), ldo, V, node_ptr,
                     child_tok, child_node, n_nodes, leaf_tok, special, n_special, state, last, miss));
  return NV_OK;
}

int nv_add_int(int* x, int n, int delta, void* stream) {
  if (n == 0) return NV_OK;
  NV_CUDA(launch_pdl(add_int_kernel, dim3((n + 255) / 256), dim3(256), 0, S_(stream), x, n, delta));
  return NV_OK;
}

}  // extern "C"
