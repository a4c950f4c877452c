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
#include <climits>
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

// Rotary embedding of the chunk pair (c * 8 .. c * 8 + 7, 64 + c * 8 ..) of one pre-RoPE head row at position p, with the
// rounding points of rope_kernel: o1 / o2 are the rotated bf16 chunks.
__device__ __forceinline__ void rope_chunk(const __nv_bfloat16* base, const __nv_bfloat16* __restrict__ cos_t,
                                           const __nv_bfloat16* __restrict__ sin_t, int p, int c, uint4& o1, uint4& o2) {
  float x1[8], x2[8], c1[8], s1[8], c2[8], s2[8];
  unpack8d(*reinterpret_cast<const uint4*>(base + c * 8), x1);
  unpack8d(*reinterpret_cast<const uint4*>(base + 64 + c * 8), x2);
  unpack8d(*reinterpret_cast<const uint4*>(cos_t + (int64_t)p * 128 + c * 8), c1);
  unpack8d(*reinterpret_cast<const uint4*>(sin_t + (int64_t)p * 128 + c * 8), s1);
  unpack8d(*reinterpret_cast<const uint4*>(cos_t + (int64_t)p * 128 + 64 + c * 8), c2);
  unpack8d(*reinterpret_cast<const uint4*>(sin_t + (int64_t)p * 128 + 64 + c * 8), s2);
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

// BEAM = true (beam search): blockIdx.x / H is a beam row r of prompt r / nbeam.  Keys [0, plens[prompt]) come from the
// prompt cache pk / pv ([B, Sp, HD], exponents pke / pve [B, Sp, H]) that all beams of the prompt share; generated key i (key
// plens + i) from row (src[r, i], i) of the generated cache kc / vc ([B * nbeam, Smax, HD]).  The new token is generated key
// lens[r] - plens: it is written at (r, that index), and src[r, that index] must name r.  Only the addresses differ from the
// contiguous kernel: the same keys in the same order give the same bits.
template <bool FP8>
struct BeamKV {
  const kv_elem_t<FP8>* pk;
  const kv_elem_t<FP8>* pv;
  const int8_t* pke;
  const int8_t* pve;
  const int* src;
  const int* plens;
  int nbeam;
  int Sp;
};

template <bool ROPE, bool FP8 = false, bool BEAM = false>
__global__ void __launch_bounds__(DA_WARPS * 32) decode_attn_kernel(const __nv_bfloat16* __restrict__ q, int64_t ldq,
                                                          kv_elem_t<FP8>* __restrict__ kc, kv_elem_t<FP8>* __restrict__ vc,
                                                          const int* __restrict__ lens, __nv_bfloat16* __restrict__ out,
                                                          int64_t ldo, int Smax, int H, float scale,
                                                          const __nv_bfloat16* __restrict__ cos_t,
                                                          const __nv_bfloat16* __restrict__ sin_t,
                                                          int8_t* __restrict__ ke, int8_t* __restrict__ ve, BeamKV<FP8> bk) {
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
  int P = 0, bp = 0;                                    // BEAM: prompt keys of this row, and its prompt
  if constexpr (BEAM) {
    bp = b / bk.nbeam;
    P = bk.plens[bp];
  }
  if (ROPE) {
    const int p = n - 1;
    const int pw = p - P;                               // cache row of the new k / v
    if (w == 0) {
      uint4 r0 = make_uint4(0, 0, 0, 0), r1 = r0;       // FP8: this lane's chunks of the new k row (lanes 8..15) or v row (16..31)
      if (lane < 16) {                                  // lanes 0..7: q chunk c, lanes 8..15: k chunk c
        const int c = lane & 7, is_k = lane >> 3;
        const __nv_bfloat16* base = q + (int64_t)b * ldq + (is_k ? HD : 0) + h * 128;
        uint4 o1, o2;
        rope_chunk(base, cos_t, sin_t, p, c, o1, o2);
        if (!is_k) {
          s_q[c] = o1; s_q[8 + c] = o2;
        } else if constexpr (FP8) {
          r0 = o1; r1 = o2;
        } else if (pw < Smax) {
          __nv_bfloat16* dst = kc + ((int64_t)b * Smax + pw) * HD + h * 128;
          *reinterpret_cast<uint4*>(dst + c * 8) = o1;
          *reinterpret_cast<uint4*>(dst + 64 + c * 8) = o2;
        }
      } else if constexpr (FP8) {
        r0 = *reinterpret_cast<const uint4*>(q + (int64_t)b * ldq + 2 * HD + h * 128 + (lane - 16) * 8);
      } else if (pw < Smax) {                           // lanes 16..31: this head's v (16 x 16 bytes)
        const int v = lane - 16;
        *reinterpret_cast<uint4*>(vc + ((int64_t)b * Smax + pw) * HD + h * 128 + v * 8) =
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
        if (lane >= 8 && pw < Smax) {
          const int64_t row = (int64_t)b * Smax + pw;
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
        const kv_elem_t<FP8>* kb = kc;
        const kv_elem_t<FP8>* vb = vc;
        const int8_t* keb = ke;
        const int8_t* veb = ve;
        int64_t row = (int64_t)b * Smax + jb + u;
        if constexpr (BEAM) {
          const int j = jb + u;
          if (j < P) {
            row = (int64_t)bp * bk.Sp + j;
            kb = bk.pk; vb = bk.pv; keb = bk.pke; veb = bk.pve;
          } else {
            row = (int64_t)bk.src[(int64_t)b * Smax + (j - P)] * Smax + (j - P);
          }
        }
        const int64_t off = row * HD + h * 128 + hl * 8;
        kr[u] = *reinterpret_cast<const raw_t*>(kb + off);
        vr[u] = *reinterpret_cast<const raw_t*>(vb + off);
        if constexpr (FP8) {
          kx[u] = keb[row * H + h];
          vx[u] = veb[row * H + h];
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

// ---- speculative verify step: w consecutive query rows per sequence (prompt-lookup decoding) ----
// decode_attn_kernel<true, FP8> for a window of W <= WIN_MAX new tokens per sequence: qkv row b * W + r (pre-RoPE) is the token at
// position lens[b] + r.  Every CTA rotates the q, k and v of the window rows its queries see into shared memory, stores the
// rotated k and the v of its own query rows at rows lens[b] + r of the caches (fp8: quantized as the decode kernel quantizes
// them), and query r attends over keys 0 .. lens[b] + r: cached keys from global memory, the window's from shared memory.  A
// cached key is read once for the QPC queries of the CTA; grid (B * H, ceil(W / QPC)), so a window of more than QPC rows reads
// the cache once per QPC queries (the second read mostly from L2).
// Bit-identity: for each query the keys go to warps and half-warps by absolute index and the per-warp states merge in warp
// order, exactly as in decode_attn_kernel at lens[b] + r; a key past a query's range leaves its (m, l, acc) unchanged (the
// correction factor is exp2(0) = 1, and no term is added), so query r's output and every cache byte equal those of W
// sequential decode_attn_rope calls.  The arithmetic is spelled out with _rn intrinsics in the order ptxas gives
// decode_attn_kernel (fma dot products from 0, the rescale a separate multiply, p * v fused into the sum, the merges as
// fma(x, a, y * ao)), so that no contraction choice can differ between the two kernels.
constexpr int WIN_MAX = 16;

template <bool FP8, int QPC>
__global__ void __launch_bounds__(DA_WARPS * 32) decode_attn_window_kernel(const __nv_bfloat16* __restrict__ qkv, int64_t ld,
                                                                           kv_elem_t<FP8>* __restrict__ kc, kv_elem_t<FP8>* __restrict__ vc,
                                                                           int8_t* __restrict__ ke, int8_t* __restrict__ ve,
                                                                           const int* __restrict__ lens, __nv_bfloat16* __restrict__ out,
                                                                           int64_t ldo, int Smax, int H, int W, float scale,
                                                                           const __nv_bfloat16* __restrict__ cos_t,
                                                                           const __nv_bfloat16* __restrict__ sin_t) {
  using raw_t = typename std::conditional<FP8, uint2, uint4>::type;
  __shared__ float s_m[QPC][DA_WARPS], s_l[QPC][DA_WARPS];
  __shared__ float s_acc[QPC][DA_WARPS][128];
  __shared__ uint4 s_q[QPC][16];                       // rotated q of the CTA's queries (bf16 x 128)
  __shared__ raw_t s_kw[WIN_MAX][16], s_vw[WIN_MAX][16];   // the window's K / V rows as the cache holds them
  __shared__ int s_kx[WIN_MAX], s_vx[WIN_MAX];         // FP8: their exponents
  griddep_launch();
  griddep_wait();
  const int b = blockIdx.x / H, h = blockIdx.x % H;
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int half = lane >> 4, hl = lane & 15;
  const int HD = H * 128;
  const int L = lens[b];
  const int q0 = blockIdx.y * QPC, qe = min(W, q0 + QPC);   // this CTA's queries q0 .. qe - 1
  // rotate: warp w takes window rows w, w + 8, ..; lanes 0..7 the q chunk pairs, 8..15 the k chunk pairs, 16..31 the v chunks
  for (int r = w; r < qe; r += DA_WARPS) {
    const int p = L + r;
    const __nv_bfloat16* row = qkv + (int64_t)(b * W + r) * ld;
    const bool store = r >= q0 && p < Smax;            // this CTA writes the K / V of its own query rows
    uint4 r0 = make_uint4(0, 0, 0, 0), r1 = r0;
    if (lane < 16) {
      const int c = lane & 7, is_k = lane >> 3;
      if (is_k || r >= q0) {
        rope_chunk(row + (is_k ? HD : 0) + h * 128, cos_t, sin_t, p, c, r0, r1);
        if (!is_k) {
          s_q[r - q0][c] = r0; s_q[r - q0][8 + c] = r1;
        } else if constexpr (!FP8) {
          s_kw[r][c] = r0; s_kw[r][8 + c] = r1;
          if (store) {
            __nv_bfloat16* dst = kc + ((int64_t)b * Smax + p) * HD + h * 128;
            *reinterpret_cast<uint4*>(dst + c * 8) = r0;
            *reinterpret_cast<uint4*>(dst + 64 + c * 8) = r1;
          }
        }
      }
    } else {
      r0 = *reinterpret_cast<const uint4*>(row + 2 * HD + h * 128 + (lane - 16) * 8);
      if constexpr (!FP8) {
        s_vw[r][lane - 16] = r0;
        if (store) *reinterpret_cast<uint4*>(vc + ((int64_t)b * Smax + p) * HD + h * 128 + (lane - 16) * 8) = r0;
      }
    }
    if constexpr (FP8) {
      // the row amax and exponent of the k row (lanes 8..15) and the v row (16..31), as decode_attn_kernel finds them
      if (lane < 8) r0 = r1 = make_uint4(0, 0, 0, 0);
      uint32_t m = max(bf16x8_amax_bits(r0), bf16x8_amax_bits(r1));
#pragma unroll
      for (int o = 1; o < 8; o <<= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
      const uint32_t m8 = __shfl_xor_sync(0xffffffffu, m, 8);
      if (lane >= 16) m = max(m, m8);
      const int e = fp8_row_exponent(__uint_as_float(m << 16));
      const float inv = fp8_pow2(-e);
      const int64_t crow = (int64_t)b * Smax + p;
      if (lane >= 8 && lane < 16) {
        const int c = lane & 7;
        const uint2 k0 = fp8x8_from_bf16x8(r0, inv), k1 = fp8x8_from_bf16x8(r1, inv);
        s_kw[r][c] = k0; s_kw[r][8 + c] = k1;
        if (lane == 8) s_kx[r] = e;
        if (store) {
          *reinterpret_cast<uint2*>(kc + crow * HD + h * 128 + c * 8) = k0;
          *reinterpret_cast<uint2*>(kc + crow * HD + h * 128 + 64 + c * 8) = k1;
          if (lane == 8) ke[crow * H + h] = (int8_t)e;
        }
      } else if (lane >= 16) {
        const uint2 v0 = fp8x8_from_bf16x8(r0, inv);
        s_vw[r][lane - 16] = v0;
        if (lane == 16) s_vx[r] = e;
        if (store) {
          *reinterpret_cast<uint2*>(vc + crow * HD + h * 128 + (lane - 16) * 8) = v0;
          if (lane == 16) ve[crow * H + h] = (int8_t)e;
        }
      }
    }
  }
  __syncthreads();
  const int nq = qe - q0;
  const int n = L + qe;                                 // keys the CTA's last query sees
  const float sl2 = scale * 1.4426950408889634f;
  float m[QPC], l[QPC], acc[QPC][8];
#pragma unroll
  for (int qi = 0; qi < QPC; ++qi) {
    m[qi] = -INFINITY; l[qi] = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[qi][i] = 0.f;
  }
  constexpr int KPI = 4;
  auto load_keys = [&](int jb, raw_t (&kr)[KPI], raw_t (&vr)[KPI], int (&kx)[KPI], int (&vx)[KPI]) {
#pragma unroll
    for (int u = 0; u < KPI; ++u) {
      const int j = jb + u;
      if (j < L) {
        const int64_t row = (int64_t)b * Smax + j;
        const int64_t off = row * HD + h * 128 + hl * 8;
        kr[u] = *reinterpret_cast<const raw_t*>(kc + off);
        vr[u] = *reinterpret_cast<const raw_t*>(vc + off);
        if constexpr (FP8) {
          kx[u] = ke[row * H + h];
          vx[u] = ve[row * H + h];
        }
      } else if (j < n) {
        kr[u] = s_kw[j - L][hl];
        vr[u] = s_vw[j - L][hl];
        if constexpr (FP8) {
          kx[u] = s_kx[j - L];
          vx[u] = s_vx[j - L];
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
#pragma unroll
    for (int qi = 0; qi < QPC; ++qi) {
      if (qi < nq) {                                    // uniform over the CTA
        const int nk = L + q0 + qi + 1;                 // keys visible to this query
        float qf[8];
        unpack8d(s_q[qi][hl], qf);
        float sc[KPI];
#pragma unroll
        for (int u = 0; u < KPI; ++u) {
          float kf[8];
          unpack(kraw[u], kx[u], kf);
          float s = 0.f;
#pragma unroll
          for (int i = 0; i < 8; ++i) s = __fmaf_rn(qf[i], kf[i], s);
          sc[u] = s;
        }
#pragma unroll
        for (int o = 8; o > 0; o >>= 1)
#pragma unroll
          for (int u = 0; u < KPI; ++u) sc[u] += __shfl_xor_sync(0xffffffffu, sc[u], o);
        float mn = m[qi];
#pragma unroll
        for (int u = 0; u < KPI; ++u)
          if (jb + u < nk) mn = fmaxf(mn, sc[u]);
        if (mn != -INFINITY) {
          const float a = exp2f(__fmul_rn(__fsub_rn(m[qi], mn), sl2));
          l[qi] = __fmul_rn(l[qi], a);
#pragma unroll
          for (int i = 0; i < 8; ++i) acc[qi][i] = __fmul_rn(acc[qi][i], a);
#pragma unroll
          for (int u = 0; u < KPI; ++u) {
            if (jb + u < nk) {
              const float p = exp2f(__fmul_rn(__fsub_rn(sc[u], mn), sl2));
              float vf[8];
              unpack(vraw[u], vx[u], vf);
              l[qi] = __fadd_rn(l[qi], p);
#pragma unroll
              for (int i = 0; i < 8; ++i) acc[qi][i] = __fmaf_rn(p, vf[i], acc[qi][i]);
            }
          }
          m[qi] = mn;
        }
      }
    }
  }
#pragma unroll
  for (int qi = 0; qi < QPC; ++qi) {
    if (qi < nq) {
      const float mo = __shfl_xor_sync(0xffffffffu, m[qi], 16), lo = __shfl_xor_sync(0xffffffffu, l[qi], 16);
      const float mn = fmaxf(m[qi], mo);
      const float a = (m[qi] == -INFINITY) ? 0.f : exp2f(__fmul_rn(__fsub_rn(m[qi], mn), sl2));
      const float ao = (mo == -INFINITY) ? 0.f : exp2f(__fmul_rn(__fsub_rn(mo, mn), sl2));
      l[qi] = __fmaf_rn(l[qi], a, __fmul_rn(lo, ao));
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float other = __shfl_xor_sync(0xffffffffu, acc[qi][i], 16);
        acc[qi][i] = __fmaf_rn(acc[qi][i], a, __fmul_rn(other, ao));
      }
      m[qi] = mn;
      if (lane < 16) {
        if (lane == 0) { s_m[qi][w] = m[qi]; s_l[qi][w] = l[qi]; }
#pragma unroll
        for (int i = 0; i < 8; ++i) s_acc[qi][w][hl * 8 + i] = acc[qi][i];
      }
    }
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < nq * 128; idx += DA_WARPS * 32) {
    const int qi = idx >> 7, d = idx & 127;
    float mm = s_m[qi][0];
#pragma unroll
    for (int k = 1; k < DA_WARPS; ++k) mm = fmaxf(mm, s_m[qi][k]);
    float num = 0.f, den = 0.f;
#pragma unroll
    for (int k = 0; k < DA_WARPS; ++k) {
      const float a = (s_m[qi][k] == -INFINITY) ? 0.f : exp2f(__fmul_rn(__fsub_rn(s_m[qi][k], mm), sl2));
      num = __fmaf_rn(s_acc[qi][k][d], a, num);
      den = __fmaf_rn(s_l[qi][k], a, den);
    }
    out[(int64_t)(b * W + q0 + qi) * ldo + h * 128 + d] = __float2bfloat16_rn(num / den);
  }
}

// Special ids masked by argmax_kernel and sample_topk_kernel: they are staged in shared memory, so the host entry points
// reject longer lists.
constexpr int MAX_SPECIAL = 64;

// The masked argmax of one logits row over the whole CTA (s_special: the n_special special ids, already in shared memory;
// sv / si: 32 floats / ints of shared scratch): the first index of the largest value over non-special columns, like
// torch.argmax.  Valid in thread 0.
__device__ __forceinline__ int argmax_row(const __nv_bfloat16* __restrict__ row, int64_t ld, int V, const int* s_special, int ns,
                                          float* sv, int* si) {
  float best = -INFINITY;
  int bi = V;
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
  }
  return bi;
}

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
  const int bi = argmax_row(logits + (int64_t)b * ld, ld, V, s_special, ns, sv, si);
  if (threadIdx.x == 0) {
    int tok = bi;
    if (finished[b]) tok = pad_id;
    else if (stop_on_eos && tok == eos_id) finished[b] = 1;
    next[b] = tok;
  }
}

// ---- prompt-lookup drafts and their verification (generation.lookup_decode) ----
constexpr int LD_THREADS = 128;

// One CTA per row: HF's PromptLookupCandidateGenerator on the row's history hist[b, :hist_len[b]] (its non-pad prompt ids, then
// its generated tokens).  For n = min(ngram, len - 1) down to 1, the earliest i with hist[i .. i + n) equal to the last n tokens
// and i + n < len: the drafts are the up to K tokens from i + n on, cut at the end of the history and at the first special id or
// EOS (the argmax never accepts a special id; HF cuts at EOS); the first n that matches decides, even if its drafts come out
// empty.  drafts [B, K] = the drafts, -1 past them; win [B, K + 1] = the verify window's ids: the last token, then the drafts,
// then the last token again in place of a missing draft (any valid id: its row's argmax is never looked at).  A finished row
// gets no drafts.
__global__ void __launch_bounds__(LD_THREADS) lookup_draft_kernel(const int* __restrict__ hist, int ld_hist,
                                                                  const int* __restrict__ hist_len, const int* __restrict__ finished,
                                                                  const int* __restrict__ special, int n_special, int eos_id, int K,
                                                                  int ngram, int* __restrict__ drafts, int* __restrict__ win) {
  __shared__ int s_special[MAX_SPECIAL];
  __shared__ int s_best;
  griddep_launch();
  griddep_wait();
  const int b = blockIdx.x, tid = threadIdx.x;
  const int* row = hist + (int64_t)b * ld_hist;
  const int L = hist_len[b];
  const bool live = !finished[b];
  if (tid < n_special) s_special[tid] = special[tid];
  int start = -1;
  for (int n = live ? min(ngram, L - 1) : 0; n >= 1; --n) {  // uniform over the CTA
    __syncthreads();                                         // s_best of the previous n is read
    if (tid == 0) s_best = INT_MAX;
    __syncthreads();
    for (int i = tid; i + n < L; i += LD_THREADS) {
      bool match = true;
      for (int t = 0; t < n && match; ++t) match = row[i + t] == row[L - n + t];
      if (match) atomicMin(&s_best, i);
    }
    __syncthreads();
    if (s_best != INT_MAX) {
      start = s_best + n;
      break;
    }
  }
  __syncthreads();
  if (tid == 0) {
    const int last = row[L - 1];
    win[b * (K + 1)] = last;
    bool go = start >= 0;
    for (int i = 0; i < K; ++i) {
      int tok = -1;
      if (go && start + i < L) {
        tok = row[start + i];
        bool sp = tok == eos_id;
        for (int s = 0; s < n_special; ++s) sp |= s_special[s] == tok;
        if (sp) tok = -1;
      }
      go = tok >= 0;
      drafts[b * K + i] = tok;
      win[b * (K + 1) + 1 + i] = go ? tok : last;
    }
  }
}

// One CTA per row of a verify window (K + 1 logits rows b * (K + 1) + j, row j the prediction after window token j): t_j = the
// masked argmax of row j (argmax_kernel's rule), computed for j = 0, 1, .. while draft d_{j+1} = drafts[b, j] equals t_j.  The row
// emits t_0 .. t_m (m accepted drafts), cut after the first EOS when stop_on_eos and at max_new tokens: each goes to out[b, n_out[b]]
// and to the history.  lens[b] advances by the tokens emitted (the window rows whose K / V are now valid), n_acc[b] by the
// accepted drafts among them, and a row that emitted EOS or reached max_new is finished: it emits nothing more.
__global__ void __launch_bounds__(1024) lookup_accept_kernel(const __nv_bfloat16* __restrict__ logits, int64_t ld, int V,
                                                             const int* __restrict__ special, int n_special,
                                                             const int* __restrict__ drafts, int K, int* __restrict__ finished,
                                                             int eos_id, int stop_on_eos, int max_new, int* __restrict__ out,
                                                             int ld_out, int* __restrict__ hist, int ld_hist,
                                                             int* __restrict__ hist_len, int* __restrict__ n_out,
                                                             int* __restrict__ lens, int* __restrict__ n_acc) {
  __shared__ float sv[32];
  __shared__ int si[32];
  __shared__ int s_special[MAX_SPECIAL];
  __shared__ int s_t[WIN_MAX];
  __shared__ int s_more;
  griddep_launch();
  griddep_wait();
  const int b = blockIdx.x;
  if (finished[b]) return;                                   // uniform over the CTA
  if (threadIdx.x < n_special) s_special[threadIdx.x] = special[threadIdx.x];
  __syncthreads();
  int m = 0;
  for (int j = 0; j <= K; ++j) {
    const int t = argmax_row(logits + (int64_t)(b * (K + 1) + j) * ld, ld, V, s_special, n_special, sv, si);
    if (threadIdx.x == 0) {
      s_t[j] = t;
      s_more = j < K && drafts[b * K + j] == t;
    }
    __syncthreads();
    m = j;
    if (!s_more) break;
    __syncthreads();                                         // sv / si and s_more are read before the next row
  }
  if (threadIdx.x == 0) {
    int cnt = n_out[b], hl = hist_len[b], e = 0;
    bool fin = false;
    for (int j = 0; j <= m && cnt < max_new; ++j) {
      const int tok = s_t[j];
      out[(int64_t)b * ld_out + cnt++] = tok;
      hist[(int64_t)b * ld_hist + hl++] = tok;
      ++e;
      if (stop_on_eos && tok == eos_id) {
        fin = true;
        break;
      }
    }
    n_out[b] = cnt;
    hist_len[b] = hl;
    lens[b] += e;
    n_acc[b] += e > 0 ? e - 1 : 0;
    if (fin || cnt >= max_new) finished[b] = 1;
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

// ---- per-step scores (generate(return_dict_in_generate=True, output_scores=True): HF's `scores`) ----
// The scores live in bf16 planes [G, rows, ld]; the plane a launch writes is read on the device, step[b * step_stride] (a
// counter the captured step advances, or the beams' prompt_state), so one captured graph writes a new plane at every replay.
struct ScoresOut {
  __nv_bfloat16* p;
  int64_t ld;                                // row stride
  int64_t plane;                             // plane stride (elements)
  const int* step;
  int step_stride;
  __device__ __forceinline__ __nv_bfloat16* row(int b, int r) const {
    return p + (int64_t)step[b * step_stride] * plane + (int64_t)r * ld;
  }
};

constexpr int SS_THREADS = 256;
constexpr int SS_CHUNK = SS_THREADS * 8;     // columns per CTA: one 16-byte copy per thread

// Columns [c0, c0 + SS_CHUNK) of one row: out = in, then the special ids among them -inf (models/modified_lm.py:121-123: the
// reference's logits carry the mask).  16-byte copies when both rows are 16-byte aligned (the logits and scores buffers are),
// element copies otherwise and at the row's end.
__device__ __forceinline__ void scores_copy_chunk(const __nv_bfloat16* __restrict__ in, __nv_bfloat16* __restrict__ out, int V,
                                                  int c0, const int* __restrict__ special, int ns) {
  const int c = c0 + threadIdx.x * 8;
  const bool vec = ((reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(out)) & 15) == 0;
  if (vec && c + 8 <= V) {
    *reinterpret_cast<uint4*>(out + c) = *reinterpret_cast<const uint4*>(in + c);
  } else {
    for (int i = c; i < min(c + 8, V); ++i) out[i] = in[i];
  }
  __syncthreads();
  if (threadIdx.x < ns) {
    const int sp = special[threadIdx.x];
    if (sp >= c0 && sp < c0 + SS_CHUNK && sp < V) out[sp] = __float2bfloat16_rn(-INFINITY);
  }
}

// Grid (R, column chunks): plane step[0], row r = src row r with the special ids -inf (greedy / trie / contrastive: the values
// the pick reads, which mask the special ids internally).
__global__ void __launch_bounds__(SS_THREADS) scores_store_kernel(const __nv_bfloat16* __restrict__ src, int64_t ld, int V,
                                                                  const int* __restrict__ special, int n_special, ScoresOut so) {
  griddep_launch();
  griddep_wait();
  scores_copy_chunk(src + (int64_t)blockIdx.x * ld, so.row(0, blockIdx.x), V, blockIdx.y * SS_CHUNK, special, n_special);
}

// Grid (B, W, column chunks): after nv_lookup_accept, window row j of prompt b emitted a token iff j < n_out[b] - n_prev[b]; its
// logits (the row that picked it) go to plane n_prev[b] + j, row b, special ids -inf.
__global__ void __launch_bounds__(SS_THREADS) lookup_scores_kernel(const __nv_bfloat16* __restrict__ logits, int64_t ld, int V,
                                                                   const int* __restrict__ special, int n_special,
                                                                   const int* __restrict__ n_prev, const int* __restrict__ n_out, int W,
                                                                   __nv_bfloat16* __restrict__ scores, int64_t ld_s, int64_t plane) {
  griddep_launch();
  griddep_wait();
  const int b = blockIdx.x, j = blockIdx.y, t0 = n_prev[b];
  if (j >= n_out[b] - t0) return;                            // uniform over the CTA
  scores_copy_chunk(logits + (int64_t)(b * W + j) * ld, scores + (int64_t)(t0 + j) * plane + (int64_t)b * ld_s, V,
                    blockIdx.z * SS_CHUNK, special, n_special);
}

// ---- sampled decoding (HF GenerationMixin.sample as the reference reaches it with do_sample=True, tasks/agents/llava.py:58-62
// -> models/nav_model.py:388-396): next-token scores -> TemperatureLogitsWarper (scores / T, in the logits' dtype: bf16) ->
// TopKLogitsWarper (transformers' generation default top_k = 50: every score strictly below the k-th largest becomes -inf,
// ties at the k-th value stay) -> TopPLogitsWarper when top_p < 1 (see SMP_LIST) -> softmax (fp32 inside, rounded to bf16) -> one multinomial draw.  One CTA per row: the
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

// sum of one float per thread over the CTA (SMP_THREADS = 32 warps): warp butterflies, then the 32 warp sums in warp order
__device__ __forceinline__ float smp_cta_sum(float part, float* red) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
  if (lane == 0) red[w] = part;
  __syncthreads();
  float s = red[lane];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  __syncthreads();
  return s;
}

// exclusive prefix of one int per thread over the CTA, in thread order
__device__ __forceinline__ int smp_cta_exclusive(int x, int* ired) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int incl = x;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  if (lane == 31) ired[w] = incl;
  __syncthreads();
  const int ws = ired[lane];
  int wincl = ws;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, wincl, o);
    if (lane >= o) wincl += t;
  }
  const int wprefix = __shfl_sync(0xffffffffu, wincl - ws, w);
  __syncthreads();
  return wprefix + incl - x;
}

// Top-p (TopPLogitsWarper of transformers 4.28, after top-k): the survivors of top-k sorted by (score, token index) ascending,
// their bf16 softmax probabilities p summed in that order, and every position whose bf16-rounded running sum is <= p_thr
// (= bf16(1 - top_p)) removed, the last (largest) always kept.  Up to SMP_LIST survivors (top_k = 50 plus ties) are sorted
// and walked with an fp32 running sum (torch's CPU cumsum of a bf16 tensor).  Above that (top_k = 0: the full vocabulary)
// two radix passes over the 16-bit key sum the probability mass per key exactly (fixed point, 2^-60) to find the key whose
// prefix crosses the threshold; there the running sum is the exact prefix rounded to bf16, which differs from the fp32
// walk only within fp32 summation noise.  Scores are bf16 values, so all tokens of one key share one p, and only the
// order inside the crossing key needs the token index: its lowest indices go first (a stable ascending sort).
constexpr int SMP_LIST = 1024;
constexpr double SMP_FIX = 1152921504606846976.0;      // 2^60: p < 2 always, so a sum of p fits 64 bits

__device__ __forceinline__ unsigned long long smp_fix(float p) { return (unsigned long long)((double)p * SMP_FIX); }
__device__ __forceinline__ float smp_unfix_bf16(unsigned long long x) { return __bfloat162float(__double2bfloat16((double)x / SMP_FIX)); }

// SCORES (nv_sample_scores): the warped bf16 scores -- bf16(logit / T), -inf for the special ids and outside the kept set of
// top-k / top-p (4.28's next_token_scores after logits_warper) -- also go to so.row(0, b).
template <bool SCORES>
__device__ __forceinline__ void sample_body(const __nv_bfloat16* __restrict__ logits, int64_t ld, int V, const int* __restrict__ special,
                                            int n_special, int* __restrict__ finished, int eos_id, int pad_id, int stop_on_eos,
                                            float temperature, int top_k, int use_top_p, float p_thr, const float* __restrict__ u,
                                            int* __restrict__ next, float* __restrict__ probs_out, const ScoresOut& so) {
  extern __shared__ float sc[];                              // [V] scores, then probabilities
  __shared__ int hist[256];
  __shared__ float red[32];
  __shared__ int s_special[MAX_SPECIAL];
  __shared__ int s_idx, s_last;
  __shared__ uint32_t s_lst[SMP_LIST], s_srt[SMP_LIST];     // top-p: (key << 16 | slot) of the survivors of top-k, sorted
  __shared__ float s_lv[SMP_LIST];                           // their scores, by slot
  __shared__ unsigned long long s_mass[256];
  __shared__ int s_n, s_ck, s_cr, s_ci, s_bin;
  __shared__ unsigned long long s_acc;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int ns = n_special;
  if (tid < ns) s_special[tid] = special[tid];
  if (tid < 256) hist[tid] = 0;
  if (tid == 0) { s_idx = V; s_last = -1; s_n = 0; s_ck = 0; s_cr = 0; s_ci = 0; }
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
  float denom;
  __nv_bfloat16* srow = nullptr;
  if constexpr (SCORES) srow = so.row(0, b);
  if (!use_top_p) {
    float part = 0.f;
    for (int c = tid; c < V; c += SMP_THREADS) {
      const float v = sc[c];
      const float e = (smp_key16(v) >= thr_key && v > -INFINITY) ? expf(v - mx) : 0.f;
      if constexpr (SCORES) srow[c] = __float2bfloat16_rn((smp_key16(v) >= thr_key && v > -INFINITY) ? v : -INFINITY);
      sc[c] = e;
      part += e;
    }
    denom = smp_cta_sum(part, red);
  } else {
    // 3a. the same denominator with the scores kept in sc; the survivors of top-k go to the list while it has room
    float part = 0.f;
    for (int c = tid; c < V; c += SMP_THREADS) {
      const float v = sc[c];
      const uint32_t key = smp_key16(v);
      const bool kept = key >= thr_key && v > -INFINITY;
      // one shared-memory atomic per warp and iteration, not per survivor (top_k = 0 keeps the whole row)
      const unsigned act = __activemask();
      const unsigned kb = __ballot_sync(act, kept);
      const int leader = __ffs(act) - 1;
      int base = 0;
      if (lane == leader && kb) base = atomicAdd(&s_n, __popc(kb));
      base = __shfl_sync(act, base, leader);
      if (kept) {
        part += expf(v - mx);
        const int slot = base + __popc(kb & ((1u << lane) - 1u));
        if (slot < SMP_LIST) { s_lst[slot] = (key << 16) | (uint32_t)slot; s_lv[slot] = v; }
      }
    }
    denom = smp_cta_sum(part, red);
    const int n = s_n;
    auto prob = [&](float v) { return bf16_round(expf(v - mx) / denom); };
    // 3b. the cut: tie group s_ck, of which the s_cr lowest token indices are removed (everything below it is removed)
    if (n <= SMP_LIST) {
      if (tid < n) {                                         // rank sort: the list entries are distinct
        const uint32_t x = s_lst[tid];
        int r = 0;
        for (int j = 0; j < n; ++j) r += s_lst[j] < x;
        s_srt[r] = x;
      }
      __syncthreads();
      if (tid == 0 && n > 0) {
        float run = 0.f;
        int m = 0;
        for (; m < n - 1; ++m) {
          run += prob(s_lv[s_srt[m] & 0xffffu]);
          if (bf16_round(run) > p_thr) break;
        }
        const uint32_t ck = s_srt[m] >> 16;
        int first = m;
        while (first > 0 && (s_srt[first - 1] >> 16) == ck) --first;
        s_ck = (int)ck;
        s_cr = m - first;
      }
    } else {
      // hist / s_mass: count and fixed-point mass per high key byte, then per low byte of the crossing high byte
      for (int pass = 0; pass < 2; ++pass) {
        if (tid < 256) { hist[tid] = 0; s_mass[tid] = 0ull; }
        __syncthreads();
        for (int c = tid; c < V; c += SMP_THREADS) {
          const float v = sc[c];
          const uint32_t key = smp_key16(v);
          if (key >= thr_key && v > -INFINITY && (pass == 0 || (int)(key >> 8) == s_bin)) {
            const int bin = pass == 0 ? (int)(key >> 8) : (int)(key & 255u);
            atomicAdd(&hist[bin], 1);
            atomicAdd(&s_mass[bin], smp_fix(prob(v)));
          }
        }
        __syncthreads();
        if (tid == 0) {
          unsigned long long acc = pass == 0 ? 0ull : s_acc, at = acc;   // at: the mass below bin `last`
          int cross = -1, last = -1;
          for (int i = 0; i < 256 && cross < 0; ++i) {
            if (hist[i] == 0) continue;
            last = i;
            at = acc;
            if (smp_unfix_bf16(acc + s_mass[i]) > p_thr) cross = i;
            else acc += s_mass[i];
          }
          const int bin = last;                                  // the crossing bin, or the top one when none crosses
          acc = at;
          if (pass == 0) {
            s_bin = bin;
            s_acc = acc;
          } else {
            const int ng = hist[bin];
            const unsigned long long pg = s_mass[bin] / (unsigned long long)ng;   // every token of one key has the same p
            int lo = 0, hi = ng - 1;                             // the first group member whose running sum exceeds p_thr
            if (cross >= 0) {
              while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (smp_unfix_bf16(acc + (unsigned long long)(mid + 1) * pg) > p_thr) hi = mid;
                else lo = mid + 1;
              }
            }
            s_ck = (s_bin << 8) | bin;
            s_cr = cross >= 0 ? lo : ng - 1;
          }
        }
        __syncthreads();
      }
    }
    __syncthreads();
    // 3c. the token index where the cut falls: the s_cr-th (0-based) token of key s_ck in index order
    const uint32_t ck = (uint32_t)s_ck;
    const int cr = s_cr;
    {
      const int CH = (V + SMP_THREADS - 1) / SMP_THREADS;
      const int c0 = min(tid * CH, V), c1 = min(c0 + CH, V);
      int cnt = 0;
      for (int c = c0; c < c1; ++c) cnt += smp_key16(sc[c]) == ck;
      const int before = smp_cta_exclusive(cnt, hist);
      if (before <= cr && cr < before + cnt) {
        int k = before;
        for (int c = c0; c < c1; ++c)
          if (smp_key16(sc[c]) == ck && k++ == cr) { s_ci = c; break; }
      }
      __syncthreads();
    }
    const int ci = s_ci;
    // 3d. a fresh softmax over the survivors of top-p (the maximum always survives, so mx stands)
    part = 0.f;
    for (int c = tid; c < V; c += SMP_THREADS) {
      const float v = sc[c];
      const uint32_t key = smp_key16(v);
      const bool keep = key >= thr_key && v > -INFINITY && (key > ck || (key == ck && c >= ci));
      const float e = keep ? expf(v - mx) : 0.f;
      if constexpr (SCORES) srow[c] = __float2bfloat16_rn(keep ? v : -INFINITY);
      sc[c] = e;
      part += e;
    }
    denom = smp_cta_sum(part, red);
  }
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

__global__ void __launch_bounds__(SMP_THREADS) sample_topk_kernel(const __nv_bfloat16* __restrict__ logits, int64_t ld, int V,
                                                                  const int* __restrict__ special, int n_special,
                                                                  int* __restrict__ finished, int eos_id, int pad_id, int stop_on_eos,
                                                                  float temperature, int top_k, int use_top_p, float p_thr,
                                                                  const float* __restrict__ u, int* __restrict__ next,
                                                                  float* __restrict__ probs_out) {
  sample_body<false>(logits, ld, V, special, n_special, finished, eos_id, pad_id, stop_on_eos, temperature, top_k, use_top_p, p_thr,
                     u, next, probs_out, ScoresOut{});
}

__global__ void __launch_bounds__(SMP_THREADS) sample_scores_kernel(const __nv_bfloat16* __restrict__ logits, int64_t ld, int V,
                                                                    const int* __restrict__ special, int n_special,
                                                                    int* __restrict__ finished, int eos_id, int pad_id,
                                                                    int stop_on_eos, float temperature, int top_k, int use_top_p,
                                                                    float p_thr, const float* __restrict__ u, int* __restrict__ next,
                                                                    float* __restrict__ probs_out, ScoresOut so) {
  sample_body<true>(logits, ld, V, special, n_special, finished, eos_id, pad_id, stop_on_eos, temperature, top_k, use_top_p, p_thr,
                    u, next, probs_out, so);
}

// ---- logits processors (transformers 4.28 _get_logits_processor order: RepetitionPenaltyLogitsProcessor,
// NoRepeatNGramLogitsProcessor, MinLengthLogitsProcessor, MinNewTokensLengthLogitsProcessor) ----
// A row's history is HF's input_ids: the S padded prompt columns (left pads included) followed by its t generated tokens.
struct ProcHist {
  const int* prompt;                         // the row's padded prompt ids [S]
  const int* gen;                            // its generated tokens [t]
  int S;
  __device__ __forceinline__ int operator[](int i) const { return i < S ? prompt[i] : gen[i - S]; }
};

// The processor scalars; "off" is penalty 1, ngram 0, min_length 0, min_new 0.
struct ProcParams {
  float penalty;
  int ngram, min_length, min_new, eos;
};

// RepetitionPenaltyLogitsProcessor on one bf16 score: torch.where(s < 0, s * p, s / p) in fp32 opmath, rounded to bf16; the
// division is the IEEE one (the build's --use_fast_math would otherwise make it approximate).
__device__ __forceinline__ float rep_penalize(float s, float p) {
  return bf16_round(s < 0.f ? __fmul_rn(s, p) : __fdiv_rn(s, p));
}

// Set bits[h[j + n - 1]] for every n-gram h[j .. j + n - 1] of the L-token history whose first n - 1 tokens equal the last
// n - 1 tokens of the history (4.28 _get_ngrams / _get_generated_ngrams); nothing while L + 1 < n.  Positions strided over
// the CTA's threads.
__device__ __forceinline__ void ngram_bans(const ProcHist& h, int L, int n, int V, uint32_t* bits) {
  for (int j = threadIdx.x; j + n <= L; j += blockDim.x) {
    bool match = true;
    for (int q = 0; q < n - 1 && match; ++q) match = h[j + q] == h[L - n + 1 + q];
    if (match) {
      const int id = h[j + n - 1];
      if (id >= 0 && id < V) atomicOr(&bits[id >> 5], 1u << (id & 31));
    }
  }
}

__device__ __forceinline__ bool eos_banned(const ProcParams& p, int S, int t) {
  return S + t < p.min_length || t < p.min_new;
}

constexpr int LP_THREADS = 256;

// One CTA per decode row r, in place on the bf16 logits row.  Row r reads prompt row r / rows_per_prompt (the samples of a
// prompt share it) and its generated history hist[r, 0 .. hist_len[r]); with `append`, append[r] (the token picked at the
// previous step) is first appended there.  Phase 1: each distinct history id is penalised once (a V-bit shared bitmap; the
// thread whose atomicOr set the bit writes).  Phase 2: n-gram bans and phase 3: the EOS bans, both -inf.  Work per row is
// O(V / 32 + (S + t) * n), independent of V beyond clearing the bitmap.
__global__ void __launch_bounds__(LP_THREADS) logits_process_kernel(__nv_bfloat16* __restrict__ logits, int64_t ld, int V,
                                                                    const int* __restrict__ prompt, int64_t ld_prompt,
                                                                    const int* __restrict__ prompt_width, int rows_per_prompt,
                                                                    int* __restrict__ hist, int G, int* __restrict__ hist_len,
                                                                    const int* __restrict__ append, ProcParams p) {
  extern __shared__ uint32_t lp_bits[];                          // (V + 31) / 32 words
  __shared__ int s_t;
  griddep_launch();
  griddep_wait();
  const int r = blockIdx.x, tid = threadIdx.x;
  const int nw = (V + 31) >> 5;
  int* grow = hist + (int64_t)r * G;
  if (tid == 0) {
    int t = hist_len[r];
    if (append != nullptr && t < G) {
      grow[t] = append[r];
      hist_len[r] = ++t;
    }
    s_t = t;
  }
  for (int i = tid; i < nw; i += LP_THREADS) lp_bits[i] = 0u;
  __syncthreads();                                               // also publishes the appended token to the CTA
  const int S = *prompt_width, t = s_t, L = S + t;
  const ProcHist h{prompt + (int64_t)(r / rows_per_prompt) * ld_prompt, grow, S};
  __nv_bfloat16* row = logits + (int64_t)r * ld;
  if (p.penalty != 1.f) {
    for (int i = tid; i < L; i += LP_THREADS) {
      const int id = h[i];
      if (id < 0 || id >= V) continue;
      const uint32_t m = 1u << (id & 31);
      if (!(atomicOr(&lp_bits[id >> 5], m) & m)) row[id] = __float2bfloat16_rn(rep_penalize(__bfloat162float(row[id]), p.penalty));
    }
  }
  __syncthreads();
  const __nv_bfloat16 ninf = __ushort_as_bfloat16((unsigned short)0xFF80u);
  if (p.ngram > 0) {
    for (int j = tid; j + p.ngram <= L; j += LP_THREADS) {
      bool match = true;
      for (int q = 0; q < p.ngram - 1 && match; ++q) match = h[j + q] == h[L - p.ngram + 1 + q];
      if (match) {
        const int id = h[j + p.ngram - 1];
        if (id >= 0 && id < V) row[id] = ninf;
      }
    }
  }
  if (tid == 0 && p.eos >= 0 && p.eos < V && eos_banned(p, S, t)) row[p.eos] = ninf;
}

// ---- beam search (HF GenerationMixin.beam_search / BeamSearchScorer of transformers 4.28, the version the reference pins) ----
constexpr int BEAM_MAX = 8;                  // beams per prompt
constexpr int BT_THREADS = 512;
constexpr int BT_LIST = 2 * BEAM_MAX;        // candidates kept per thread: the 2K best overall are among each thread's 2K best

__device__ __forceinline__ uint32_t f32_order(float v) {          // monotone: larger float -> larger key; -inf lowest
  const uint32_t u = __float_as_uint(v);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ float f32_unorder(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// One CTA per prompt b.  Beam k's next-token scores are bf16(log_softmax(logits row (b, k))) + beam_score[b, k]: special ids
// -inf, the row max and sum in fp32 / fp64, each log-prob rounded once to bf16, then the fp32 add of HF.  The 2K best of the
// K * V scores by (score desc, flat index k * V + c asc) go to cand_* [B, 2K] in that order.  A score and its flat index
// make one 64-bit key, so every comparison is one integer compare and equal scores order by index.
// PROC (nv_beam_topk_processed): the logits processors of ProcParams act on each bf16 log-prob before the add, as 4.28's
// beam_search applies them to log_softmax's output.  Beam k of prompt b has the history prompt[b, 0 .. S) ++ hist[b * K + k,
// 0 .. t), t = prompt_state[b, 0] (nv_beam_select keeps hist in beam order); per beam, a "seen" and a "banned" V-bit bitmap
// are built in dynamic shared memory before the beam's scores are scanned.
struct BeamProc {
  const int* prompt;                         // [B, ld_prompt] padded prompt ids
  int64_t ld_prompt;
  const int* prompt_width;                   // device S
  const int* hist;                           // [B * K, G]
  int G;
  const int* prompt_state;                   // [B, 5]; field 0: tokens generated
  ProcParams p;
};

// TRIE (nv_beam_topk_trie, always with PROC): after the processors, every log-prob the trie does not allow at the beam's node
// becomes -inf, as 4.28's PrefixConstrainedLogitsProcessor does to log_softmax's output.  The node is found statelessly: one
// thread walks the beam's generated tokens hist[b * K + k, 0 .. t) from the root by the rule of nv_trie_mask (a node without
// children stays; a token that is not a child leads to the dead node n_nodes), so the walk follows the beam through every
// reorder nv_beam_select makes.  The allowed tokens (the node's children, or leaf_tok at a node without any) fill a third
// V-bit bitmap beside seen / banned.
struct BeamTrie {
  const int* node_ptr;                       // [n_nodes + 2]
  const int* child_tok;                      // [E], ascending per node
  const int* child_node;                     // [E]
  int n_nodes;
  int leaf_tok;
};

__device__ __forceinline__ int trie_walk(const BeamTrie& tr, const int* __restrict__ toks, int t) {
  int node = 0;
  for (int i = 0; i < t; ++i) {
    const int e0 = tr.node_ptr[node], e1 = tr.node_ptr[node + 1];
    if (e1 == e0) break;                                          // childless: the walk stays here for good
    const int tok = toks[i];
    int lo = e0, hi = e1;                                         // first edge with child_tok >= tok
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (tr.child_tok[mid] < tok) lo = mid + 1;
      else hi = mid;
    }
    node = (lo < e1 && tr.child_tok[lo] == tok) ? tr.child_node[lo] : tr.n_nodes;
  }
  return node;
}

// SCORES (nv_beam_topk*_scores): each beam's processed bf16 log-probs before the beam-score add (4.28's
// next_token_scores_processed; special ids -inf) also go to so.row(b, b * K + k), the plane of step t = prompt_state[b, 0].
// GROUP (nv_beam_topk_group*, diverse beam search): the CTA scans only the Kg = K / n_groups beams k0 + [0, Kg) of group g
// (k0 = g * Kg) and writes that group's 2Kg best to cand_* [B, 2Kg], the parent local to the group.  Before the processors, each
// bf16 log-prob of token c becomes bf16(lp - fp32(penalty) * freq[c]) in fp32, 4.28's HammingDiversityLogitsProcessor
// (scores -= diversity_penalty * bincount): freq counts c among next_ids of rows b * K + [0, k0), the tokens the earlier groups'
// selects of this step have already written there (at most BEAM_MAX - 1 of them).
struct BeamGroup {
  const int* next_ids;                       // [B * K]
  float penalty;                             // diversity_penalty
  int g, Kg;
};

template <bool PROC, bool TRIE = false, bool SCORES = false, bool GROUP = false>
__device__ __forceinline__ void beam_topk_body(const __nv_bfloat16* __restrict__ logits, int64_t ld_prompt, int64_t ld_beam, int V,
                                               const int* __restrict__ special, int n_special, const float* __restrict__ beam_score,
                                                int K, float* __restrict__ cand_score, int* __restrict__ cand_tok,
                                               int* __restrict__ cand_par, const BeamProc& bp, const BeamTrie& tr = BeamTrie{},
                                               const ScoresOut& so = ScoresOut{}, const BeamGroup& gr = BeamGroup{}) {
  static_assert(PROC || !TRIE, "the trie mask runs inside the processed scan");
  static_assert(!(GROUP && TRIE), "group beams have no trie form");
  __shared__ int s_special[MAX_SPECIAL];
  __shared__ float s_m[BEAM_MAX], s_ls[BEAM_MAX], s_bs[BEAM_MAX];
  __shared__ float redf[32];
  __shared__ double redd[32];
  __shared__ unsigned long long redk[32];
  griddep_launch();
  griddep_wait();
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  constexpr int NW = BT_THREADS / 32;
  const int ns = n_special;
  const int nb = GROUP ? gr.Kg : K;                              // beams scanned, from beam k0 of the prompt
  const int k0 = GROUP ? gr.g * gr.Kg : 0;
  if (tid < ns) s_special[tid] = special[tid];
  if (tid < nb) s_bs[tid] = beam_score[b * K + k0 + tid];
  int* s_div = nullptr;                                          // GROUP: the earlier groups' tokens of this step
  if constexpr (GROUP) {
    __shared__ int s_div_tok[BEAM_MAX];
    s_div = s_div_tok;
    if (tid < k0) s_div[tid] = gr.next_ids[b * K + tid];
  }
  __syncthreads();
  auto is_special = [&](int c) {
    bool sp = false;
    for (int s = 0; s < ns; ++s) sp |= (s_special[s] == c);
    return sp;
  };
  auto diversity = [&](float lp, int c) {                        // the Hamming penalty on a bf16 log-prob
    if constexpr (GROUP) {
      int f = 0;
      for (int i = 0; i < k0; ++i) f += (s_div[i] == c);
      if (f) lp = bf16_round(__fsub_rn(lp, __fmul_rn(gr.penalty, (float)f)));
    }
    return lp;
  };
  for (int k = 0; k < nb; ++k) {
    const __nv_bfloat16* row = logits + (int64_t)b * ld_prompt + (int64_t)(k0 + k) * ld_beam;
    float mx = -INFINITY;
    for (int c = tid; c < V; c += BT_THREADS)
      if (!is_special(c)) mx = fmaxf(mx, __bfloat162float(row[c]));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (lane == 0) redf[w] = mx;
    __syncthreads();
    mx = lane < NW ? redf[lane] : -INFINITY;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    double s = 0.0;                                              // fp64: the fp32 sum of torch up to its own rounding
    for (int c = tid; c < V; c += BT_THREADS)
      if (!is_special(c)) s += exp((double)(__bfloat162float(row[c]) - mx));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) redd[w] = s;
    __syncthreads();
    s = lane < NW ? redd[lane] : 0.0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (tid == 0) {
      s_m[k] = mx;
      s_ls[k] = (float)log(s);
    }
    __syncthreads();
  }
  unsigned long long L[BT_LIST];                                 // this thread's best keys, descending; 0 = empty
#pragma unroll
  for (int i = 0; i < BT_LIST; ++i) L[i] = 0ull;
  for (int k = 0; k < nb; ++k) {
    const __nv_bfloat16* row = logits + (int64_t)b * ld_prompt + (int64_t)(k0 + k) * ld_beam;
    const float m = s_m[k], ls = s_ls[k], bs = s_bs[k];
    __nv_bfloat16* srow = nullptr;
    if constexpr (SCORES) srow = so.row(b, b * K + k0 + k);
    uint32_t* seen = nullptr;
    uint32_t* banned = nullptr;
    uint32_t* allowed = nullptr;
    if constexpr (PROC) {
      extern __shared__ uint32_t bt_bits[];                      // seen | banned (| allowed), (V + 31) / 32 words each
      const int nw = (V + 31) >> 5;
      constexpr int NMAPS = TRIE ? 3 : 2;
      seen = bt_bits;
      banned = bt_bits + nw;
      __syncthreads();                                           // the previous beam's scan is done with the bitmaps
      for (int i = tid; i < NMAPS * nw; i += BT_THREADS) bt_bits[i] = 0u;
      __syncthreads();
      const int S = *bp.prompt_width, t = bp.prompt_state[b * 5], L = S + t;
      const ProcHist h{bp.prompt + (int64_t)b * bp.ld_prompt, bp.hist + (int64_t)(b * K + k0 + k) * bp.G, S};
      __shared__ int s_node;                                     // TRIE: the beam's node
      if constexpr (TRIE)
        if (tid == 0) s_node = trie_walk(tr, bp.hist + (int64_t)(b * K + k) * bp.G, t);
      if (bp.p.penalty != 1.f)
        for (int i = tid; i < L; i += BT_THREADS) {
          const int id = h[i];
          if (id >= 0 && id < V) atomicOr(&seen[id >> 5], 1u << (id & 31));
        }
      if (bp.p.ngram > 0) ngram_bans(h, L, bp.p.ngram, V, banned);
      if (tid == 0 && bp.p.eos >= 0 && bp.p.eos < V && eos_banned(bp.p, S, t)) atomicOr(&banned[bp.p.eos >> 5], 1u << (bp.p.eos & 31));
      __syncthreads();
      if constexpr (TRIE) {
        allowed = bt_bits + 2 * nw;
        const int node = s_node, e0 = tr.node_ptr[node], e1 = tr.node_ptr[node + 1];
        if (e1 == e0) {
          if (tid == 0) atomicOr(&allowed[tr.leaf_tok >> 5], 1u << (tr.leaf_tok & 31));
        } else {
          for (int e = e0 + tid; e < e1; e += BT_THREADS) {        // fan-outs of any size: looped, not capped
            const int c = tr.child_tok[e];
            if (c >= 0 && c < V) atomicOr(&allowed[c >> 5], 1u << (c & 31));
          }
        }
        __syncthreads();
      }
    }
    for (int c = tid; c < V; c += BT_THREADS) {
      float sc = -INFINITY;
      if constexpr (PROC) {
        if (!is_special(c)) {
          float lp = diversity(bf16_round((__bfloat162float(row[c]) - m) - ls), c);
          const uint32_t bit = 1u << (c & 31);
          if (seen[c >> 5] & bit) lp = rep_penalize(lp, bp.p.penalty);
          if (banned[c >> 5] & bit) lp = -INFINITY;
          if constexpr (TRIE)
            if (!(allowed[c >> 5] & bit)) lp = -INFINITY;
          if constexpr (SCORES) srow[c] = __float2bfloat16_rn(lp);
          sc = lp + bs;
        } else if constexpr (SCORES) {
          srow[c] = __float2bfloat16_rn(-INFINITY);
        }
      } else {
        if constexpr (SCORES) {
          if (!is_special(c)) {
            const float lp = diversity(bf16_round((__bfloat162float(row[c]) - m) - ls), c);
            srow[c] = __float2bfloat16_rn(lp);
            sc = lp + bs;
          } else {
            srow[c] = __float2bfloat16_rn(-INFINITY);
          }
        } else {
          if (!is_special(c)) sc = diversity(bf16_round((__bfloat162float(row[c]) - m) - ls), c) + bs;
        }
      }
      if (sc != sc) sc = -INFINITY;
      const unsigned long long key =
          ((unsigned long long)f32_order(sc) << 32) | (unsigned long long)(0xffffffffu - (uint32_t)(k * V + c));
      if (key > L[BT_LIST - 1]) {
        L[BT_LIST - 1] = key;
#pragma unroll
        for (int i = BT_LIST - 1; i > 0; --i)
          if (L[i] > L[i - 1]) {
            const unsigned long long t = L[i]; L[i] = L[i - 1]; L[i - 1] = t;
          }
      }
    }
  }
  // 2K rounds: the CTA-wide largest head wins and its owner pops it
  for (int r = 0; r < 2 * nb; ++r) {
    unsigned long long best = L[0];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long x = __shfl_xor_sync(0xffffffffu, best, o);
      best = x > best ? x : best;
    }
    if (lane == 0) redk[w] = best;
    __syncthreads();
    best = lane < NW ? redk[lane] : 0ull;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long x = __shfl_xor_sync(0xffffffffu, best, o);
      best = x > best ? x : best;
    }
    if (L[0] == best) {
#pragma unroll
      for (int i = 0; i < BT_LIST - 1; ++i) L[i] = L[i + 1];
      L[BT_LIST - 1] = 0ull;
    }
    if (tid == 0) {
      const uint32_t flat = 0xffffffffu - (uint32_t)(best & 0xffffffffull);
      cand_score[b * 2 * nb + r] = f32_unorder((uint32_t)(best >> 32));
      cand_tok[b * 2 * nb + r] = (int)(flat % (uint32_t)V);
      cand_par[b * 2 * nb + r] = (int)(flat / (uint32_t)V);
    }
    __syncthreads();                                             // redk is reused by the next round
  }
}

__global__ void __launch_bounds__(BT_THREADS) beam_topk_kernel(const __nv_bfloat16* __restrict__ logits, int64_t ld_prompt,
                                                               int64_t ld_beam, int V, const int* __restrict__ special,
                                                               int n_special, const float* __restrict__ beam_score, int K,
                                                               float* __restrict__ cand_score, int* __restrict__ cand_tok,
                                                               int* __restrict__ cand_par) {
  beam_topk_body<false>(logits, ld_prompt, ld_beam, V, special, n_special, beam_score, K, cand_score, cand_tok, cand_par, BeamProc{});
}

// one CTA per SM is what B <= 132 prompts use anyway; the bound lets the bitmap tests stay in registers beside the 2K-key list
__global__ void __launch_bounds__(BT_THREADS, 1) beam_topk_proc_kernel(const __nv_bfloat16* __restrict__ logits, int64_t ld_prompt,
                                                                       int64_t ld_beam, int V, const int* __restrict__ special,
                                                                       int n_special, const float* __restrict__ beam_score, int K,
                                                                       float* __restrict__ cand_score, int* __restrict__ cand_tok,
                                                                       int* __restrict__ cand_par, BeamProc bp) {
  beam_topk_body<true>(logits, ld_prompt, ld_beam, V, special, n_special, beam_score, K, cand_score, cand_tok, cand_par, bp);
}

// the bound as for beam_topk_proc_kernel; the walk and the third bitmap add no per-thread state to the scan
__global__ void __launch_bounds__(BT_THREADS, 1) beam_topk_trie_kernel(const __nv_bfloat16* __restrict__ logits, int64_t ld_prompt,
                                                                       int64_t ld_beam, int V, const int* __restrict__ special,
                                                                       int n_special, const float* __restrict__ beam_score, int K,
                                                                       float* __restrict__ cand_score, int* __restrict__ cand_tok,
                                                                       int* __restrict__ cand_par, BeamProc bp, BeamTrie tr) {
  beam_topk_body<true, true>(logits, ld_prompt, ld_beam, V, special, n_special, beam_score, K, cand_score, cand_tok, cand_par, bp, tr);
}

// the three beam top-k kernels with the SCORES output (nv_beam_topk*_scores); bounds as above
__global__ void __launch_bounds__(BT_THREADS) beam_topk_scores_kernel(const __nv_bfloat16* __restrict__ logits, int64_t ld_prompt,
                                                                      int64_t ld_beam, int V, const int* __restrict__ special,
                                                                      int n_special, const float* __restrict__ beam_score, int K,
                                                                      float* __restrict__ cand_score, int* __restrict__ cand_tok,
                                                                      int* __restrict__ cand_par, ScoresOut so) {
  beam_topk_body<false, false, true>(logits, ld_prompt, ld_beam, V, special, n_special, beam_score, K, cand_score, cand_tok, cand_par,
                                     BeamProc{}, BeamTrie{}, so);
}

__global__ void __launch_bounds__(BT_THREADS, 1) beam_topk_proc_scores_kernel(const __nv_bfloat16* __restrict__ logits,
                                                                              int64_t ld_prompt, int64_t ld_beam, int V,
                                                                              const int* __restrict__ special, int n_special,
                                                                              const float* __restrict__ beam_score, int K,
                                                                              float* __restrict__ cand_score, int* __restrict__ cand_tok,
                                                                              int* __restrict__ cand_par, BeamProc bp, ScoresOut so) {
  beam_topk_body<true, false, true>(logits, ld_prompt, ld_beam, V, special, n_special, beam_score, K, cand_score, cand_tok, cand_par,
                                    bp, BeamTrie{}, so);
}

__global__ void __launch_bounds__(BT_THREADS, 1) beam_topk_trie_scores_kernel(const __nv_bfloat16* __restrict__ logits,
                                                                              int64_t ld_prompt, int64_t ld_beam, int V,
                                                                              const int* __restrict__ special, int n_special,
                                                                              const float* __restrict__ beam_score, int K,
                                                                              float* __restrict__ cand_score, int* __restrict__ cand_tok,
                                                                              int* __restrict__ cand_par, BeamProc bp, BeamTrie tr,
                                                                              ScoresOut so) {
  beam_topk_body<true, true, true>(logits, ld_prompt, ld_beam, V, special, n_special, beam_score, K, cand_score, cand_tok, cand_par,
                                   bp, tr, so);
}

// the group top-k kernels (nv_beam_topk_group[_processed][_scores]); bounds as above
__global__ void __launch_bounds__(BT_THREADS) beam_topk_group_kernel(const __nv_bfloat16* __restrict__ logits, int64_t ld_prompt,
                                                                     int64_t ld_beam, int V, const int* __restrict__ special,
                                                                     int n_special, const float* __restrict__ beam_score, int K,
                                                                     float* __restrict__ cand_score, int* __restrict__ cand_tok,
                                                                     int* __restrict__ cand_par, BeamGroup gr) {
  beam_topk_body<false, false, false, true>(logits, ld_prompt, ld_beam, V, special, n_special, beam_score, K, cand_score, cand_tok,
                                            cand_par, BeamProc{}, BeamTrie{}, ScoresOut{}, gr);
}

__global__ void __launch_bounds__(BT_THREADS, 1) beam_topk_group_proc_kernel(const __nv_bfloat16* __restrict__ logits,
                                                                             int64_t ld_prompt, int64_t ld_beam, int V,
                                                                             const int* __restrict__ special, int n_special,
                                                                             const float* __restrict__ beam_score, int K,
                                                                             float* __restrict__ cand_score, int* __restrict__ cand_tok,
                                                                             int* __restrict__ cand_par, BeamProc bp, BeamGroup gr) {
  beam_topk_body<true, false, false, true>(logits, ld_prompt, ld_beam, V, special, n_special, beam_score, K, cand_score, cand_tok,
                                           cand_par, bp, BeamTrie{}, ScoresOut{}, gr);
}

__global__ void __launch_bounds__(BT_THREADS) beam_topk_group_scores_kernel(const __nv_bfloat16* __restrict__ logits, int64_t ld_prompt,
                                                                            int64_t ld_beam, int V, const int* __restrict__ special,
                                                                            int n_special, const float* __restrict__ beam_score, int K,
                                                                            float* __restrict__ cand_score, int* __restrict__ cand_tok,
                                                                            int* __restrict__ cand_par, ScoresOut so, BeamGroup gr) {
  beam_topk_body<false, false, true, true>(logits, ld_prompt, ld_beam, V, special, n_special, beam_score, K, cand_score, cand_tok,
                                           cand_par, BeamProc{}, BeamTrie{}, so, gr);
}

__global__ void __launch_bounds__(BT_THREADS, 1) beam_topk_group_proc_scores_kernel(const __nv_bfloat16* __restrict__ logits,
                                                                                    int64_t ld_prompt, int64_t ld_beam, int V,
                                                                                    const int* __restrict__ special, int n_special,
                                                                                    const float* __restrict__ beam_score, int K,
                                                                                    float* __restrict__ cand_score,
                                                                                    int* __restrict__ cand_tok, int* __restrict__ cand_par,
                                                                                    BeamProc bp, ScoresOut so, BeamGroup gr) {
  beam_topk_body<true, false, true, true>(logits, ld_prompt, ld_beam, V, special, n_special, beam_score, K, cand_score, cand_tok,
                                          cand_par, bp, BeamTrie{}, so, gr);
}

// ---- answer scoring (nv_trie_score): every answer of a trie teacher-forced over one tree-masked forward ----
constexpr int TS_THREADS = 512;
constexpr int TF_THREADS = 256;

// One CTA per logits row: the row's max and log-sum over the non-special ids, as beam_topk_body computes them (fp32 max, fp64
// sum of exp(x - m), log rounded to fp32), into stats[row] = (m, ls).
__global__ void __launch_bounds__(TS_THREADS) trie_row_stats_kernel(const __nv_bfloat16* __restrict__ logits, int64_t ld, int V,
                                                                    const int* __restrict__ special, int n_special,
                                                                    float* __restrict__ stats) {
  __shared__ int s_special[MAX_SPECIAL];
  __shared__ float redf[32];
  __shared__ double redd[32];
  griddep_launch();
  griddep_wait();
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  constexpr int NW = TS_THREADS / 32;
  const int ns = n_special;
  if (tid < ns) s_special[tid] = special[tid];
  __syncthreads();
  auto is_special = [&](int c) {
    bool sp = false;
    for (int s = 0; s < ns; ++s) sp |= (s_special[s] == c);
    return sp;
  };
  const __nv_bfloat16* row = logits + (int64_t)blockIdx.x * ld;
  float mx = -INFINITY;
  for (int c = tid; c < V; c += TS_THREADS)
    if (!is_special(c)) mx = fmaxf(mx, __bfloat162float(row[c]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if (lane == 0) redf[w] = mx;
  __syncthreads();
  mx = lane < NW ? redf[lane] : -INFINITY;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  double s = 0.0;
#pragma unroll 1                                                  // unrolled, ptxas spills a register around exp
  for (int c = tid; c < V; c += TS_THREADS)
    if (!is_special(c)) s += exp((double)(__bfloat162float(row[c]) - mx));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) redd[w] = s;
  __syncthreads();
  s = lane < NW ? redd[lane] : 0.0;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (tid == 0) {
    stats[2 * blockIdx.x] = mx;
    stats[2 * blockIdx.x + 1] = (float)log(s);
  }
}

// One CTA per prompt, one thread per answer: the answer's path folded root to leaf in fp32, each term the bf16 log-prob of
// beam_topk_body (special ids -inf, NaN -> -inf).
__global__ void __launch_bounds__(TF_THREADS) trie_fold_kernel(const __nv_bfloat16* __restrict__ logits, int64_t ld, int V,
                                                               const int* __restrict__ special, int n_special,
                                                               const int* __restrict__ tok, const int* __restrict__ path_off,
                                                               const int* __restrict__ path_rows, int eos,
                                                               const float* __restrict__ stats, float* __restrict__ logprob,
                                                               int R, int A) {
  __shared__ int s_special[MAX_SPECIAL];
  griddep_launch();
  griddep_wait();
  const int b = blockIdx.x, tid = threadIdx.x, ns = n_special;
  if (tid < ns) s_special[tid] = special[tid];
  __syncthreads();
  const int64_t row0 = (int64_t)b * R;
  auto lp = [&](int r, int c) {                                   // log-prob of token c at source row r of prompt b
    bool sp = false;
    for (int i = 0; i < ns; ++i) sp |= (s_special[i] == c);
    if (sp) return -INFINITY;
    const float m = stats[2 * (row0 + r)], ls = stats[2 * (row0 + r) + 1];
    const float v = bf16_round((__bfloat162float(logits[(row0 + r) * ld + c]) - m) - ls);
    return v != v ? -INFINITY : v;
  };
  for (int a = tid; a < A; a += TF_THREADS) {
    float s = 0.f;
    int src = 0;                                                  // row 0: the prompt's last row
    for (int p = path_off[a]; p < path_off[a + 1]; ++p) {
      const int node = path_rows[p];
      s = lp(src, tok[node]) + s;
      src = node + 1;
    }
    s = lp(src, eos) + s;
    logprob[(int64_t)b * A + a] = s;
  }
}

// prompt_state [B, BS_FIELDS] of nv_beam_select
constexpr int BS_STEP = 0, BS_PLEN = 1, BS_COUNT = 2, BS_SEQ = 3, BS_DONE = 4, BS_FIELDS = 5;
constexpr int BS_THREADS = 128, BS_CHUNK = 256;

// One CTA per prompt: BeamSearchScorer.process + BeamHypotheses.add / is_done of transformers 4.28 over the 2K candidates of
// nv_beam_topk, then the reorder of the running beams (input_ids[beam_idx] and _reorder_cache) as gathers of the generated-
// token history and of the KV source table by parent.  t = prompt_state[b, BS_STEP] tokens have been generated; norm[t] is
// (S + t) ** length_penalty as the host's Python floats compute it (S padded prompt columns: hyp.shape[-1] in 4.28), so the fp64
// hypothesis scores sum_logprobs / norm[t] are 4.28's to the bit.  hyp_score [B, K + 1] holds the K kept scores and the worst kept score, hyp_meta [B, K, 2] (generated
// length, insertion number: the later of equal scores wins in finalize), hyp_tok [B, K, G] their generated tokens.
// SCORES (nv_beam_select_scores): 4.28's beam_indices as well.  par_hist [R, G] holds each running beam's rows (b * K + parent)
// of the steps so far and is gathered by parent like hist; a hypothesis added at step t gets its parent's rows and then that
// parent's row at t in hyp_par [B, K, G]; done_step[b] = t + 1 at the step prompt b becomes done.
struct BeamTrace {
  int* par_hist;
  int* hyp_par;
  int* done_step;
};

// GROUP (nv_beam_select_group*, diverse beam search): process over group g's 2Kg candidates of nv_beam_topk_group (cand_*
// [B, 2Kg], parents local to the group) with group_size Kg, against the prompt's one set of K hypotheses (4.28's
// BeamSearchScorer with num_beam_groups: EOS at rank >= Kg is skipped, Kg survivors).  It reads the current done flag, so a
// prompt an earlier group finished in this step pads, and it reorders and writes only the group's rows b * K + k0 + [0, Kg)
// (k0 = g * Kg; parents, par_hist and hyp_par in global rows).  Only the last group's launch (``last``) advances BS_STEP, so
// the scans of later groups still see step t.
struct BeamSelGroup {
  int g, Kg, last;
};

template <bool SCORES, bool GROUP = false>
__device__ __forceinline__ void beam_select_body(const float* __restrict__ cand_score, const int* __restrict__ cand_tok,
                                                 const int* __restrict__ cand_par, float* __restrict__ beam_score,
                                                 int* __restrict__ hist, int* __restrict__ src, double* __restrict__ hyp_score,
                                                 int* __restrict__ hyp_meta, int* __restrict__ hyp_tok, int* __restrict__ pstate,
                                                 int* __restrict__ next_ids, int* __restrict__ lens, const double* __restrict__ norm,
                                                 int K, int G, int eos_id, int pad_id, int early_stopping, const BeamTrace& tr,
                                                 const BeamSelGroup& gr = BeamSelGroup{}) {
  __shared__ int s_tok[BEAM_MAX], s_par[BEAM_MAX];
  __shared__ float s_sc[BEAM_MAX];
  __shared__ int s_op_slot[BEAM_MAX], s_op_par[BEAM_MAX], s_nops;
  __shared__ int s_h[BEAM_MAX][BS_CHUNK], s_s[BEAM_MAX][BS_CHUNK];
  griddep_launch();
  griddep_wait();
  const int b = blockIdx.x, tid = threadIdx.x;
  int* ps = pstate + b * BS_FIELDS;
  const int t = ps[BS_STEP];
  if (t >= G) return;                                            // the host sizes G to the call's max_new_tokens
  const int nb = GROUP ? gr.Kg : K;                              // beams selected: rows b * K + k0 + [0, nb)
  const int k0 = GROUP ? gr.g * gr.Kg : 0;
  if (tid == 0) {
    int nops = 0;
    if (ps[BS_DONE]) {                                           // a done prompt's beams emit pad with score 0
      for (int j = 0; j < nb; ++j) { s_tok[j] = pad_id; s_par[j] = j; s_sc[j] = 0.f; }
    } else {
      double* hs = hyp_score + b * (K + 1);
      int* hm = hyp_meta + b * K * 2;
      double worst = hs[K];
      int cnt = ps[BS_COUNT], seq = ps[BS_SEQ];
      const double nt = norm[t];
      int j = 0;
      for (int rank = 0; rank < 2 * nb; ++rank) {
        const int tok = cand_tok[b * 2 * nb + rank], par = cand_par[b * 2 * nb + rank];
        const float sc = cand_score[b * 2 * nb + rank];
        if (tok == eos_id) {
          if (rank >= nb) continue;                              // EOS below the top K is not a hypothesis
          const double score = (double)sc / nt;
          if (cnt < K || score > worst) {
            int slot;
            if (cnt < K) {
              slot = cnt++;
              worst = fmin(score, worst);
            } else {                                             // drop the lowest (score, insertion) and take its slot
              slot = 0;
              for (int i = 1; i < K; ++i)
                if (hs[i] < hs[slot] || (hs[i] == hs[slot] && hm[2 * i + 1] < hm[2 * slot + 1])) slot = i;
            }
            hs[slot] = score;
            hm[2 * slot] = t;
            hm[2 * slot + 1] = seq++;
            if (cnt == K) {
              worst = hs[0];
              for (int i = 1; i < K; ++i) worst = fmin(worst, hs[i]);
            }
            s_op_slot[nops] = slot;
            s_op_par[nops] = par;
            ++nops;
          }
        } else {
          s_tok[j] = tok; s_par[j] = par; s_sc[j] = sc;
          ++j;
        }
        if (j == nb) break;
      }
      int done = 0;
      if (cnt >= K) done = early_stopping ? 1 : (worst >= (double)cand_score[b * 2 * nb] / nt);
      if constexpr (SCORES)
        if (done) tr.done_step[b] = t + 1;
      hs[K] = worst;
      ps[BS_COUNT] = cnt;
      ps[BS_SEQ] = seq;
      ps[BS_DONE] = done;
    }
    s_nops = nops;
  }
  __syncthreads();
  for (int o = 0; o < s_nops; ++o) {                             // in order: a later hypothesis may take an earlier one's slot
    const int* from = hist + (int64_t)(b * K + k0 + s_op_par[o]) * G;
    int* to = hyp_tok + (int64_t)(b * K + s_op_slot[o]) * G;
    for (int i = tid; i < t; i += BS_THREADS) to[i] = from[i];
    if constexpr (SCORES) {
      const int* pf = tr.par_hist + (int64_t)(b * K + k0 + s_op_par[o]) * G;
      int* pt = tr.hyp_par + (int64_t)(b * K + s_op_slot[o]) * G;
      for (int i = tid; i < t; i += BS_THREADS) pt[i] = pf[i];
      if (tid == 0) pt[t] = b * K + k0 + s_op_par[o];
    }
  }
  for (int c0 = 0; c0 < t; c0 += BS_CHUNK) {                     // rows of the new beams = rows of their parents
    const int n = min(BS_CHUNK, t - c0);
    for (int idx = tid; idx < nb * BS_CHUNK; idx += BS_THREADS) {
      const int j = idx / BS_CHUNK, i = idx % BS_CHUNK;
      if (i < n) {
        const int64_t from = (int64_t)(b * K + k0 + s_par[j]) * G + c0 + i;
        s_h[j][i] = hist[from];
        s_s[j][i] = src[from];
      }
    }
    __syncthreads();
    for (int idx = tid; idx < nb * BS_CHUNK; idx += BS_THREADS) {
      const int j = idx / BS_CHUNK, i = idx % BS_CHUNK;
      if (i < n) {
        const int64_t to = (int64_t)(b * K + k0 + j) * G + c0 + i;
        hist[to] = s_h[j][i];
        src[to] = s_s[j][i];
      }
    }
    __syncthreads();
  }
  if constexpr (SCORES) {
    for (int c0 = 0; c0 < t; c0 += BS_CHUNK) {                   // par_hist by parent, through s_h
      const int n = min(BS_CHUNK, t - c0);
      for (int idx = tid; idx < nb * BS_CHUNK; idx += BS_THREADS) {
        const int j = idx / BS_CHUNK, i = idx % BS_CHUNK;
        if (i < n) s_h[j][i] = tr.par_hist[(int64_t)(b * K + k0 + s_par[j]) * G + c0 + i];
      }
      __syncthreads();
      for (int idx = tid; idx < nb * BS_CHUNK; idx += BS_THREADS) {
        const int j = idx / BS_CHUNK, i = idx % BS_CHUNK;
        if (i < n) tr.par_hist[(int64_t)(b * K + k0 + j) * G + c0 + i] = s_h[j][i];
      }
      __syncthreads();
    }
  }
  if (tid < nb) {
    const int r = b * K + k0 + tid;
    if constexpr (SCORES) tr.par_hist[(int64_t)r * G + t] = b * K + k0 + s_par[tid];
    hist[(int64_t)r * G + t] = s_tok[tid];
    src[(int64_t)r * G + t] = r;                                 // the next step writes generated key t of row r at (r, t)
    next_ids[r] = s_tok[tid];
    lens[r] = ps[BS_PLEN] + t;
    beam_score[r] = s_sc[tid];
  }
  __syncthreads();
  if (tid == 0 && (!GROUP || gr.last)) ps[BS_STEP] = t + 1;
}

__global__ void __launch_bounds__(BS_THREADS) beam_select_kernel(const float* __restrict__ cand_score, const int* __restrict__ cand_tok,
                                                                 const int* __restrict__ cand_par, float* __restrict__ beam_score,
                                                                 int* __restrict__ hist, int* __restrict__ src,
                                                                 double* __restrict__ hyp_score, int* __restrict__ hyp_meta,
                                                                 int* __restrict__ hyp_tok, int* __restrict__ pstate,
                                                                 int* __restrict__ next_ids, int* __restrict__ lens,
                                                                 const double* __restrict__ norm, int K, int G, int eos_id, int pad_id,
                                                                 int early_stopping) {
  beam_select_body<false>(cand_score, cand_tok, cand_par, beam_score, hist, src, hyp_score, hyp_meta, hyp_tok, pstate, next_ids, lens,
                          norm, K, G, eos_id, pad_id, early_stopping, BeamTrace{});
}

__global__ void __launch_bounds__(BS_THREADS) beam_select_scores_kernel(const float* __restrict__ cand_score,
                                                                        const int* __restrict__ cand_tok, const int* __restrict__ cand_par,
                                                                        float* __restrict__ beam_score, int* __restrict__ hist,
                                                                        int* __restrict__ src, double* __restrict__ hyp_score,
                                                                        int* __restrict__ hyp_meta, int* __restrict__ hyp_tok,
                                                                        int* __restrict__ pstate, int* __restrict__ next_ids,
                                                                        int* __restrict__ lens, const double* __restrict__ norm, int K,
                                                                        int G, int eos_id, int pad_id, int early_stopping, BeamTrace tr) {
  beam_select_body<true>(cand_score, cand_tok, cand_par, beam_score, hist, src, hyp_score, hyp_meta, hyp_tok, pstate, next_ids, lens,
                         norm, K, G, eos_id, pad_id, early_stopping, tr);
}

__global__ void __launch_bounds__(BS_THREADS, 1) beam_select_group_kernel(const float* __restrict__ cand_score,
                                                                       const int* __restrict__ cand_tok, const int* __restrict__ cand_par,
                                                                       float* __restrict__ beam_score, int* __restrict__ hist,
                                                                       int* __restrict__ src, double* __restrict__ hyp_score,
                                                                       int* __restrict__ hyp_meta, int* __restrict__ hyp_tok,
                                                                       int* __restrict__ pstate, int* __restrict__ next_ids,
                                                                       int* __restrict__ lens, const double* __restrict__ norm, int K,
                                                                       int G, int eos_id, int pad_id, int early_stopping, BeamSelGroup gr) {
  beam_select_body<false, true>(cand_score, cand_tok, cand_par, beam_score, hist, src, hyp_score, hyp_meta, hyp_tok, pstate, next_ids,
                                lens, norm, K, G, eos_id, pad_id, early_stopping, BeamTrace{}, gr);
}

__global__ void __launch_bounds__(BS_THREADS, 1) beam_select_group_scores_kernel(const float* __restrict__ cand_score,
                                                                              const int* __restrict__ cand_tok,
                                                                              const int* __restrict__ cand_par, float* __restrict__ beam_score,
                                                                              int* __restrict__ hist, int* __restrict__ src,
                                                                              double* __restrict__ hyp_score, int* __restrict__ hyp_meta,
                                                                              int* __restrict__ hyp_tok, int* __restrict__ pstate,
                                                                              int* __restrict__ next_ids, int* __restrict__ lens,
                                                                              const double* __restrict__ norm, int K, int G, int eos_id,
                                                                              int pad_id, int early_stopping, BeamTrace tr,
                                                                              BeamSelGroup gr) {
  beam_select_body<true, true>(cand_score, cand_tok, cand_par, beam_score, hist, src, hyp_score, hyp_meta, hyp_tok, pstate, next_ids,
                               lens, norm, K, G, eos_id, pad_id, early_stopping, tr, gr);
}

// ---- contrastive search (GenerationMixin.contrastive_search / _ranking_fast of transformers 4.28) ----
// A step: the K candidates of prompt b (the K most probable tokens) run as decode rows b * K + j over the prompt cache, each is
// scored bf16(bf16((1 - a) p_j) - bf16(a pen_j)) with pen_j = max_i bf16(c^_i . h^_j) over the normalised context rows of the
// prompt, and the best one's token, K/V and hidden state are kept.  x^ = bf16(x / bf16(||x||)) (4.28's bf16 tensor ops: a norm
// summed in fp32 and rounded, an fp32 division rounded).  --use_fast_math makes '/' and sqrtf approximate, hence the _rn forms.
constexpr int CT_KMAX = 64;                  // candidates per prompt
constexpr int CT_THREADS = 1024;             // nv_contrastive_topk: one CTA per prompt (the smp_* helpers assume 32 warps)
constexpr int CR_SPLIT = 16;                 // nv_contrastive_rank: CTAs per prompt over its context rows
constexpr int CR_CHUNK = 8;                  // candidates staged in shared memory per pass over the rows
constexpr int CR_THREADS = 256;
constexpr int CS_THREADS = 128;

// x^ of a D-element bf16 row (D % 8 == 0) by one warp; `out` may be shared or global memory
__device__ __forceinline__ void ct_normalize_row(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ out, int D, int lane) {
  float ss = 0.f;
  for (int c = lane * 8; c < D; c += 256) {
    float f[8];
    unpack8d(*reinterpret_cast<const uint4*>(x + c), f);
#pragma unroll
    for (int i = 0; i < 8; ++i) ss = __fmaf_rn(f[i], f[i], ss);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  const float nrm = bf16_round(__fsqrt_rn(ss));
  for (int c = lane * 8; c < D; c += 256) {
    float f[8];
    unpack8d(*reinterpret_cast<const uint4*>(x + c), f);
    uint4 o;
    o.x = pack_bf16x2(__fdiv_rn(f[0], nrm), __fdiv_rn(f[1], nrm));
    o.y = pack_bf16x2(__fdiv_rn(f[2], nrm), __fdiv_rn(f[3], nrm));
    o.z = pack_bf16x2(__fdiv_rn(f[4], nrm), __fdiv_rn(f[5], nrm));
    o.w = pack_bf16x2(__fdiv_rn(f[6], nrm), __fdiv_rn(f[7], nrm));
    *reinterpret_cast<uint4*>(out + c) = o;
  }
}

// exp(x) in fp64 for x <= 0 (or -inf), within 2e-16 relative: exp(x) = 2^k exp(r), |r| <= ln2 / 2, Taylor to degree 12.  The
// library's exp calls an out-of-line slow path that spills at 1024 threads.
__device__ __forceinline__ double ct_exp_neg(double x) {
  if (!(x > -745.0)) return 0.0;
  const double k = rint(x * 1.4426950408889634);
  const double r = fma(k, -1.90821492927058770002e-10, fma(k, -6.93147180369123816490e-01, x));
  double e = 1.0 / 479001600.0;
#pragma unroll
  for (int n = 11; n >= 1; --n) {
    double f = 1.0;
    for (int i = 2; i <= n; ++i) f *= i;
    e = fma(e, r, 1.0 / f);
  }
  e = fma(e, r, 1.0);
  const int k1 = (int)k / 2, k2 = (int)k - k1;
  return e * __hiloint2double((1023 + k1) << 20, 0) * __hiloint2double((1023 + k2) << 20, 0);
}

// One CTA per prompt: p = bf16(softmax(logits)) with special ids -inf (row max, exponentials and their sum in fp64, one
// rounding to bf16; 4.28's bf16 softmax computes in fp32 with torch's own summation order, so the two can differ by one bf16
// ulp where the fp32 value sits next to a rounding midpoint: fp64 gives the exact value, independent of any order), then the K largest p ordered by (p desc, token id asc).  The K-th largest key is found with sample_topk_kernel's
// two radix passes over the 16-bit key; of the tokens sharing it, the lowest ids are taken (contiguous chunks in token order).
__global__ void __launch_bounds__(CT_THREADS) contrastive_topk_kernel(const __nv_bfloat16* __restrict__ logits, int64_t ld, int V,
                                                                      const int* __restrict__ special, int n_special, int K,
                                                                      __nv_bfloat16* __restrict__ p_out, int* __restrict__ tok_out) {
  extern __shared__ float sc[];                              // [V] logits, then p
  __shared__ int hist[256];
  __shared__ float red[32];
  __shared__ double redd[32];
  __shared__ int s_special[MAX_SPECIAL];
  __shared__ int s_n;
  __shared__ uint32_t s_key[CT_KMAX];                        // (p bits << 17) | (0x1ffff - token): larger is better
  griddep_launch();
  griddep_wait();
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  if (tid < n_special) s_special[tid] = special[tid];
  if (tid < 256) hist[tid] = 0;
  if (tid == 0) s_n = 0;
  __syncthreads();
  const __nv_bfloat16* row = logits + (int64_t)b * ld;
  float mx = -INFINITY;
  for (int c = tid; c < V; c += CT_THREADS) {
    bool sp = false;
    for (int s = 0; s < n_special; ++s) sp |= (s_special[s] == c);
    const float v = sp ? -INFINITY : __bfloat162float(row[c]);
    sc[c] = v;
    mx = fmaxf(mx, v);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if (lane == 0) red[w] = mx;
  __syncthreads();
  mx = red[lane];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  double s = 0.0;
  for (int c = tid; c < V; c += CT_THREADS) s += ct_exp_neg((double)sc[c] - (double)mx);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) redd[w] = s;
  __syncthreads();
  s = redd[lane];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const double inv = __drcp_rn(s);                         // 1 ulp of fp64 is far below the bf16 rounding of p
  for (int c = tid; c < V; c += CT_THREADS) {
    const float p = __bfloat162float(__double2bfloat16(ct_exp_neg((double)sc[c] - (double)mx) * inv));
    sc[c] = p;
    atomicAdd(&hist[smp_key16(p) >> 8], 1);
  }
  __syncthreads();
  int hi_bin, above;
  smp_pick_bin(hist, K, hi_bin, above);
  if (tid < 256) hist[tid] = 0;
  __syncthreads();
  for (int c = tid; c < V; c += CT_THREADS) {
    const uint32_t key = smp_key16(sc[c]);
    if ((int)(key >> 8) == hi_bin) atomicAdd(&hist[key & 255u], 1);
  }
  __syncthreads();
  int lo_bin, above2;
  smp_pick_bin(hist, K - above, lo_bin, above2);
  const uint32_t thr = ((uint32_t)hi_bin << 8) | (uint32_t)lo_bin;
  const int need = K - above - above2;                      // tokens of key thr taken, lowest ids first
  const int CH = (V + CT_THREADS - 1) / CT_THREADS;
  const int c0 = min(tid * CH, V), c1 = min(c0 + CH, V);
  int cnt = 0;
  for (int c = c0; c < c1; ++c) cnt += smp_key16(sc[c]) == thr;
  int before = smp_cta_exclusive(cnt, hist);
  for (int c = c0; c < c1; ++c) {
    const float p = sc[c];
    const uint32_t key = smp_key16(p);
    bool take = key > thr;
    if (key == thr) take = before++ < need;
    if (take) s_key[atomicAdd(&s_n, 1)] = ((__float_as_uint(p) >> 16) << 17) | (0x1ffffu - (uint32_t)c);
  }
  __syncthreads();
  if (tid < K) {                                             // rank sort: the keys are distinct
    const uint32_t x = s_key[tid];
    int r = 0;
    for (int j = 0; j < K; ++j) r += s_key[j] > x;
    tok_out[b * K + r] = (int)(0x1ffffu - (x & 0x1ffffu));
    p_out[b * K + r] = __ushort_as_bfloat16((unsigned short)(x >> 17));
  }
}

// One warp per packed prompt row: ctx[b, i] = x^ of hn[cu[b] + i] (i < Sc), ctx_len[b] = the prompt's length.
__global__ void __launch_bounds__(256) contrastive_context_kernel(const __nv_bfloat16* __restrict__ hn, const int* __restrict__ cu, int B,
                                                                 int T, __nv_bfloat16* __restrict__ ctx, int* __restrict__ ctx_len, int Sc,
                                                                 int D) {
  griddep_launch();
  griddep_wait();
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= T) return;
  int b = 0;
  while (b + 1 < B && cu[b + 1] <= row) ++b;
  const int i = row - cu[b];
  if (i < Sc) ct_normalize_row(hn + (int64_t)row * D, ctx + ((int64_t)b * Sc + i) * D, D, lane);
  if (i == 0 && lane == 0) ctx_len[b] = cu[b + 1] - cu[b];
}

// grid (CR_SPLIT, B): CTA (s, b) takes its share of the ctx_len[b] context rows of prompt b and folds max_i bf16(c^_i . h^_j) of
// each candidate j into pen_key[b * K + j] (an f32_order key; 0 is below every value, and the select kernel resets it).  The
// candidates are normalised into shared memory CR_CHUNK at a time; a warp walks a context row per iteration.
__global__ void __launch_bounds__(CR_THREADS) contrastive_pen_kernel(const __nv_bfloat16* __restrict__ hn, const __nv_bfloat16* __restrict__ ctx,
                                                                     const int* __restrict__ ctx_len, int Sc, int D, int K,
                                                                     unsigned* __restrict__ pen_key) {
  extern __shared__ uint4 cr_smem[];                         // [CR_CHUNK, D] bf16 normalised candidates
  __nv_bfloat16* s_h = reinterpret_cast<__nv_bfloat16*>(cr_smem);
  __shared__ unsigned s_max[CR_CHUNK];
  griddep_launch();
  griddep_wait();
  constexpr int NW = CR_THREADS / 32;
  const int b = blockIdx.y, tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int n = min(ctx_len[b], Sc);
  const int per = (n + CR_SPLIT - 1) / CR_SPLIT;
  const int i0 = blockIdx.x * per, i1 = min(n, i0 + per);
  if (i0 >= i1) return;                                      // uniform over the CTA
  for (int j0 = 0; j0 < K; j0 += CR_CHUNK) {
    const int nj = min(CR_CHUNK, K - j0);
    __syncthreads();                                         // the previous chunk is consumed
    for (int jj = w; jj < nj; jj += NW) ct_normalize_row(hn + (int64_t)(b * K + j0 + jj) * D, s_h + (int64_t)jj * D, D, lane);
    if (tid < CR_CHUNK) s_max[tid] = 0u;
    __syncthreads();
    unsigned wmax[CR_CHUNK];
#pragma unroll
    for (int jj = 0; jj < CR_CHUNK; ++jj) wmax[jj] = 0u;
    for (int i = i0 + w; i < i1; i += NW) {
      const __nv_bfloat16* c = ctx + ((int64_t)b * Sc + i) * D;
      float acc[CR_CHUNK];
#pragma unroll
      for (int jj = 0; jj < CR_CHUNK; ++jj) acc[jj] = 0.f;
      for (int d = lane * 8; d < D; d += 256) {
        float cf[8];
        unpack8d(*reinterpret_cast<const uint4*>(c + d), cf);
#pragma unroll
        for (int jj = 0; jj < CR_CHUNK; ++jj) {
          if (jj < nj) {
            float hf[8];
            unpack8d(*reinterpret_cast<const uint4*>(s_h + (int64_t)jj * D + d), hf);
#pragma unroll
            for (int e = 0; e < 8; ++e) acc[jj] = __fmaf_rn(cf[e], hf[e], acc[jj]);
          }
        }
      }
#pragma unroll
      for (int jj = 0; jj < CR_CHUNK; ++jj) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc[jj] += __shfl_xor_sync(0xffffffffu, acc[jj], o);
        wmax[jj] = max(wmax[jj], f32_order(bf16_round(acc[jj])));
      }
    }
    if (lane == 0)
      for (int jj = 0; jj < nj; ++jj) atomicMax(&s_max[jj], wmax[jj]);
    __syncthreads();
    if (tid < nj) atomicMax(&pen_key[b * K + j0 + tid], s_max[tid]);
  }
}

// One CTA per prompt: scores, the first best candidate sel[b], its token (pad once the row is finished; EOS finishes it as in
// argmax_kernel), x^ of its row appended to the context, its final-norm row gathered into hsel[b] for the lm_head; then plens[b]
// and the K candidate rows' lens advance (nv_contrastive_commit stores the K/V at plens[b] - 1).  pen_key is reset for the next
// step.  pen_out / score_out (optional, fp32 [B, K]) receive pen and the score.
__global__ void __launch_bounds__(CS_THREADS) contrastive_select_kernel(const __nv_bfloat16* __restrict__ hn, __nv_bfloat16* __restrict__ ctx,
                                                                        int* __restrict__ ctx_len, int Sc, int D, int K,
                                                                        unsigned* __restrict__ pen_key, const __nv_bfloat16* __restrict__ p,
                                                                        const int* __restrict__ tok, float a1, float a,
                                                                        int* __restrict__ finished, int eos_id, int pad_id, int stop_on_eos,
                                                                        int* __restrict__ next, int* __restrict__ sel,
                                                                        __nv_bfloat16* __restrict__ hsel, int* __restrict__ plens,
                                                                        int* __restrict__ lens, float* __restrict__ pen_out,
                                                                        float* __restrict__ score_out) {
  __shared__ int s_sel;
  griddep_launch();
  griddep_wait();
  const int b = blockIdx.x, tid = threadIdx.x;
  if (tid == 0) {
    float best = -INFINITY;
    int bj = 0;
    for (int j = 0; j < K; ++j) {
      const float pen = f32_unorder(pen_key[b * K + j]);
      pen_key[b * K + j] = 0u;
      const float pj = __bfloat162float(p[b * K + j]);
      const float score = bf16_round(__fsub_rn(bf16_round(__fmul_rn(a1, pj)), bf16_round(__fmul_rn(a, pen))));
      if (j == 0 || score > best) { best = score; bj = j; }
      if (pen_out) pen_out[b * K + j] = pen;
      if (score_out) score_out[b * K + j] = score;
    }
    s_sel = bj;
    sel[b] = bj;
    int t = tok[b * K + bj];
    if (finished[b]) t = pad_id;
    else if (stop_on_eos && t == eos_id) finished[b] = 1;
    next[b] = t;
  }
  __syncthreads();
  const int64_t r = (int64_t)b * K + s_sel;
  const int n = ctx_len[b];
  if (tid < 32 && n < Sc) ct_normalize_row(hn + r * D, ctx + ((int64_t)b * Sc + n) * D, D, tid);
  for (int c = tid * 8; c < D; c += CS_THREADS * 8)
    *reinterpret_cast<uint4*>(hsel + (int64_t)b * D + c) = *reinterpret_cast<const uint4*>(hn + r * D + c);
  __syncthreads();
  if (tid == 0) {
    if (n < Sc) ctx_len[b] = n + 1;
    plens[b] += 1;
  }
  if (tid < K) lens[b * K + tid] += 1;
}

// grid (L, B): layer l's K and V rows of the selected candidate (row b * K + sel[b] of the one-slot candidate caches) go to row
// plens[b] - 1 of prompt b's cache.  table[l * 8 ..]: kc, vc, pk, pv, then for fp8 the four exponent arrays (else null).  A row
// is row_bytes of K or V (bf16, or e4m3 bytes) and exp_bytes exponents; a plain byte copy, so the bits are the candidate's.
__global__ void __launch_bounds__(256) contrastive_commit_kernel(const unsigned long long* __restrict__ table, const int* __restrict__ sel,
                                                                 const int* __restrict__ plens, int K, int Sp, int row_bytes,
                                                                 int exp_bytes) {
  griddep_launch();
  griddep_wait();
  const int l = blockIdx.x, b = blockIdx.y;
  const unsigned long long* t = table + (int64_t)l * 8;
  const int64_t src = (int64_t)b * K + sel[b], dst = (int64_t)b * Sp + plens[b] - 1;
  const int n16 = row_bytes >> 4;
  for (int kv = 0; kv < 2; ++kv) {
    const uint4* s = reinterpret_cast<const uint4*>(t[kv]) + src * n16;
    uint4* d = reinterpret_cast<uint4*>(t[2 + kv]) + dst * n16;
    for (int i = threadIdx.x; i < n16; i += blockDim.x) d[i] = s[i];
    if (exp_bytes) {
      const int8_t* se = reinterpret_cast<const int8_t*>(t[4 + kv]) + src * exp_bytes;
      int8_t* de = reinterpret_cast<int8_t*>(t[6 + kv]) + dst * exp_bytes;
      for (int i = threadIdx.x; i < exp_bytes; i += blockDim.x) de[i] = se[i];
    }
  }
}

}  // namespace nv

using namespace nv;
#define S_(x) reinterpret_cast<cudaStream_t>(x)
#define BF(x) reinterpret_cast<__nv_bfloat16*>(x)
#define CBF(x) reinterpret_cast<const __nv_bfloat16*>(x)

// Prompt-lookup speculative decoding (generation.lookup_decode): the verify window's attention, the drafts and the accept step.
template <bool FP8>
static int launch_window(const char* name, const void* qkv, int64_t ld, const int* lens, const void* cos_t, const void* sin_t,
                         void* kc, void* vc, void* kexp, void* vexp, void* out, int64_t ldo, int B, int W, int Smax, int H,
                         int head_dim, float scale, void* stream) {
  NV_REQUIRE(head_dim == 128 && (ld & 7) == 0 && (ldo & 7) == 0, "%s: head_dim must be 128, ld %% 8 == 0, ldo %% 8 == 0", name);
  NV_REQUIRE(B >= 0 && W >= 1 && W <= WIN_MAX && Smax > 0 && H > 0, "%s: bad sizes (B=%d W=%d Smax=%d H=%d; 1 <= W <= %d)", name, B,
             W, Smax, H, WIN_MAX);
  if (B == 0) return NV_OK;
  NV_REQUIRE(qkv && lens && cos_t && sin_t && kc && vc && out && (!FP8 || (kexp && vexp)), "%s: null argument", name);
  NV_REQUIRE(((uintptr_t)qkv & 15) == 0 && ((uintptr_t)kc & 7) == 0 && ((uintptr_t)vc & 7) == 0, "%s: alignment", name);
  using E = kv_elem_t<FP8>;
  E* k = reinterpret_cast<E*>(kc);
  E* v = reinterpret_cast<E*>(vc);
  int8_t* kx = reinterpret_cast<int8_t*>(kexp);
  int8_t* vx = reinterpret_cast<int8_t*>(vexp);
  // the fewest queries per CTA that hold the window, at most 8 (the registers of 8 queries' states next to the loads in flight)
  const int qpc = W <= 2 ? 2 : W <= 4 ? 4 : 8;
  const dim3 grid(B * H, (W + qpc - 1) / qpc), block(DA_WARPS * 32);
  if (qpc == 2)
    NV_CUDA(launch_pdl(decode_attn_window_kernel<FP8, 2>, grid, block, 0, S_(stream), CBF(qkv), ld, k, v, kx, vx, lens, BF(out), ldo,
                       Smax, H, W, scale, CBF(cos_t), CBF(sin_t)));
  else if (qpc == 4)
    NV_CUDA(launch_pdl(decode_attn_window_kernel<FP8, 4>, grid, block, 0, S_(stream), CBF(qkv), ld, k, v, kx, vx, lens, BF(out), ldo,
                       Smax, H, W, scale, CBF(cos_t), CBF(sin_t)));
  else
    NV_CUDA(launch_pdl(decode_attn_window_kernel<FP8, 8>, grid, block, 0, S_(stream), CBF(qkv), ld, k, v, kx, vx, lens, BF(out), ldo,
                       Smax, H, W, scale, CBF(cos_t), CBF(sin_t)));
  return NV_OK;
}

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
                     (const __nv_bfloat16*)nullptr, (const __nv_bfloat16*)nullptr, (int8_t*)nullptr, (int8_t*)nullptr,
                     BeamKV<false>{}));
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
                     BF(out), ldo, Smax, H, scale, CBF(cos_t), CBF(sin_t), (int8_t*)nullptr, (int8_t*)nullptr, BeamKV<false>{}));
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
                     CBF(sin_t), reinterpret_cast<int8_t*>(kexp), reinterpret_cast<int8_t*>(vexp), BeamKV<true>{}));
  return NV_OK;
}

int nv_decode_attn_rope_window(const void* qkv, int64_t ld, const int* lens, const void* cos_t, const void* sin_t, void* kcache,
                               void* vcache, void* out, int64_t ldo, int B, int W, int Smax, int H, int head_dim, float scale,
                               void* stream) {
  return launch_window<false>("nv_decode_attn_rope_window", qkv, ld, lens, cos_t, sin_t, kcache, vcache, nullptr, nullptr, out, ldo,
                              B, W, Smax, H, head_dim, scale, stream);
}

int nv_decode_attn_rope_window_fp8(const void* qkv, int64_t ld, const int* lens, const void* cos_t, const void* sin_t, void* kq,
                                   void* vq, void* kexp, void* vexp, void* out, int64_t ldo, int B, int W, int Smax, int H,
                                   int head_dim, float scale, void* stream) {
  return launch_window<true>("nv_decode_attn_rope_window_fp8", qkv, ld, lens, cos_t, sin_t, kq, vq, kexp, vexp, out, ldo, B, W, Smax,
                             H, head_dim, scale, stream);
}

int nv_lookup_draft(const int* hist, int ld_hist, const int* hist_len, const int* finished, const int* special, int n_special,
                    int eos_id, int K, int ngram, int* drafts, int* win_ids, int B, void* stream) {
  NV_REQUIRE(K >= 1 && K < WIN_MAX && ngram >= 1 && n_special >= 0 && n_special <= MAX_SPECIAL && B >= 0,
             "nv_lookup_draft: bad arguments (K=%d ngram=%d n_special=%d B=%d)", K, ngram, n_special, B);
  if (B == 0) return NV_OK;
  NV_REQUIRE(hist && hist_len && finished && drafts && win_ids && (special || n_special == 0), "nv_lookup_draft: null argument");
  NV_CUDA(launch_pdl(lookup_draft_kernel, dim3(B), dim3(LD_THREADS), 0, S_(stream), hist, ld_hist, hist_len, finished, special,
                     n_special, eos_id, K, ngram, drafts, win_ids));
  return NV_OK;
}

int nv_lookup_accept(const void* logits, int64_t ld, int V, const int* special, int n_special, const int* drafts, int K, int* finished,
                     int eos_id, int stop_on_eos, int max_new, int* out, int ld_out, int* hist, int ld_hist, int* hist_len, int* n_out,
                     int* lens, int* n_acc, int B, void* stream) {
  NV_REQUIRE(K >= 1 && K < WIN_MAX && V > 0 && n_special >= 0 && n_special <= MAX_SPECIAL && B >= 0 && max_new <= ld_out,
             "nv_lookup_accept: bad arguments (K=%d V=%d n_special=%d B=%d max_new=%d ld_out=%d)", K, V, n_special, B, max_new,
             ld_out);
  if (B == 0) return NV_OK;
  NV_REQUIRE(logits && drafts && finished && out && hist && hist_len && n_out && lens && n_acc && (special || n_special == 0),
             "nv_lookup_accept: null argument");
  NV_CUDA(launch_pdl(lookup_accept_kernel, dim3(B), dim3(1024), 0, S_(stream), CBF(logits), ld, V, special, n_special, drafts, K,
                     finished, eos_id, stop_on_eos, max_new, out, ld_out, hist, ld_hist, hist_len, n_out, lens, n_acc));
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

// Sampled next token (HF sample: temperature -> top-k -> top-p -> softmax -> multinomial); see sample_topk_kernel.  logits
// [B, V] bf16, u [B] uniform numbers in [0, 1), probs_out: optional fp32 [B, V] copy of the sampling distribution (tests).
// top_p in [0, 1]; 1 is off, as in HF, which only adds the top-p warper below 1.
int nv_sample(const void* logits, int64_t ld, int V, const int* special, int n_special, int* finished, int eos_id, int pad_id,
              int stop_on_eos, float temperature, int top_k, float top_p, const float* u, int* next, float* probs_out, int B,
              void* stream) {
  NV_REQUIRE(logits && u && next && finished && V > 0 && temperature > 0.f, "nv_sample: bad arguments (temperature must be > 0)");
  NV_REQUIRE(top_p >= 0.f && top_p <= 1.f, "nv_sample: top_p=%g outside [0, 1]", (double)top_p);
  NV_REQUIRE(n_special >= 0 && n_special <= MAX_SPECIAL, "nv_sample: n_special=%d out of range (max %d)", n_special, MAX_SPECIAL);
  NV_REQUIRE((int64_t)V * 4 <= 200 * 1024, "nv_sample: vocabulary of %d does not fit the shared-memory score row", V);
  if (B == 0) return NV_OK;
  static bool attr_set = false;
  if (!attr_set) {
    NV_CUDA(cudaFuncSetAttribute(sample_topk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr_set = true;
  }
  // TopPLogitsWarper compares the bf16 running sum with the Python scalar 1 - top_p, which takes the bf16 dtype
  const float p_thr = __bfloat162float(__float2bfloat16_rn((float)(1.0 - (double)top_p)));
  sample_topk_kernel<<<B, SMP_THREADS, (size_t)V * 4, S_(stream)>>>(CBF(logits), ld, V, special, n_special, finished, eos_id, pad_id,
                                                                     stop_on_eos, temperature, top_k, top_p < 1.f ? 1 : 0, p_thr, u,
                                                                     next, probs_out);
  NV_LAUNCH_CHECK();
  return NV_OK;
}

int nv_sample_topk(const void* logits, int64_t ld, int V, const int* special, int n_special, int* finished, int eos_id, int pad_id,
                   int stop_on_eos, float temperature, int top_k, const float* u, int* next, float* probs_out, int B, void* stream) {
  return nv_sample(logits, ld, V, special, n_special, finished, eos_id, pad_id, stop_on_eos, temperature, top_k, 1.f, u, next,
                   probs_out, B, stream);
}

static int check_scores(const char* name, const void* scores, int64_t ld_scores, int64_t plane, const int* step, int V, int rows) {
  NV_REQUIRE(scores && step && ld_scores >= V && plane >= (int64_t)rows * ld_scores,
             "%s: scores planes [G, %d, ld_scores >= %d] and a step pointer expected (ld_scores=%lld, plane=%lld)", name, rows, V,
             (long long)ld_scores, (long long)plane);
  return NV_OK;
}

// nv_sample that also writes the warped scores of each row to plane step[0] of scores (see sample_body<true>).  The argument
// checks are nv_sample's (its B = 0 call launches nothing).
int nv_sample_scores(const void* logits, int64_t ld, int V, const int* special, int n_special, int* finished, int eos_id, int pad_id,
                     int stop_on_eos, float temperature, int top_k, float top_p, const float* u, int* next, float* probs_out,
                     void* scores, int64_t ld_scores, int64_t plane, const int* step, int B, void* stream) {
  int st = nv_sample(logits, ld, V, special, n_special, finished, eos_id, pad_id, stop_on_eos, temperature, top_k, top_p, u, next,
                     probs_out, 0, stream);
  if (st == NV_OK) st = check_scores("nv_sample_scores", scores, ld_scores, plane, step, V, B);
  if (st != NV_OK || B == 0) return st;
  static bool attr_set = false;
  if (!attr_set) {
    NV_CUDA(cudaFuncSetAttribute(sample_scores_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr_set = true;
  }
  const float p_thr = __bfloat162float(__float2bfloat16_rn((float)(1.0 - (double)top_p)));
  sample_scores_kernel<<<B, SMP_THREADS, (size_t)V * 4, S_(stream)>>>(CBF(logits), ld, V, special, n_special, finished, eos_id, pad_id,
                                                                       stop_on_eos, temperature, top_k, top_p < 1.f ? 1 : 0, p_thr, u,
                                                                       next, probs_out, ScoresOut{BF(scores), ld_scores, plane, step, 0});
  NV_LAUNCH_CHECK();
  return NV_OK;
}

// R rows of src to plane step[0] of scores, special ids -inf (see scores_store_kernel).
int nv_scores_store(const void* src, int64_t ld, int V, const int* special, int n_special, void* scores, int64_t ld_scores,
                    int64_t plane, const int* step, int R, void* stream) {
  NV_REQUIRE(src && V > 0 && ld >= V && R >= 0 && n_special >= 0 && n_special <= MAX_SPECIAL && (special || n_special == 0),
             "nv_scores_store: bad arguments (V=%d ld=%lld R=%d n_special=%d)", V, (long long)ld, R, n_special);
  const int st = check_scores("nv_scores_store", scores, ld_scores, plane, step, V, R);
  if (st != NV_OK || R == 0) return st;
  NV_CUDA(launch_pdl(scores_store_kernel, dim3(R, (V + SS_CHUNK - 1) / SS_CHUNK), dim3(SS_THREADS), 0, S_(stream), CBF(src), ld, V,
                     special, n_special,
                     ScoresOut{BF(scores), ld_scores, plane, step, 0}));
  return NV_OK;
}

// After nv_lookup_accept: the logits rows of the emitted tokens to their planes (see lookup_scores_kernel).
int nv_lookup_scores(const void* logits, int64_t ld, int V, const int* special, int n_special, const int* n_prev, const int* n_out,
                     int W, void* scores, int64_t ld_scores, int64_t plane, int B, void* stream) {
  NV_REQUIRE(logits && n_prev && n_out && scores && V > 0 && ld >= V && ld_scores >= V && plane >= (int64_t)B * ld_scores && W >= 1 &&
             W <= WIN_MAX && B >= 0 && n_special >= 0 && n_special <= MAX_SPECIAL && (special || n_special == 0),
             "nv_lookup_scores: bad arguments (V=%d W=%d B=%d ld_scores=%lld plane=%lld)", V, W, B, (long long)ld_scores,
             (long long)plane);
  if (B == 0) return NV_OK;
  NV_CUDA(launch_pdl(lookup_scores_kernel, dim3(B, W, (V + SS_CHUNK - 1) / SS_CHUNK), dim3(SS_THREADS), 0, S_(stream), CBF(logits),
                     ld, V, special, n_special, n_prev, n_out, W, BF(scores), ld_scores, plane));
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

// Beam search (see beam_topk_kernel / beam_select_kernel).  Beam k of prompt b reads logits row b * ld_prompt + k * ld_beam
// (ld_beam = 0 at the first step, whose K beams all read the prompt's prefill row).
int nv_beam_topk(const void* logits, int64_t ld_prompt, int64_t ld_beam, int V, const int* special, int n_special,
                 const float* beam_score, float* cand_score, int* cand_tok, int* cand_parent, int B, int K, void* stream) {
  NV_REQUIRE(logits && beam_score && cand_score && cand_tok && cand_parent && V > 0 && B >= 0,
             "nv_beam_topk: bad arguments (V=%d B=%d)", V, B);
  NV_REQUIRE(K >= 1 && K <= BEAM_MAX && 2 * K <= V, "nv_beam_topk: %d beams: 1..%d beams and V >= 2K supported", K, BEAM_MAX);
  NV_REQUIRE((int64_t)K * V < 0xffffffffll, "nv_beam_topk: K * V = %lld does not fit the 32-bit candidate index", (long long)K * V);
  NV_REQUIRE(n_special >= 0 && n_special <= MAX_SPECIAL && (n_special == 0 || special),
             "nv_beam_topk: n_special=%d out of range (max %d)", n_special, MAX_SPECIAL);
  if (B == 0) return NV_OK;
  NV_CUDA(launch_pdl(beam_topk_kernel, dim3(B), dim3(BT_THREADS), 0, S_(stream), CBF(logits), ld_prompt, ld_beam, V, special,
                     n_special, beam_score, K, cand_score, cand_tok, cand_parent));
  return NV_OK;
}

// nv_beam_topk that also writes each beam's bf16 log-probs to plane prompt_state[b, 0] of scores [G, B * K, ld_scores] (see
// beam_topk_body<..., true>).  The argument checks are nv_beam_topk's (its B = 0 call launches nothing).
int nv_beam_topk_scores(const void* logits, int64_t ld_prompt, int64_t ld_beam, int V, const int* special, int n_special,
                        const float* beam_score, float* cand_score, int* cand_tok, int* cand_parent, const int* prompt_state,
                        void* scores, int64_t ld_scores, int64_t plane, int B, int K, void* stream) {
  int st = nv_beam_topk(logits, ld_prompt, ld_beam, V, special, n_special, beam_score, cand_score, cand_tok, cand_parent, 0, K, stream);
  if (st == NV_OK) st = check_scores("nv_beam_topk_scores", scores, ld_scores, plane, prompt_state, V, B * K);
  if (st != NV_OK || B == 0) return st;
  NV_CUDA(launch_pdl(beam_topk_scores_kernel, dim3(B), dim3(BT_THREADS), 0, S_(stream), CBF(logits), ld_prompt, ld_beam, V, special,
                     n_special, beam_score, K, cand_score, cand_tok, cand_parent,
                     ScoresOut{BF(scores), ld_scores, plane, prompt_state, BS_FIELDS}));
  return NV_OK;
}

static int check_proc(const char* name, int V, float penalty, int ngram, int min_length, int min_new_tokens) {
  NV_REQUIRE(penalty > 0.f && ngram >= 0 && min_length >= 0 && min_new_tokens >= 0,
             "%s: penalty=%g must be > 0, ngram=%d / min_length=%d / min_new_tokens=%d >= 0", name, (double)penalty, ngram, min_length,
             min_new_tokens);
  NV_REQUIRE(V > 0 && (int64_t)((V + 31) / 32) * 4 * 2 <= 48 * 1024, "%s: vocabulary of %d does not fit the shared bitmaps", name, V);
  return NV_OK;
}

// Logits processors in place on R bf16 rows (see logits_process_kernel).
int nv_logits_process(void* logits, int64_t ld, int V, const int* prompt_ids, int64_t ld_prompt, const int* prompt_width,
                      int rows_per_prompt, int* hist, int G, int* hist_len, const int* append, float penalty, int ngram,
                      int min_length, int min_new_tokens, int eos_id, int R, void* stream) {
  NV_REQUIRE(logits && prompt_ids && prompt_width && hist && hist_len && rows_per_prompt >= 1 && G > 0 && R >= 0 && ld >= V,
             "nv_logits_process: bad arguments (R=%d G=%d rows_per_prompt=%d)", R, G, rows_per_prompt);
  const int st = check_proc("nv_logits_process", V, penalty, ngram, min_length, min_new_tokens);
  if (st != NV_OK) return st;
  if (R == 0) return NV_OK;
  NV_CUDA(launch_pdl(logits_process_kernel, dim3(R), dim3(LP_THREADS), (size_t)((V + 31) / 32) * 4, S_(stream), BF(logits), ld, V,
                     prompt_ids, ld_prompt, prompt_width, rows_per_prompt, hist, G, hist_len, append,
                     ProcParams{penalty, ngram, min_length, min_new_tokens, eos_id}));
  return NV_OK;
}

// nv_beam_topk with the logits processors on each log-prob (see beam_topk_kernel<true>).
int nv_beam_topk_processed(const void* logits, int64_t ld_prompt, int64_t ld_beam, int V, const int* special, int n_special,
                           const float* beam_score, float* cand_score, int* cand_tok, int* cand_parent, const int* prompt_ids,
                           int64_t ld_ids, const int* prompt_width, const int* hist, int G, const int* prompt_state, float penalty,
                           int ngram, int min_length, int min_new_tokens, int eos_id, int B, int K, void* stream) {
  NV_REQUIRE(logits && beam_score && cand_score && cand_tok && cand_parent && prompt_ids && prompt_width && hist && prompt_state &&
             V > 0 && B >= 0 && G > 0, "nv_beam_topk_processed: bad arguments (V=%d B=%d G=%d)", V, B, G);
  NV_REQUIRE(K >= 1 && K <= BEAM_MAX && 2 * K <= V, "nv_beam_topk_processed: %d beams: 1..%d beams and V >= 2K supported", K,
             BEAM_MAX);
  NV_REQUIRE((int64_t)K * V < 0xffffffffll, "nv_beam_topk_processed: K * V = %lld does not fit the 32-bit candidate index",
             (long long)K * V);
  NV_REQUIRE(n_special >= 0 && n_special <= MAX_SPECIAL && (n_special == 0 || special),
             "nv_beam_topk_processed: n_special=%d out of range (max %d)", n_special, MAX_SPECIAL);
  const int st = check_proc("nv_beam_topk_processed", V, penalty, ngram, min_length, min_new_tokens);
  if (st != NV_OK) return st;
  if (B == 0) return NV_OK;
  const BeamProc bp{prompt_ids, ld_ids, prompt_width, hist, G, prompt_state, ProcParams{penalty, ngram, min_length, min_new_tokens, eos_id}};
  NV_CUDA(launch_pdl(beam_topk_proc_kernel, dim3(B), dim3(BT_THREADS), (size_t)((V + 31) / 32) * 4 * 2, S_(stream), CBF(logits),
                     ld_prompt, ld_beam, V, special, n_special, beam_score, K, cand_score, cand_tok, cand_parent, bp));
  return NV_OK;
}

// nv_beam_topk_processed with the scores output of nv_beam_topk_scores.
int nv_beam_topk_processed_scores(const void* logits, int64_t ld_prompt, int64_t ld_beam, int V, const int* special, int n_special,
                                  const float* beam_score, float* cand_score, int* cand_tok, int* cand_parent, const int* prompt_ids,
                                  int64_t ld_ids, const int* prompt_width, const int* hist, int G, const int* prompt_state,
                                  float penalty, int ngram, int min_length, int min_new_tokens, int eos_id, void* scores,
                                  int64_t ld_scores, int64_t plane, int B, int K, void* stream) {
  int st = nv_beam_topk_processed(logits, ld_prompt, ld_beam, V, special, n_special, beam_score, cand_score, cand_tok, cand_parent,
                                  prompt_ids, ld_ids, prompt_width, hist, G, prompt_state, penalty, ngram, min_length, min_new_tokens,
                                  eos_id, 0, K, stream);
  if (st == NV_OK) st = check_scores("nv_beam_topk_processed_scores", scores, ld_scores, plane, prompt_state, V, B * K);
  if (st != NV_OK || B == 0) return st;
  const BeamProc bp{prompt_ids, ld_ids, prompt_width, hist, G, prompt_state, ProcParams{penalty, ngram, min_length, min_new_tokens, eos_id}};
  NV_CUDA(launch_pdl(beam_topk_proc_scores_kernel, dim3(B), dim3(BT_THREADS), (size_t)((V + 31) / 32) * 4 * 2, S_(stream),
                     CBF(logits), ld_prompt, ld_beam, V, special, n_special, beam_score, K, cand_score, cand_tok, cand_parent, bp,
                     ScoresOut{BF(scores), ld_scores, plane, prompt_state, BS_FIELDS}));
  return NV_OK;
}

// nv_beam_topk_processed with the trie mask after the processors (see beam_topk_trie_kernel).  The CSR trie as nv_trie_mask
// reads it; V must fit three V-bit bitmaps in 48 KB.
int nv_beam_topk_trie(const void* logits, int64_t ld_prompt, int64_t ld_beam, int V, const int* special, int n_special,
                      const float* beam_score, float* cand_score, int* cand_tok, int* cand_parent, const int* prompt_ids,
                      int64_t ld_ids, const int* prompt_width, const int* hist, int G, const int* prompt_state, float penalty,
                      int ngram, int min_length, int min_new_tokens, int eos_id, const int* node_ptr, const int* child_tok,
                      const int* child_node, int n_nodes, int leaf_tok, int B, int K, void* stream) {
  NV_REQUIRE(logits && beam_score && cand_score && cand_tok && cand_parent && prompt_ids && prompt_width && hist && prompt_state &&
             node_ptr && child_tok && child_node && V > 0 && B >= 0 && G > 0,
             "nv_beam_topk_trie: bad arguments (V=%d B=%d G=%d)", V, B, G);
  NV_REQUIRE(K >= 1 && K <= BEAM_MAX && 2 * K <= V, "nv_beam_topk_trie: %d beams: 1..%d beams and V >= 2K supported", K, BEAM_MAX);
  NV_REQUIRE((int64_t)K * V < 0xffffffffll, "nv_beam_topk_trie: K * V = %lld does not fit the 32-bit candidate index",
             (long long)K * V);
  NV_REQUIRE(n_special >= 0 && n_special <= MAX_SPECIAL && (n_special == 0 || special),
             "nv_beam_topk_trie: n_special=%d out of range (max %d)", n_special, MAX_SPECIAL);
  NV_REQUIRE(n_nodes >= 1 && leaf_tok >= 0 && leaf_tok < V, "nv_beam_topk_trie: n_nodes=%d (>= 1), leaf_tok=%d outside [0, %d)",
             n_nodes, leaf_tok, V);
  const int st = check_proc("nv_beam_topk_trie", V, penalty, ngram, min_length, min_new_tokens);
  if (st != NV_OK) return st;
  const size_t smem = (size_t)((V + 31) / 32) * 4 * 3;
  NV_REQUIRE(smem <= 48 * 1024, "nv_beam_topk_trie: vocabulary of %d does not fit the three shared bitmaps", V);
  if (B == 0) return NV_OK;
  const BeamProc bp{prompt_ids, ld_ids, prompt_width, hist, G, prompt_state, ProcParams{penalty, ngram, min_length, min_new_tokens, eos_id}};
  const BeamTrie tr{node_ptr, child_tok, child_node, n_nodes, leaf_tok};
  NV_CUDA(launch_pdl(beam_topk_trie_kernel, dim3(B), dim3(BT_THREADS), smem, S_(stream), CBF(logits), ld_prompt, ld_beam, V,
                     special, n_special, beam_score, K, cand_score, cand_tok, cand_parent, bp, tr));
  return NV_OK;
}

// nv_beam_topk_trie with the scores output of nv_beam_topk_scores.
int nv_beam_topk_trie_scores(const void* logits, int64_t ld_prompt, int64_t ld_beam, int V, const int* special, int n_special,
                             const float* beam_score, float* cand_score, int* cand_tok, int* cand_parent, const int* prompt_ids,
                             int64_t ld_ids, const int* prompt_width, const int* hist, int G, const int* prompt_state, float penalty,
                             int ngram, int min_length, int min_new_tokens, int eos_id, const int* node_ptr, const int* child_tok,
                             const int* child_node, int n_nodes, int leaf_tok, void* scores, int64_t ld_scores, int64_t plane, int B,
                             int K, void* stream) {
  int st = nv_beam_topk_trie(logits, ld_prompt, ld_beam, V, special, n_special, beam_score, cand_score, cand_tok, cand_parent,
                             prompt_ids, ld_ids, prompt_width, hist, G, prompt_state, penalty, ngram, min_length, min_new_tokens, eos_id,
                             node_ptr, child_tok, child_node, n_nodes, leaf_tok, 0, K, stream);
  if (st == NV_OK) st = check_scores("nv_beam_topk_trie_scores", scores, ld_scores, plane, prompt_state, V, B * K);
  if (st != NV_OK || B == 0) return st;
  const BeamProc bp{prompt_ids, ld_ids, prompt_width, hist, G, prompt_state, ProcParams{penalty, ngram, min_length, min_new_tokens, eos_id}};
  const BeamTrie tr{node_ptr, child_tok, child_node, n_nodes, leaf_tok};
  NV_CUDA(launch_pdl(beam_topk_trie_scores_kernel, dim3(B), dim3(BT_THREADS), (size_t)((V + 31) / 32) * 4 * 3, S_(stream),
                     CBF(logits), ld_prompt, ld_beam, V, special, n_special, beam_score, K, cand_score, cand_tok, cand_parent, bp, tr,
                     ScoresOut{BF(scores), ld_scores, plane, prompt_state, BS_FIELDS}));
  return NV_OK;
}

// nv_trie_score: see include/navillm_b200.h.
int nv_trie_score(const void* logits, int64_t ld, int V, const int* special, int n_special, const int* tok, const int* path_off,
                  const int* path_rows, int eos, float* stats, float* logprob, int B, int R, int A, void* stream) {
  NV_REQUIRE(logits && (R == 1 || (tok && path_rows)) && path_off && stats && logprob && (special || n_special == 0) && V > 0 &&
             ld >= V && B > 0 && R >= 1 && A >= 1, "nv_trie_score: bad arguments (V=%d ld=%lld B=%d R=%d A=%d)", V, (long long)ld,
             B, R, A);
  NV_REQUIRE(n_special >= 0 && n_special <= MAX_SPECIAL, "nv_trie_score: n_special=%d out of range (max %d)", n_special,
             MAX_SPECIAL);
  NV_REQUIRE(eos >= 0 && eos < V, "nv_trie_score: eos=%d outside [0, %d)", eos, V);
  NV_CUDA(launch_pdl(trie_row_stats_kernel, dim3(B * R), dim3(TS_THREADS), 0, S_(stream), CBF(logits), ld, V, special, n_special,
                     stats));
  NV_CUDA(launch_pdl(trie_fold_kernel, dim3(B), dim3(TF_THREADS), 0, S_(stream), CBF(logits), ld, V, special, n_special, tok,
                     path_off, path_rows, eos, (const float*)stats, logprob, R, A));
  return NV_OK;
}

int nv_beam_select(const float* cand_score, const int* cand_tok, const int* cand_parent, float* beam_score, int* hist, int* src,
                   double* hyp_score, int* hyp_meta, int* hyp_tok, int* prompt_state, int* next_ids, int* lens, const double* norm,
                   int B, int K, int G, int eos_id, int pad_id, int early_stopping, void* stream) {
  NV_REQUIRE(cand_score && cand_tok && cand_parent && beam_score && hist && src && hyp_score && hyp_meta && hyp_tok &&
             prompt_state && next_ids && lens && norm, "nv_beam_select: null argument");
  NV_REQUIRE(K >= 1 && K <= BEAM_MAX && G > 0 && B >= 0, "nv_beam_select: bad sizes (B=%d K=%d G=%d)", B, K, G);
  if (B == 0) return NV_OK;
  NV_CUDA(launch_pdl(beam_select_kernel, dim3(B), dim3(BS_THREADS), 0, S_(stream), cand_score, cand_tok, cand_parent, beam_score,
                     hist, src, hyp_score, hyp_meta, hyp_tok, prompt_state, next_ids, lens, norm, K, G, eos_id, pad_id,
                     early_stopping));
  return NV_OK;
}

// nv_beam_select that also keeps 4.28's beam_indices: par_hist [R, G], hyp_par [B, K, G], done_step [B] (see beam_select_body<true>).
int nv_beam_select_scores(const float* cand_score, const int* cand_tok, const int* cand_parent, float* beam_score, int* hist, int* src,
                          double* hyp_score, int* hyp_meta, int* hyp_tok, int* prompt_state, int* next_ids, int* lens,
                          const double* norm, int* par_hist, int* hyp_par, int* done_step, int B, int K, int G, int eos_id, int pad_id,
                          int early_stopping, void* stream) {
  NV_REQUIRE(par_hist && hyp_par && done_step, "nv_beam_select_scores: null argument");
  const int st = nv_beam_select(cand_score, cand_tok, cand_parent, beam_score, hist, src, hyp_score, hyp_meta, hyp_tok, prompt_state,
                                next_ids, lens, norm, 0, K, G, eos_id, pad_id, early_stopping, stream);
  if (st != NV_OK || B == 0) return st;
  NV_CUDA(launch_pdl(beam_select_scores_kernel, dim3(B), dim3(BS_THREADS), 0, S_(stream), cand_score, cand_tok, cand_parent,
                     beam_score, hist, src, hyp_score, hyp_meta, hyp_tok, prompt_state, next_ids, lens, norm, K, G, eos_id, pad_id,
                     early_stopping, BeamTrace{par_hist, hyp_par, done_step}));
  return NV_OK;
}

// Diverse (group) beam search: group g of n_groups (see beam_topk_body / beam_select_body with GROUP).  One static entry for the
// four top-k forms: prompt_ids null = no processors, scores null = no scores output.
static int beam_topk_group(const char* name, const void* logits, int64_t ld_prompt, int64_t ld_beam, int V, const int* special,
                           int n_special, const float* beam_score, float* cand_score, int* cand_tok, int* cand_parent,
                           const int* prompt_ids, int64_t ld_ids, const int* prompt_width, const int* hist, int G,
                           const int* prompt_state, float penalty, int ngram, int min_length, int min_new_tokens, int eos_id,
                           void* scores, int64_t ld_scores, int64_t plane, const int* next_ids, float diversity_penalty, int group,
                           int n_groups, int B, int K, void* stream) {
  NV_REQUIRE(logits && beam_score && cand_score && cand_tok && cand_parent && next_ids && V > 0 && B >= 0,
             "%s: bad arguments (V=%d B=%d)", name, V, B);
  NV_REQUIRE(K >= 2 && K <= BEAM_MAX && n_groups >= 2 && n_groups <= K && K % n_groups == 0 && group >= 0 && group < n_groups &&
             2 * (K / n_groups) <= V, "%s: K=%d beams in %d groups (group %d): 2..%d beams, 2..K groups dividing K", name, K,
             n_groups, group, BEAM_MAX);
  NV_REQUIRE((int64_t)K * V < 0xffffffffll, "%s: K * V = %lld does not fit the 32-bit candidate index", name, (long long)K * V);
  NV_REQUIRE(n_special >= 0 && n_special <= MAX_SPECIAL && (n_special == 0 || special), "%s: n_special=%d out of range (max %d)",
             name, n_special, MAX_SPECIAL);
  NV_REQUIRE(diversity_penalty > 0.f, "%s: diversity_penalty=%g must be > 0", name, (double)diversity_penalty);
  if (prompt_ids) {
    NV_REQUIRE(prompt_width && hist && prompt_state && G > 0, "%s: processors need prompt_width, hist and prompt_state", name);
    const int st = check_proc(name, V, penalty, ngram, min_length, min_new_tokens);
    if (st != NV_OK) return st;
  }
  if (scores) {
    const int st = check_scores(name, scores, ld_scores, plane, prompt_state, V, B * K);
    if (st != NV_OK) return st;
  }
  if (B == 0) return NV_OK;
  const int Kg = K / n_groups;
  const BeamGroup gr{next_ids, diversity_penalty, group, Kg};
  const ScoresOut so{BF(scores), ld_scores, plane, prompt_state, BS_FIELDS};
  if (prompt_ids) {
    const BeamProc bp{prompt_ids, ld_ids, prompt_width, hist, G, prompt_state, ProcParams{penalty, ngram, min_length, min_new_tokens, eos_id}};
    const size_t smem = (size_t)((V + 31) / 32) * 4 * 2;
    if (scores)
      NV_CUDA(launch_pdl(beam_topk_group_proc_scores_kernel, dim3(B), dim3(BT_THREADS), smem, S_(stream), CBF(logits), ld_prompt,
                         ld_beam, V, special, n_special, beam_score, K, cand_score, cand_tok, cand_parent, bp, so, gr));
    else
      NV_CUDA(launch_pdl(beam_topk_group_proc_kernel, dim3(B), dim3(BT_THREADS), smem, S_(stream), CBF(logits), ld_prompt, ld_beam,
                         V, special, n_special, beam_score, K, cand_score, cand_tok, cand_parent, bp, gr));
  } else if (scores) {
    NV_CUDA(launch_pdl(beam_topk_group_scores_kernel, dim3(B), dim3(BT_THREADS), 0, S_(stream), CBF(logits), ld_prompt, ld_beam, V,
                       special, n_special, beam_score, K, cand_score, cand_tok, cand_parent, so, gr));
  } else {
    NV_CUDA(launch_pdl(beam_topk_group_kernel, dim3(B), dim3(BT_THREADS), 0, S_(stream), CBF(logits), ld_prompt, ld_beam, V, special,
                       n_special, beam_score, K, cand_score, cand_tok, cand_parent, gr));
  }
  return NV_OK;
}

int nv_beam_topk_group(const void* logits, int64_t ld_prompt, int64_t ld_beam, int V, const int* special, int n_special,
                       const float* beam_score, float* cand_score, int* cand_tok, int* cand_parent, const int* next_ids,
                       float diversity_penalty, int group, int n_groups, int B, int K, void* stream) {
  return beam_topk_group("nv_beam_topk_group", logits, ld_prompt, ld_beam, V, special, n_special, beam_score, cand_score, cand_tok,
                         cand_parent, nullptr, 0, nullptr, nullptr, 0, nullptr, 1.f, 0, 0, 0, -1, nullptr, 0, 0, next_ids,
                         diversity_penalty, group, n_groups, B, K, stream);
}

int nv_beam_topk_group_scores(const void* logits, int64_t ld_prompt, int64_t ld_beam, int V, const int* special, int n_special,
                              const float* beam_score, float* cand_score, int* cand_tok, int* cand_parent, const int* prompt_state,
                              void* scores, int64_t ld_scores, int64_t plane, const int* next_ids, float diversity_penalty, int group,
                              int n_groups, int B, int K, void* stream) {
  NV_REQUIRE(scores && prompt_state, "nv_beam_topk_group_scores: null scores or prompt_state");
  return beam_topk_group("nv_beam_topk_group_scores", logits, ld_prompt, ld_beam, V, special, n_special, beam_score, cand_score,
                         cand_tok, cand_parent, nullptr, 0, nullptr, nullptr, 0, prompt_state, 1.f, 0, 0, 0, -1, scores, ld_scores,
                         plane, next_ids, diversity_penalty, group, n_groups, B, K, stream);
}

int nv_beam_topk_group_processed(const void* logits, int64_t ld_prompt, int64_t ld_beam, int V, const int* special, int n_special,
                                 const float* beam_score, float* cand_score, int* cand_tok, int* cand_parent, const int* prompt_ids,
                                 int64_t ld_ids, const int* prompt_width, const int* hist, int G, const int* prompt_state,
                                 float penalty, int ngram, int min_length, int min_new_tokens, int eos_id, const int* next_ids,
                                 float diversity_penalty, int group, int n_groups, int B, int K, void* stream) {
  NV_REQUIRE(prompt_ids, "nv_beam_topk_group_processed: null prompt_ids");
  return beam_topk_group("nv_beam_topk_group_processed", logits, ld_prompt, ld_beam, V, special, n_special, beam_score, cand_score,
                         cand_tok, cand_parent, prompt_ids, ld_ids, prompt_width, hist, G, prompt_state, penalty, ngram, min_length,
                         min_new_tokens, eos_id, nullptr, 0, 0, next_ids, diversity_penalty, group, n_groups, B, K, stream);
}

int nv_beam_topk_group_processed_scores(const void* logits, int64_t ld_prompt, int64_t ld_beam, int V, const int* special,
                                        int n_special, const float* beam_score, float* cand_score, int* cand_tok, int* cand_parent,
                                        const int* prompt_ids, int64_t ld_ids, const int* prompt_width, const int* hist, int G,
                                        const int* prompt_state, float penalty, int ngram, int min_length, int min_new_tokens,
                                        int eos_id, void* scores, int64_t ld_scores, int64_t plane, const int* next_ids,
                                        float diversity_penalty, int group, int n_groups, int B, int K, void* stream) {
  NV_REQUIRE(prompt_ids && scores, "nv_beam_topk_group_processed_scores: null prompt_ids or scores");
  return beam_topk_group("nv_beam_topk_group_processed_scores", logits, ld_prompt, ld_beam, V, special, n_special, beam_score,
                         cand_score, cand_tok, cand_parent, prompt_ids, ld_ids, prompt_width, hist, G, prompt_state, penalty, ngram,
                         min_length, min_new_tokens, eos_id, scores, ld_scores, plane, next_ids, diversity_penalty, group, n_groups,
                         B, K, stream);
}

// nv_beam_select over group g's candidates [B, 2 * (K / n_groups)] (see beam_select_body<..., true>); trace pointers all null
// or all set (nv_beam_select_scores' beam_indices).
static int beam_select_group(const char* name, const float* cand_score, const int* cand_tok, const int* cand_parent, float* beam_score,
                             int* hist, int* src, double* hyp_score, int* hyp_meta, int* hyp_tok, int* prompt_state, int* next_ids,
                             int* lens, const double* norm, int* par_hist, int* hyp_par, int* done_step, int group, int n_groups, int B,
                             int K, int G, int eos_id, int pad_id, int early_stopping, void* stream) {
  NV_REQUIRE(cand_score && cand_tok && cand_parent && beam_score && hist && src && hyp_score && hyp_meta && hyp_tok &&
             prompt_state && next_ids && lens && norm, "%s: null argument", name);
  NV_REQUIRE(K >= 2 && K <= BEAM_MAX && n_groups >= 2 && n_groups <= K && K % n_groups == 0 && group >= 0 && group < n_groups &&
             G > 0 && B >= 0, "%s: bad sizes (B=%d K=%d groups=%d group=%d G=%d)", name, B, K, n_groups, group, G);
  if (B == 0) return NV_OK;
  const BeamSelGroup gr{group, K / n_groups, group == n_groups - 1 ? 1 : 0};
  if (par_hist)
    NV_CUDA(launch_pdl(beam_select_group_scores_kernel, dim3(B), dim3(BS_THREADS), 0, S_(stream), cand_score, cand_tok, cand_parent,
                       beam_score, hist, src, hyp_score, hyp_meta, hyp_tok, prompt_state, next_ids, lens, norm, K, G, eos_id, pad_id,
                       early_stopping, BeamTrace{par_hist, hyp_par, done_step}, gr));
  else
    NV_CUDA(launch_pdl(beam_select_group_kernel, dim3(B), dim3(BS_THREADS), 0, S_(stream), cand_score, cand_tok, cand_parent,
                       beam_score, hist, src, hyp_score, hyp_meta, hyp_tok, prompt_state, next_ids, lens, norm, K, G, eos_id, pad_id,
                       early_stopping, gr));
  return NV_OK;
}

int nv_beam_select_group(const float* cand_score, const int* cand_tok, const int* cand_parent, float* beam_score, int* hist, int* src,
                         double* hyp_score, int* hyp_meta, int* hyp_tok, int* prompt_state, int* next_ids, int* lens,
                         const double* norm, int group, int n_groups, int B, int K, int G, int eos_id, int pad_id, int early_stopping,
                         void* stream) {
  return beam_select_group("nv_beam_select_group", cand_score, cand_tok, cand_parent, beam_score, hist, src, hyp_score, hyp_meta,
                           hyp_tok, prompt_state, next_ids, lens, norm, nullptr, nullptr, nullptr, group, n_groups, B, K, G, eos_id,
                           pad_id, early_stopping, stream);
}

int nv_beam_select_group_scores(const float* cand_score, const int* cand_tok, const int* cand_parent, float* beam_score, int* hist,
                                int* src, double* hyp_score, int* hyp_meta, int* hyp_tok, int* prompt_state, int* next_ids, int* lens,
                                const double* norm, int* par_hist, int* hyp_par, int* done_step, int group, int n_groups, int B, int K,
                                int G, int eos_id, int pad_id, int early_stopping, void* stream) {
  NV_REQUIRE(par_hist && hyp_par && done_step, "nv_beam_select_group_scores: null argument");
  return beam_select_group("nv_beam_select_group_scores", cand_score, cand_tok, cand_parent, beam_score, hist, src, hyp_score,
                           hyp_meta, hyp_tok, prompt_state, next_ids, lens, norm, par_hist, hyp_par, done_step, group, n_groups, B, K,
                           G, eos_id, pad_id, early_stopping, stream);
}

// nv_decode_attn_rope for R = B * K beam rows over a prompt cache shared by the K beams of a prompt and a generated cache
// addressed through src (see BeamKV).
int nv_decode_attn_rope_beam(const void* qkv, int64_t ld, const int* lens, const void* cos_t, const void* sin_t, const void* pk,
                             const void* pv, int Sp, const int* plens, void* kgen, void* vgen, const int* src, int G, void* out,
                             int64_t ldo, int R, int K, int H, int head_dim, float scale, void* stream) {
  NV_REQUIRE(head_dim == 128 && (ld & 7) == 0, "nv_decode_attn_rope_beam: head_dim must be 128, ld %% 8 == 0");
  NV_REQUIRE(R >= 0 && K >= 1 && R % K == 0 && Sp > 0 && G > 0 && H > 0, "nv_decode_attn_rope_beam: bad sizes (R=%d K=%d Sp=%d G=%d H=%d)",
             R, K, Sp, G, H);
  if (R == 0) return NV_OK;
  NV_REQUIRE(qkv && lens && cos_t && sin_t && pk && pv && plens && kgen && vgen && src && out, "nv_decode_attn_rope_beam: null argument");
  const BeamKV<false> bk{CBF(pk), CBF(pv), nullptr, nullptr, src, plens, K, Sp};
  NV_CUDA(launch_pdl(decode_attn_kernel<true, false, true>, dim3(R * H), dim3(DA_WARPS * 32), 0, S_(stream), CBF(qkv), ld, BF(kgen),
                     BF(vgen), lens, BF(out), ldo, G, H, scale, CBF(cos_t), CBF(sin_t), (int8_t*)nullptr, (int8_t*)nullptr, bk));
  return NV_OK;
}

int nv_decode_attn_rope_beam_fp8(const void* qkv, int64_t ld, const int* lens, const void* cos_t, const void* sin_t, const void* pkq,
                                 const void* pvq, const void* pkexp, const void* pvexp, int Sp, const int* plens, void* kq, void* vq,
                                 void* kexp, void* vexp, const int* src, int G, void* out, int64_t ldo, int R, int K, int H,
                                 int head_dim, float scale, void* stream) {
  NV_REQUIRE(head_dim == 128 && (ld & 7) == 0, "nv_decode_attn_rope_beam_fp8: head_dim must be 128, ld %% 8 == 0");
  NV_REQUIRE(R >= 0 && K >= 1 && R % K == 0 && Sp > 0 && G > 0 && H > 0,
             "nv_decode_attn_rope_beam_fp8: bad sizes (R=%d K=%d Sp=%d G=%d H=%d)", R, K, Sp, G, H);
  if (R == 0) return NV_OK;
  NV_REQUIRE(qkv && lens && cos_t && sin_t && pkq && pvq && pkexp && pvexp && plens && kq && vq && kexp && vexp && src && out,
             "nv_decode_attn_rope_beam_fp8: null argument");
  NV_REQUIRE(((uintptr_t)qkv & 15) == 0 && ((uintptr_t)kq & 7) == 0 && ((uintptr_t)vq & 7) == 0 && ((uintptr_t)pkq & 7) == 0 &&
             ((uintptr_t)pvq & 7) == 0, "nv_decode_attn_rope_beam_fp8: alignment (16-byte qkv, 8-byte caches)");
  const BeamKV<true> bk{reinterpret_cast<const uint8_t*>(pkq), reinterpret_cast<const uint8_t*>(pvq),
                        reinterpret_cast<const int8_t*>(pkexp), reinterpret_cast<const int8_t*>(pvexp), src, plens, K, Sp};
  NV_CUDA(launch_pdl(decode_attn_kernel<true, true, true>, dim3(R * H), dim3(DA_WARPS * 32), 0, S_(stream), CBF(qkv), ld,
                     reinterpret_cast<uint8_t*>(kq), reinterpret_cast<uint8_t*>(vq), lens, BF(out), ldo, G, H, scale, CBF(cos_t),
                     CBF(sin_t), reinterpret_cast<int8_t*>(kexp), reinterpret_cast<int8_t*>(vexp), bk));
  return NV_OK;
}

int nv_add_int(int* x, int n, int delta, void* stream) {
  if (n == 0) return NV_OK;
  NV_CUDA(launch_pdl(add_int_kernel, dim3((n + 255) / 256), dim3(256), 0, S_(stream), x, n, delta));
  return NV_OK;
}

// Contrastive search (see contrastive_topk_kernel .. contrastive_commit_kernel).
int nv_contrastive_topk(const void* logits, int64_t ld, int V, const int* special, int n_special, int K, void* p, int* tok, int B,
                        void* stream) {
  NV_REQUIRE(logits && p && tok && B >= 0 && ld >= V, "nv_contrastive_topk: bad arguments (B=%d V=%d)", B, V);
  NV_REQUIRE(K >= 1 && K <= CT_KMAX && K <= V, "nv_contrastive_topk: top_k=%d: 1..%d candidates (and <= V) supported", K, CT_KMAX);
  NV_REQUIRE(V > 0 && V <= (1 << 17) && (int64_t)V * 4 <= 200 * 1024, "nv_contrastive_topk: vocabulary of %d not supported", V);
  NV_REQUIRE(n_special >= 0 && n_special <= MAX_SPECIAL && (n_special == 0 || special),
             "nv_contrastive_topk: n_special=%d out of range (max %d)", n_special, MAX_SPECIAL);
  if (B == 0) return NV_OK;
  static bool attr_set = false;
  if (!attr_set) {
    NV_CUDA(cudaFuncSetAttribute(contrastive_topk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr_set = true;
  }
  NV_CUDA(launch_pdl(contrastive_topk_kernel, dim3(B), dim3(CT_THREADS), (size_t)V * 4, S_(stream), CBF(logits), ld, V, special,
                     n_special, K, BF(p), tok));
  return NV_OK;
}

int nv_contrastive_context(const void* hn, const int* cu_seqlens, int B, int T, void* ctx, int* ctx_len, int Sc, int D, void* stream) {
  NV_REQUIRE(hn && cu_seqlens && ctx && ctx_len && B >= 1 && T >= 0 && Sc > 0 && D > 0 && (D & 7) == 0,
             "nv_contrastive_context: bad arguments (B=%d T=%d Sc=%d D=%d; D %% 8 == 0)", B, T, Sc, D);
  if (T == 0) return NV_OK;
  NV_CUDA(launch_pdl(contrastive_context_kernel, dim3((T + 7) / 8), dim3(256), 0, S_(stream), CBF(hn), cu_seqlens, B, T, BF(ctx),
                     ctx_len, Sc, D));
  return NV_OK;
}

int nv_contrastive_rank(const void* hn, void* ctx, int* ctx_len, int Sc, int D, int K, unsigned* pen_key, const void* p,
                        const int* tok, double alpha, int* finished, int eos_id, int pad_id, int stop_on_eos, int* next, int* sel,
                        void* hsel, int* plens, int* lens, float* pen_out, float* score_out, int B, void* stream) {
  NV_REQUIRE(hn && ctx && ctx_len && pen_key && p && tok && finished && next && sel && hsel && plens && lens && B >= 0,
             "nv_contrastive_rank: null argument");
  NV_REQUIRE(K >= 1 && K <= CT_KMAX && Sc > 0 && D > 0 && (D & 7) == 0 && D <= 8192,
             "nv_contrastive_rank: bad sizes (K=%d Sc=%d D=%d; K <= %d, D %% 8 == 0, D <= 8192)", K, Sc, D, CT_KMAX);
  NV_REQUIRE(alpha == alpha && alpha - alpha == 0.0, "nv_contrastive_rank: penalty_alpha must be finite");
  if (B == 0) return NV_OK;
  const size_t smem = (size_t)CR_CHUNK * D * 2;
  static size_t smem_set = 48 * 1024;
  if (smem > smem_set) {
    NV_CUDA(cudaFuncSetAttribute(contrastive_pen_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    smem_set = smem;
  }
  NV_CUDA(launch_pdl(contrastive_pen_kernel, dim3(CR_SPLIT, B), dim3(CR_THREADS), smem, S_(stream), CBF(hn), CBF(ctx), ctx_len, Sc,
                     D, K, pen_key));
  // 4.28 multiplies the bf16 tensors by the Python floats 1 - alpha and alpha, which take the fp32 opmath type
  NV_CUDA(launch_pdl(contrastive_select_kernel, dim3(B), dim3(CS_THREADS), 0, S_(stream), CBF(hn), BF(ctx), ctx_len, Sc, D, K, pen_key,
                     CBF(p), tok, (float)(1.0 - alpha), (float)alpha, finished, eos_id, pad_id, stop_on_eos, next, sel, BF(hsel),
                     plens, lens, pen_out, score_out));
  return NV_OK;
}

int nv_contrastive_commit(const unsigned long long* table, int L, const int* sel, const int* plens, int K, int Sp, int D, int H,
                          int fp8, int B, void* stream) {
  NV_REQUIRE(table && sel && plens && L >= 1 && K >= 1 && Sp > 0 && H > 0 && D == H * 128 && B >= 0,
             "nv_contrastive_commit: bad arguments (L=%d K=%d Sp=%d D=%d H=%d)", L, K, Sp, D, H);
  if (B == 0) return NV_OK;
  NV_CUDA(launch_pdl(contrastive_commit_kernel, dim3(L, B), dim3(256), 0, S_(stream), table, sel, plens, K, Sp, fp8 ? D : 2 * D,
                     fp8 ? H : 0));
  return NV_OK;
}

}  // extern "C"
