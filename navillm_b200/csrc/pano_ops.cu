// navillm_b200 — fp32 kernels of the panorama scene encoder and the navigation fusion glue (fwd + bwd).
//
// The reference keeps this part in fp32 (SURVEY.md Appendix A.6): ImageEmbeddings
// (models/image_embedding.py:51-121: img/loc projections + LayerNorms + nav-type embedding), the 2-layer
// pre-LN DETR encoder (models/detr_transformer.py:170-182: nn.MultiheadAttention with key-padding mask,
// Linear-GELU-Linear), the mapper, and NavModel's position/step/type embeddings and candidate fusion
// (models/nav_model.py:146-224).  It is ~2.2 GFLOP per panorama -- 0.02 % of a step -- so these kernels
// are written for exact-fp32 parity and low launch count, not for tensor cores: bf16/tf32 MMA would
// change the numerics of a part the reference computes in fp32.
//
// Everything is row-major fp32 with explicit leading dimensions.
#include "nv_common.cuh"
#include "nv_host.h"

namespace nv {

// ------------------------------------------------------------------------------------------------
// SGEMM  C[M,N] (+)= op(A)[M,K] * op(B)[K,N] (+ bias[N]),   64x64 tile, 16-deep, 4x4 per thread.
//   ta = 0: A stored [M,K];  ta = 1: A stored [K,M].   tb = 0: B stored [N,K] (nn.Linear weight);
//   tb = 1: B stored [K,N].
// ------------------------------------------------------------------------------------------------
constexpr int SG_BM = 64, SG_BN = 64, SG_BK = 16;
enum { SG_ACCUM = 1 };

// blockIdx.z = K split: each split handles a contiguous k range.  The splits of a tile form one thread-block cluster
// and add their partial tiles in rank order in the leader's shared memory, so the sum does not depend on timing.
__global__ void __launch_bounds__(256) sgemm_kernel(const float* __restrict__ A, int64_t lda, int ta,
                                                    const float* __restrict__ B, int64_t ldb, int tb,
                                                    float* __restrict__ C, int64_t ldc, const float* __restrict__ bias,
                                                    int M, int N, int K, int flags, int k_per_split) {
  __shared__ float As[SG_BK][SG_BM + 4];
  __shared__ float Bs[SG_BK][SG_BN + 4];
  __shared__ float red[16 * 256];                // split-K: the leader's running sum of the splits' partial tiles
  const int tid = threadIdx.x;
  const int m0 = blockIdx.y * SG_BM, n0 = blockIdx.x * SG_BN;
  const int tx = tid & 15, ty = tid >> 4;  // 16 x 16 threads, each 4x4 outputs
  float acc[4][4] = {};
  const int k_begin = blockIdx.z * k_per_split;
  const int k_end = min(K, k_begin + k_per_split);
  for (int k0 = k_begin; k0 < k_end; k0 += SG_BK) {
    // load A tile (64 x 16) and B tile (16 x 64): 1024 elements each, 4 per thread
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int e = tid + i * 256;
      {
        // choose the index order that makes consecutive threads touch consecutive addresses
        const int mm = ta ? (e & 63) : (e >> 4), kk = ta ? (e >> 6) : (e & 15);
        const int gm = m0 + mm, gk = k0 + kk;
        float v = 0.f;
        if (gm < M && gk < k_end) v = ta ? A[(int64_t)gk * lda + gm] : A[(int64_t)gm * lda + gk];
        As[kk][mm] = v;
      }
      {
        const int nn = tb ? (e & 63) : (e >> 4), kk = tb ? (e >> 6) : (e & 15);
        const int gn = n0 + nn, gk = k0 + kk;
        float v = 0.f;
        if (gn < N && gk < k_end) v = tb ? B[(int64_t)gk * ldb + gn] : B[(int64_t)gn * ldb + gk];
        Bs[kk][nn] = v;
      }
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < SG_BK; ++kk) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = As[kk][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = Bs[kk][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
  if (gridDim.z > 1) {                           // cluster (1, 1, splits): the rank is the split index
    const uint32_t rank = blockIdx.z, base = smem_u32(red) + tid * 4;
    if (rank == 0) {
#pragma unroll
      for (int i = 0; i < 16; ++i) red[i * 256 + tid] = acc[i >> 2][i & 3];
    }
    cluster_sync_all();
    for (uint32_t r = 1; r < gridDim.z; ++r) {
      if (rank == r) {
#pragma unroll
        for (int i = 0; i < 16; ++i) dsmem_add_f32(base + i * 256 * 4, 0, acc[i >> 2][i & 3]);
      }
      cluster_sync_all();
    }
    if (rank != 0) return;
#pragma unroll
    for (int i = 0; i < 16; ++i) acc[i >> 2][i & 3] = red[i * 256 + tid];
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int gm = m0 + ty * 4 + i;
    if (gm >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int gn = n0 + tx * 4 + j;
      if (gn >= N) continue;
      float v = acc[i][j];
      if (bias) v += bias[gn];
      float* c = C + (int64_t)gm * ldc + gn;
      if (flags & SG_ACCUM) v += *c;
      *c = v;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// LayerNorm (affine), one CTA per row:  y = (x - mean) * rstd * gamma + beta  [+ addend]
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float block_sum_f(float v, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = blockDim.x >> 5;
  __syncthreads();
  if (l == 0) red[w] = v;
  __syncthreads();
  float t = (l < nw) ? red[l] : 0.f;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
  return t;
}

__global__ void __launch_bounds__(256) layernorm_fwd_kernel(const float* __restrict__ x, int64_t ldx,
                                                            const float* __restrict__ gamma,
                                                            const float* __restrict__ beta,
                                                            const float* __restrict__ addend, int64_t ldadd,
                                                            float* __restrict__ y, int64_t ldy, float* __restrict__ mean,
                                                            float* __restrict__ rstd, int D, float eps) {
  __shared__ float red[33];
  const int r = blockIdx.x;
  const float* xr = x + (int64_t)r * ldx;
  float s = 0.f;
  for (int i = threadIdx.x; i < D; i += blockDim.x) s += xr[i];
  const float mu = block_sum_f(s, red) / D;
  float v = 0.f;
  for (int i = threadIdx.x; i < D; i += blockDim.x) { const float d = xr[i] - mu; v += d * d; }
  const float rs = rsqrtf(block_sum_f(v, red) / D + eps);
  if (threadIdx.x == 0) { if (mean) mean[r] = mu; if (rstd) rstd[r] = rs; }
  for (int i = threadIdx.x; i < D; i += blockDim.x) {
    float o = (xr[i] - mu) * rs * gamma[i] + beta[i];
    if (addend) o += addend[(int64_t)r * ldadd + i];
    y[(int64_t)r * ldy + i] = o;
  }
}

// dx = rstd * (g - mean(g) - xhat * mean(g * xhat)),  g = dy * gamma ;  partial dgamma/dbeta per CTA.
// Persistent CTAs over rows; partials [grid, 2, D] reduced by colsum2_kernel.
__global__ void __launch_bounds__(256) layernorm_bwd_kernel(const float* __restrict__ x, int64_t ldx,
                                                            const float* __restrict__ gamma,
                                                            const float* __restrict__ mean,
                                                            const float* __restrict__ rstd,
                                                            const float* __restrict__ dy, int64_t lddy,
                                                            float* __restrict__ dx, int64_t lddx, int accumulate_dx,
                                                            float* __restrict__ partial, int R, int D) {
  __shared__ float red[33];
  extern __shared__ float acc[];  // [2][D] per CTA
  for (int i = threadIdx.x; i < 2 * D; i += blockDim.x) acc[i] = 0.f;
  __syncthreads();
  for (int r = blockIdx.x; r < R; r += gridDim.x) {
    const float* xr = x + (int64_t)r * ldx;
    const float* dr = dy + (int64_t)r * lddy;
    const float mu = mean[r], rs = rstd[r];
    float s1 = 0.f, s2 = 0.f;
    for (int i = threadIdx.x; i < D; i += blockDim.x) {
      const float xh = (xr[i] - mu) * rs, g = dr[i] * gamma[i];
      s1 += g; s2 += g * xh;
      acc[i] += dr[i] * xh;       // each column is owned by one thread: no race
      acc[D + i] += dr[i];
    }
    s1 = block_sum_f(s1, red) / D;
    s2 = block_sum_f(s2, red) / D;
    for (int i = threadIdx.x; i < D; i += blockDim.x) {
      const float xh = (xr[i] - mu) * rs, g = dr[i] * gamma[i];
      const float o = rs * (g - s1 - xh * s2);
      float* d = dx + (int64_t)r * lddx + i;
      *d = accumulate_dx ? (*d + o) : o;
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 2 * D; i += blockDim.x) partial[(int64_t)blockIdx.x * 2 * D + i] = acc[i];
}

// dst[j] (+)= sum_p src[p*stride + j]     block = 32 columns x 8 row groups, fixed summation order
__global__ void __launch_bounds__(256) colsum_f32_kernel(const float* __restrict__ src, int64_t stride, int P, int D,
                                                         float* __restrict__ dst, int accumulate) {
  __shared__ float red[8][33];
  const int j = blockIdx.x * 32 + threadIdx.x;
  float s = 0.f;
  if (j < D)
    for (int p = threadIdx.y; p < P; p += 8) s += src[(int64_t)p * stride + j];
  red[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0 && j < D) {
#pragma unroll
    for (int y = 1; y < 8; ++y) s += red[y][threadIdx.x];
    dst[j] = accumulate ? dst[j] + s : s;
  }
}

// ------------------------------------------------------------------------------------------------
// GELU (erf form, torch default) fwd / bwd
// ------------------------------------------------------------------------------------------------
__global__ void gelu_fwd_kernel(const float* __restrict__ z, float* __restrict__ a, int64_t n) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float v = z[i];
    a[i] = 0.5f * v * (1.f + erff(v * 0.70710678118654752f));
  }
}
__global__ void gelu_bwd_kernel(const float* __restrict__ z, const float* __restrict__ da, float* __restrict__ dz,
                                int64_t n) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float v = z[i];
    const float cdf = 0.5f * (1.f + erff(v * 0.70710678118654752f));
    const float pdf = 0.3989422804014327f * expf(-0.5f * v * v);
    dz[i] = da[i] * (cdf + v * pdf);
  }
}

// ------------------------------------------------------------------------------------------------
// Dropout (train mode only; reference: nn.Dropout(hidden_dropout_prob) in models/image_embedding.py:41,72 and
// dropout / dropout1 / dropout2 + the attention-probability dropout of nn.MultiheadAttention in
// models/detr_transformer.py:136-146,170-182).  Stateless counter-based RNG: the keep decision of element idx is a
// hash of (seed, idx), so the backward regenerates the forward's mask from the seed instead of storing it.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t rng_u32(uint64_t seed, uint64_t idx) {   // splitmix64 finaliser
  uint64_t z = seed + (idx + 1) * 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z ^= z >> 31;
  return (uint32_t)(z >> 32);
}
__device__ __forceinline__ bool rng_keep(uint64_t seed, uint64_t idx, uint32_t thresh) { return rng_u32(seed, idx) >= thresh; }

// out[i] = keep(i) ? x[i] / (1 - p) : 0      (forward on activations, backward on gradients: same seed)
__global__ void dropout_kernel(const float* __restrict__ x, float* __restrict__ out, int64_t n, uint32_t thresh,
                               float inv_keep, uint64_t seed) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = rng_keep(seed, (uint64_t)i, thresh) ? x[i] * inv_keep : 0.f;
}

// ------------------------------------------------------------------------------------------------
// Small multi-head self-attention with key-padding mask (N <= 256 keys, head_dim <= 128), fp32.
// qkv: [B, N, 3E] (q | k | v), out: [B, N, E].  One warp per (b, h, query i); probabilities P[b,h,i,:]
// optionally stored (scratch) for the backward.  Padded query rows (i >= len) produce zeros.
// ------------------------------------------------------------------------------------------------
constexpr int MHA_MAXN = 256;

// Attention-probability dropout (Pd != null): Pd = P * keep / (1 - p) is what multiplies V; P (pre-dropout) is
// still stored for the softmax backward.
__global__ void __launch_bounds__(128) mha_fwd_kernel(const float* __restrict__ qkv, const int* __restrict__ lens,
                                                      float* __restrict__ out, float* __restrict__ P, int B, int N,
                                                      int H, int hd, float scale, float* __restrict__ Pd, uint32_t thresh,
                                                      float inv_keep, uint64_t seed) {
  __shared__ float sc[4][MHA_MAXN];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t gw = (int64_t)blockIdx.x * 4 + w;
  if (gw >= (int64_t)B * H * N) return;
  const int i = gw % N, h = (gw / N) % H, b = gw / ((int64_t)N * H);
  const int E = H * hd, len = lens[b];
  float* o = out + ((int64_t)b * N + i) * E + h * hd;
  float* prow = P ? P + (((int64_t)b * H + h) * N + i) * N : nullptr;
  float* pdrow = Pd ? Pd + (((int64_t)b * H + h) * N + i) * N : nullptr;
  if (i >= len) {
    for (int d = lane; d < hd; d += 32) o[d] = 0.f;
    if (prow) for (int j = lane; j < N; j += 32) prow[j] = 0.f;
    if (pdrow) for (int j = lane; j < N; j += 32) pdrow[j] = 0.f;
    return;
  }
  const float* q = qkv + ((int64_t)b * N + i) * 3 * E + h * hd;
  float qr[4];
#pragma unroll
  for (int t = 0; t < 4; ++t) qr[t] = (lane + 32 * t < hd) ? q[lane + 32 * t] * scale : 0.f;
  float mx = -INFINITY;
  for (int j = 0; j < len; ++j) {
    const float* k = qkv + ((int64_t)b * N + j) * 3 * E + E + h * hd;
    float p = 0.f;
#pragma unroll
    for (int t = 0; t < 4; ++t) if (lane + 32 * t < hd) p += qr[t] * k[lane + 32 * t];
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) p += __shfl_xor_sync(0xffffffffu, p, off);
    if (lane == 0) sc[w][j] = p;
    mx = fmaxf(mx, p);
  }
  __syncwarp();
  float sum = 0.f;
  for (int j = lane; j < len; j += 32) { const float e = expf(sc[w][j] - mx); sc[w][j] = e; sum += e; }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, off);
  const float inv = 1.f / sum;
  __syncwarp();
  if (prow) for (int j = lane; j < N; j += 32) prow[j] = (j < len) ? sc[w][j] * inv : 0.f;
  if (pdrow) {                                             // dropped probabilities replace sc for the P·V product
    const uint64_t base = (((uint64_t)b * H + h) * N + i) * (uint64_t)N;
    for (int j = lane; j < len; j += 32) sc[w][j] = rng_keep(seed, base + j, thresh) ? sc[w][j] * inv_keep : 0.f;
    __syncwarp();
    for (int j = lane; j < N; j += 32) pdrow[j] = (j < len) ? sc[w][j] * inv : 0.f;
  }
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int j = 0; j < len; ++j) {
    const float p = sc[w][j] * inv;
    const float* v = qkv + ((int64_t)b * N + j) * 3 * E + 2 * E + h * hd;
#pragma unroll
    for (int t = 0; t < 4; ++t) if (lane + 32 * t < hd) acc[t] += p * v[lane + 32 * t];
  }
#pragma unroll
  for (int t = 0; t < 4; ++t) if (lane + 32 * t < hd) o[lane + 32 * t] = acc[t];
}

// Backward pass A: per (b,h,i): dP_ij = dO_i . V_j ; dS_ij = P_ij (dP_ij - sum_j P_ij dP_ij) ; dQ_i = scale sum_j dS_ij K_j.
// Overwrites nothing of P; writes dS to scratch (same shape as P).  With attention dropout Pd = P * m/(1-p) the
// gradient reaching P is g_ij * m/(1-p) (g = dO_i . V_j), so dS_ij = Pd_ij g_ij - P_ij sum_j Pd_ij g_ij (Pd == P without).
__global__ void __launch_bounds__(128) mha_bwd_a_kernel(const float* __restrict__ qkv, const float* __restrict__ dout,
                                                        const float* __restrict__ P, float* __restrict__ dS,
                                                        float* __restrict__ dqkv, const int* __restrict__ lens, int B,
                                                        int N, int H, int hd, float scale, const float* __restrict__ Pd) {
  __shared__ float sd[4][MHA_MAXN];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t gw = (int64_t)blockIdx.x * 4 + w;
  if (gw >= (int64_t)B * H * N) return;
  const int i = gw % N, h = (gw / N) % H, b = gw / ((int64_t)N * H);
  const int E = H * hd, len = lens[b];
  float* dq = dqkv + ((int64_t)b * N + i) * 3 * E + h * hd;
  float* dsrow = dS + (((int64_t)b * H + h) * N + i) * N;
  const float* prow = P + (((int64_t)b * H + h) * N + i) * N;
  const float* pdrow = Pd ? Pd + (((int64_t)b * H + h) * N + i) * N : prow;
  if (i >= len) {
    for (int d = lane; d < hd; d += 32) dq[d] = 0.f;
    for (int j = lane; j < N; j += 32) dsrow[j] = 0.f;
    return;
  }
  const float* go = dout + ((int64_t)b * N + i) * E + h * hd;
  float gr[4];
#pragma unroll
  for (int t = 0; t < 4; ++t) gr[t] = (lane + 32 * t < hd) ? go[lane + 32 * t] : 0.f;
  float dot = 0.f;
  for (int j = 0; j < len; ++j) {
    const float* v = qkv + ((int64_t)b * N + j) * 3 * E + 2 * E + h * hd;
    float p = 0.f;
#pragma unroll
    for (int t = 0; t < 4; ++t) if (lane + 32 * t < hd) p += gr[t] * v[lane + 32 * t];
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) p += __shfl_xor_sync(0xffffffffu, p, off);
    if (lane == 0) sd[w][j] = p;
    dot += pdrow[j] * p;
  }
  __syncwarp();
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int j = 0; j < len; ++j) {
    const float ds = pdrow[j] * sd[w][j] - prow[j] * dot;
    if (lane == 0) dsrow[j] = ds;
    const float* k = qkv + ((int64_t)b * N + j) * 3 * E + E + h * hd;
#pragma unroll
    for (int t = 0; t < 4; ++t) if (lane + 32 * t < hd) acc[t] += ds * k[lane + 32 * t];
  }
  for (int j = len + lane; j < N; j += 32) dsrow[j] = 0.f;
#pragma unroll
  for (int t = 0; t < 4; ++t) if (lane + 32 * t < hd) dq[lane + 32 * t] = acc[t] * scale;
}

// Backward pass B: per (b,h,j): dK_j = scale sum_i dS_ij Q_i ; dV_j = sum_i P_ij dO_i.
__global__ void __launch_bounds__(128) mha_bwd_b_kernel(const float* __restrict__ qkv, const float* __restrict__ dout,
                                                        const float* __restrict__ P, const float* __restrict__ dS,
                                                        float* __restrict__ dqkv, const int* __restrict__ lens, int B,
                                                        int N, int H, int hd, float scale) {
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t gw = (int64_t)blockIdx.x * 4 + w;
  if (gw >= (int64_t)B * H * N) return;
  const int j = gw % N, h = (gw / N) % H, b = gw / ((int64_t)N * H);
  const int E = H * hd, len = lens[b];
  float* dk = dqkv + ((int64_t)b * N + j) * 3 * E + E + h * hd;
  float* dv = dqkv + ((int64_t)b * N + j) * 3 * E + 2 * E + h * hd;
  float ak[4] = {0.f, 0.f, 0.f, 0.f}, av[4] = {0.f, 0.f, 0.f, 0.f};
  if (j < len) {
    const float* pb = P + (((int64_t)b * H + h) * N) * N + j;
    const float* sb = dS + (((int64_t)b * H + h) * N) * N + j;
    for (int i = 0; i < len; ++i) {
      const float p = pb[(int64_t)i * N], ds = sb[(int64_t)i * N];
      const float* q = qkv + ((int64_t)b * N + i) * 3 * E + h * hd;
      const float* go = dout + ((int64_t)b * N + i) * E + h * hd;
#pragma unroll
      for (int t = 0; t < 4; ++t)
        if (lane + 32 * t < hd) { ak[t] += ds * q[lane + 32 * t]; av[t] += p * go[lane + 32 * t]; }
    }
  }
#pragma unroll
  for (int t = 0; t < 4; ++t)
    if (lane + 32 * t < hd) { dk[lane + 32 * t] = ak[t] * scale; dv[lane + 32 * t] = av[t]; }
}

// ------------------------------------------------------------------------------------------------
// Row combine:  out[r] = (accumulate ? out[r] : 0) + alpha * A[ia[r]] + beta * Bm[ib[r]]
// An index < 0 contributes nothing; ia == null means identity (row r).  Covers embedding lookups,
// masked fills (index -1), candidate fusion and permuted gathers (models/nav_model.py:146-224).
// rows_scatter_add is its transpose for gradients: a thread owns one column and walks the source rows in order, so
// rows landing on the same destination row are summed in a fixed order (no atomics).
// ------------------------------------------------------------------------------------------------
__global__ void rows_combine_kernel(float* __restrict__ out, int64_t ldo, const float* __restrict__ A, int64_t lda,
                                    const int* __restrict__ ia, float alpha, const float* __restrict__ Bm, int64_t ldb,
                                    const int* __restrict__ ib, float beta, int R, int D, int accumulate) {
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < (int64_t)R * D;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int r = idx / D, c = idx % D;
    float v = accumulate ? out[(int64_t)r * ldo + c] : 0.f;
    if (A) { const int s = ia ? ia[r] : r; if (s >= 0) v += alpha * A[(int64_t)s * lda + c]; }
    if (Bm) { const int s = ib ? ib[r] : r; if (s >= 0) v += beta * Bm[(int64_t)s * ldb + c]; }
    out[(int64_t)r * ldo + c] = v;
  }
}
__global__ void rows_scatter_add_kernel(float* __restrict__ dst, int64_t ldd, const int* __restrict__ idx,
                                        const float* __restrict__ src, int64_t lds, float alpha, int R, int D) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= D) return;
  constexpr int U = 8;                           // source rows whose loads are in flight together
  for (int r0 = 0; r0 < R; r0 += U) {
    int s[U];
    float v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int r = r0 + u;
      s[u] = r < R ? (idx ? idx[r] : r) : -1;
      v[u] = s[u] >= 0 ? src[(int64_t)r * lds + c] : 0.f;
    }
#pragma unroll
    for (int u = 0; u < U; ++u)
      if (s[u] >= 0) dst[(int64_t)s[u] * ldd + c] += alpha * v[u];
  }
}

static inline int grid_1d(int64_t work, int block) {
  int64_t g = (work + block - 1) / block;
  const int64_t cap = (int64_t)sm_count() * 16;
  return (int)(g > cap ? cap : (g < 1 ? 1 : g));
}

}  // namespace nv

using namespace nv;
#define S_(x) reinterpret_cast<cudaStream_t>(x)

extern "C" {

int nv_sgemm(const float* A, int64_t lda, int ta, const float* B, int64_t ldb, int tb, float* C, int64_t ldc,
             const float* bias, int M, int N, int K, int accumulate, void* stream) {
  if (M == 0 || N == 0) return NV_OK;
  NV_REQUIRE(M > 0 && N > 0 && K > 0 && A && B && C, "nv_sgemm: bad arguments M=%d N=%d K=%d", M, N, K);
  dim3 grid((N + SG_BN - 1) / SG_BN, (M + SG_BM - 1) / SG_BM, 1);
  // Encoder GEMMs are small (<= a few hundred tiles, K up to 4096): split K until ~3 CTAs per SM are in flight (with
  // g_fixed_splits: as far as K allows, whatever the tile count).
  const int tiles = grid.x * grid.y;
  int splits = 1;
  while (splits < 8 && (g_fixed_splits || tiles * splits < 3 * sm_count()) && K / (splits * 2) >= 256) splits *= 2;
  int k_per_split = ((K + splits - 1) / splits + SG_BK - 1) / SG_BK * SG_BK;
  grid.z = (K + k_per_split - 1) / k_per_split;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = dim3(256);
  cfg.stream = S_(stream);
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;   // the K splits of a tile are one cluster (<= 8 CTAs)
  attr[0].val.clusterDim.x = 1;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = grid.z;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  NV_CUDA(cudaLaunchKernelEx(&cfg, sgemm_kernel, A, lda, ta, B, ldb, tb, C, ldc, bias, M, N, K,
                             accumulate ? (int)SG_ACCUM : 0, k_per_split));
  return NV_OK;
}

int nv_layernorm_fwd(const float* x, int64_t ldx, const float* gamma, const float* beta, const float* addend,
                     int64_t ldadd, float* y, int64_t ldy, float* mean, float* rstd, int R, int D, float eps,
                     void* stream) {
  if (R == 0) return NV_OK;
  layernorm_fwd_kernel<<<R, 256, 0, S_(stream)>>>(x, ldx, gamma, beta, addend, ldadd, y, ldy, mean, rstd, D, eps);
  NV_LAUNCH_CHECK();
  return NV_OK;
}

int nv_layernorm_bwd_partials(void) { return sm_count(); }

// workspace: fp32 [nv_layernorm_bwd_partials() * 2 * D]; dgamma/dbeta accumulated in place.
int nv_layernorm_bwd(const float* x, int64_t ldx, const float* gamma, const float* mean, const float* rstd,
                     const float* dy, int64_t lddy, float* dx, int64_t lddx, int accumulate_dx, float* dgamma,
                     float* dbeta, float* workspace, int R, int D, void* stream) {
  if (R == 0) return NV_OK;
  NV_REQUIRE(2 * D * 4 <= 96 * 1024, "nv_layernorm_bwd: D=%d too large", D);
  int P = sm_count();
  if (P > R) P = R;
  static bool attr = false;
  if (!attr) {
    NV_CUDA(cudaFuncSetAttribute(layernorm_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
    attr = true;
  }
  layernorm_bwd_kernel<<<P, 256, 2 * D * sizeof(float), S_(stream)>>>(x, ldx, gamma, mean, rstd, dy, lddy, dx, lddx,
                                                                     accumulate_dx, workspace, R, D);
  NV_LAUNCH_CHECK();
  if (dgamma) {
    colsum_f32_kernel<<<(D + 31) / 32, dim3(32, 8), 0, S_(stream)>>>(workspace, 2 * D, P, D, dgamma, 1);
    NV_LAUNCH_CHECK();
  }
  if (dbeta) {
    colsum_f32_kernel<<<(D + 31) / 32, dim3(32, 8), 0, S_(stream)>>>(workspace + D, 2 * D, P, D, dbeta, 1);
    NV_LAUNCH_CHECK();
  }
  return NV_OK;
}

int nv_colsum_f32(const float* src, int64_t ld, int R, int D, float* dst, int accumulate, void* stream) {
  if (D == 0) return NV_OK;
  colsum_f32_kernel<<<(D + 31) / 32, dim3(32, 8), 0, S_(stream)>>>(src, ld, R, D, dst, accumulate);
  NV_LAUNCH_CHECK();
  return NV_OK;
}

int nv_gelu_fwd(const float* z, float* a, int64_t n, void* stream) {
  if (n == 0) return NV_OK;
  gelu_fwd_kernel<<<grid_1d(n, 256), 256, 0, S_(stream)>>>(z, a, n);
  NV_LAUNCH_CHECK();
  return NV_OK;
}
int nv_gelu_bwd(const float* z, const float* da, float* dz, int64_t n, void* stream) {
  if (n == 0) return NV_OK;
  gelu_bwd_kernel<<<grid_1d(n, 256), 256, 0, S_(stream)>>>(z, da, dz, n);
  NV_LAUNCH_CHECK();
  return NV_OK;
}

int nv_mha_fwd(const float* qkv, const int* lens, float* out, float* P, int B, int N, int H, int hd, void* stream) {
  NV_REQUIRE(N <= MHA_MAXN && hd <= 128, "nv_mha_fwd: N=%d (max %d) hd=%d (max 128)", N, MHA_MAXN, hd);
  const int64_t warps = (int64_t)B * H * N;
  if (warps == 0) return NV_OK;
  mha_fwd_kernel<<<(unsigned)((warps + 3) / 4), 128, 0, S_(stream)>>>(qkv, lens, out, P, B, N, H, hd, rsqrtf((float)hd),
                                                                      nullptr, 0u, 1.f, 0ull);
  NV_LAUNCH_CHECK();
  return NV_OK;
}

static inline uint32_t drop_thresh(float p) { return (uint32_t)((double)p * 4294967296.0); }

// Train-mode variant with attention-probability dropout: Pd [B,H,N,N] receives the dropped probabilities.
int nv_mha_fwd_dropout(const float* qkv, const int* lens, float* out, float* P, float* Pd, int B, int N, int H, int hd,
                       float p_drop, unsigned long long seed, void* stream) {
  NV_REQUIRE(N <= MHA_MAXN && hd <= 128, "nv_mha_fwd_dropout: N=%d (max %d) hd=%d (max 128)", N, MHA_MAXN, hd);
  NV_REQUIRE(P && Pd && p_drop >= 0.f && p_drop < 1.f, "nv_mha_fwd_dropout: P, Pd required and 0 <= p < 1");
  const int64_t warps = (int64_t)B * H * N;
  if (warps == 0) return NV_OK;
  mha_fwd_kernel<<<(unsigned)((warps + 3) / 4), 128, 0, S_(stream)>>>(qkv, lens, out, P, B, N, H, hd, rsqrtf((float)hd), Pd,
                                                                      drop_thresh(p_drop), 1.f / (1.f - p_drop), seed);
  NV_LAUNCH_CHECK();
  return NV_OK;
}

int nv_dropout(const float* x, float* out, int64_t n, float p_drop, unsigned long long seed, void* stream) {
  if (n == 0) return NV_OK;
  NV_REQUIRE(p_drop >= 0.f && p_drop < 1.f, "nv_dropout: 0 <= p < 1");
  dropout_kernel<<<grid_1d(n, 256), 256, 0, S_(stream)>>>(x, out, n, drop_thresh(p_drop), 1.f / (1.f - p_drop), seed);
  NV_LAUNCH_CHECK();
  return NV_OK;
}

int nv_mha_bwd(const float* qkv, const float* dout, const float* P, float* dS, float* dqkv, const int* lens, int B,
               int N, int H, int hd, void* stream) {
  NV_REQUIRE(N <= MHA_MAXN && hd <= 128, "nv_mha_bwd: N=%d hd=%d", N, hd);
  const int64_t warps = (int64_t)B * H * N;
  if (warps == 0) return NV_OK;
  const float scale = rsqrtf((float)hd);
  mha_bwd_a_kernel<<<(unsigned)((warps + 3) / 4), 128, 0, S_(stream)>>>(qkv, dout, P, dS, dqkv, lens, B, N, H, hd, scale, nullptr);
  NV_LAUNCH_CHECK();
  mha_bwd_b_kernel<<<(unsigned)((warps + 3) / 4), 128, 0, S_(stream)>>>(qkv, dout, P, dS, dqkv, lens, B, N, H, hd, scale);
  NV_LAUNCH_CHECK();
  return NV_OK;
}

// Backward of nv_mha_fwd_dropout: Pd (dropped probabilities) feeds dV and the dropout part of dS.
int nv_mha_bwd_dropout(const float* qkv, const float* dout, const float* P, const float* Pd, float* dS, float* dqkv,
                       const int* lens, int B, int N, int H, int hd, void* stream) {
  NV_REQUIRE(N <= MHA_MAXN && hd <= 128 && P && Pd, "nv_mha_bwd_dropout: N=%d hd=%d", N, hd);
  const int64_t warps = (int64_t)B * H * N;
  if (warps == 0) return NV_OK;
  const float scale = rsqrtf((float)hd);
  mha_bwd_a_kernel<<<(unsigned)((warps + 3) / 4), 128, 0, S_(stream)>>>(qkv, dout, P, dS, dqkv, lens, B, N, H, hd, scale, Pd);
  NV_LAUNCH_CHECK();
  mha_bwd_b_kernel<<<(unsigned)((warps + 3) / 4), 128, 0, S_(stream)>>>(qkv, dout, Pd, dS, dqkv, lens, B, N, H, hd, scale);
  NV_LAUNCH_CHECK();
  return NV_OK;
}

int nv_rows_combine(float* out, int64_t ldo, const float* A, int64_t lda, const int* ia, float alpha, const float* Bm,
                    int64_t ldb, const int* ib, float beta, int R, int D, int accumulate, void* stream) {
  if (R == 0 || D == 0) return NV_OK;
  rows_combine_kernel<<<grid_1d((int64_t)R * D, 256), 256, 0, S_(stream)>>>(out, ldo, A, lda, ia, alpha, Bm, ldb, ib, beta,
                                                                           R, D, accumulate);
  NV_LAUNCH_CHECK();
  return NV_OK;
}

int nv_rows_scatter_add(float* dst, int64_t ldd, const int* idx, const float* src, int64_t lds, float alpha, int R, int D,
                        void* stream) {
  if (R == 0 || D == 0) return NV_OK;
  rows_scatter_add_kernel<<<(D + 127) / 128, 128, 0, S_(stream)>>>(dst, ldd, idx, src, lds, alpha, R, D);
  NV_LAUNCH_CHECK();
  return NV_OK;
}

}  // extern "C"
