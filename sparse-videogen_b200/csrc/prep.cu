// Pre-attention elementwise chain (SURVEY §8f-1): the reference's native `_kernels` ops
//   rms_norm_forward / layer_norm_forward            (svg/kernels/csrc/ops.h:20-75, include/norm/narrow_*.cuh)
//   apply_qk_rope_inplace_cossin{,_txtlast,_complex} (ops.h:77-260, include/rope/rope_enc*.cuh)
// as in-place drop-ins, plus ONE fused pass that replaces the whole reference chain
//   [B,S,H*D] -> unflatten/transpose/contiguous (hyvideo/attention.py:260-266) -> QK norm -> RoPE -> torch.cat
// reading each projection output once and writing Q/K/V once in the [B,H,S,D] layout the attention kernel's
// TMA descriptors read.  All kernels are HBM-bound: 16-byte vectors, a row segment of 8 elements per thread,
// D/8 lanes cooperate on one head row (sub-warp butterfly, same order as the reference's reduction).
//
// Rounding points reproduced from the reference chain: the norm result is rounded to the 16-bit dtype
// (in-place store) before RoPE reads it; RoPE computes in fp32 (fp64 for the `complex` variant,
// rope_enc_complex.cuh:29-43) and rounds once.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <type_traits>

#include "../../include/svgb200.h"
#include "host_common.h"

namespace svgb {

template <bool BF16>
__device__ __forceinline__ void unpack8(const uint4& v, float (&f)[8]) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    if constexpr (BF16) {
      f[2 * i] = __uint_as_float(w[i] << 16);
      f[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
    } else {
      const __half2 h = *reinterpret_cast<const __half2*>(&w[i]);
      f[2 * i] = __low2float(h);
      f[2 * i + 1] = __high2float(h);
    }
  }
}
template <bool BF16>
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  uint32_t w[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    if constexpr (BF16) {
      const __nv_bfloat162 b = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
      w[i] = *reinterpret_cast<const uint32_t*>(&b);
    } else {
      const __half2 h = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
      w[i] = *reinterpret_cast<const uint32_t*>(&h);
    }
  }
  return make_uint4(w[0], w[1], w[2], w[3]);
}
template <bool BF16>
__device__ __forceinline__ float round16f(float x) {
  if constexpr (BF16) return __bfloat162float(__float2bfloat16_rn(x));
  else return __half2float(__float2half_rn(x));
}
template <bool BF16>
__device__ __forceinline__ float round16d(double x) {  // static_cast<T>(double), T the 16-bit type
  if constexpr (BF16) return __bfloat162float(__double2bfloat16(x));
  else return __half2float(__double2half(x));
}

// butterfly over the LPR lanes that share a row (LPR = D/8 is a power of two <= 32)
template <int LPR>
__device__ __forceinline__ float group_sum(float v) {
#pragma unroll
  for (int o = LPR / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---- the three per-row transforms, shared by the in-place kernels and the fused pass -----------
template <int D>
__device__ __forceinline__ void rms_apply(float (&f)[8], const float (&g)[8], float eps) {
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) ss += f[i] * f[i];
  ss = group_sum<D / 8>(ss);
  const float inv = rsqrtf(ss / D + eps);
#pragma unroll
  for (int i = 0; i < 8; ++i) f[i] = f[i] * inv * g[i];
}
template <int D>
__device__ __forceinline__ void ln_apply(float (&f)[8], const float (&g)[8], const float (&b)[8]) {
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) s += f[i];
  const float mean = group_sum<D / 8>(s) / D;
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) ss += (f[i] - mean) * (f[i] - mean);
  const float inv = rsqrtf(group_sum<D / 8>(ss) / D + 1e-5f);
#pragma unroll
  for (int i = 0; i < 8; ++i) f[i] = (f[i] - mean) * inv * g[i] + b[i];
}
// RoPE rotations; kT selects the transpose (the backward; not the inverse rotation: cos / sin need not repeat within
// a pair).
// interleaved pairs (2i, 2i+1): out[e] = x[e]*cos[e] + (e even ? -x[e^1] : x[e^1]) * sin[e]
//   transpose: dx[2i] = dy[2i]*c[2i] + dy[2i+1]*s[2i+1],  dx[2i+1] = dy[2i+1]*c[2i+1] - dy[2i]*s[2i]
template <bool kT>
__device__ __forceinline__ void rope_apply(float (&f)[8], const float (&c)[8], const float (&s)[8]) {
  float o[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) o[i] = f[i] * c[i] + (((i & 1) != 0) != kT ? f[i ^ 1] : -f[i ^ 1]) * s[kT ? i ^ 1 : i];
#pragma unroll
  for (int i = 0; i < 8; ++i) f[i] = o[i];
}
// complex pairs (a, b): a' = a*c - b*s, b' = b*c + a*s (transpose: a' = a*c + b*s, b' = b*c - a*s), in fp64 with
// one rounding
template <bool BF16, bool kT>
__device__ __forceinline__ void rope_apply_complex(float (&f)[8], const float (&c)[4], const float (&s)[4]) {
  float o[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const double x = f[i], y = f[i ^ 1], cc = c[i >> 1], sn = s[i >> 1];
    o[i] = round16d<BF16>(x * cc + (((i & 1) != 0) != kT ? y : -y) * sn);
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) f[i] = o[i];
}

__device__ __forceinline__ void load_f8(const float* p, float (&f)[8]) {
  const float4 a = __ldg(reinterpret_cast<const float4*>(p));
  const float4 b = __ldg(reinterpret_cast<const float4*>(p) + 1);
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w;
  f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}
__device__ __forceinline__ void load_f4(const float* p, float (&f)[4]) {
  const float4 a = __ldg(reinterpret_cast<const float4*>(p));
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w;
}
// this thread's cos / sin of table row `row`: interleaved [n, D] into c8 / s8, complex [n, D/2] into c4 / s4
template <int D>
__device__ __forceinline__ void load_rope_tables(const float* cos_t, const float* sin_t, long long row, int seg,
                                                 bool complex, float (&c8)[8], float (&s8)[8], float (&c4)[4],
                                                 float (&s4)[4]) {
  if (complex) {
    load_f4(cos_t + row * (D / 2) + seg * 4, c4);
    load_f4(sin_t + row * (D / 2) + seg * 4, s4);
  } else {
    load_f8(cos_t + row * D + seg * 8, c8);
    load_f8(sin_t + row * D + seg * 8, s8);
  }
}

constexpr int kThreads = 256;
#ifndef SVGB_PREP_UNROLL
#define SVGB_PREP_UNROLL 4
#endif
constexpr int kUnrollRows = SVGB_PREP_UNROLL;  // independent 16-byte loads in flight per thread

// ---- in-place row norms on [m, N] ---------------------------------------------------------------
template <bool BF16, int N, bool kLayer>
__global__ void __launch_bounds__(kThreads)
row_norm_kernel(uint4* __restrict__ x, const uint4* __restrict__ gamma, const uint4* __restrict__ beta, float eps,
                long long m) {
  constexpr int LPR = N / 8, RPB = kThreads / LPR;
  const int seg = threadIdx.x % LPR, sub = threadIdx.x / LPR;
  float g[8], b[8];
  unpack8<BF16>(__ldg(gamma + seg), g);
  if constexpr (kLayer) unpack8<BF16>(__ldg(beta + seg), b);
  const long long pass = static_cast<long long>(gridDim.x) * RPB;
  for (long long base = static_cast<long long>(blockIdx.x) * RPB; base < m; base += pass * kUnrollRows) {
    uint4 v[kUnrollRows];
#pragma unroll
    for (int u = 0; u < kUnrollRows; ++u) {
      const long long r = base + u * pass + sub;
      v[u] = r < m ? x[r * LPR + seg] : make_uint4(0, 0, 0, 0);
    }
#pragma unroll
    for (int u = 0; u < kUnrollRows; ++u) {
      const long long r = base + u * pass + sub;
      float f[8];
      unpack8<BF16>(v[u], f);
      if constexpr (kLayer) ln_apply<N>(f, g, b);
      else rms_apply<N>(f, g, eps);
      if (r < m) x[r * LPR + seg] = pack8<BF16>(f);
    }
  }
}

// ---- in-place RoPE on q [B,Hq,S,D], k [B,Hk,S,D]; rows [row0, row0+valid) of every head ------------
// qk_rope_bwd_kernel is the same head walk, out of place.  This one keeps its own body and so its instruction stream;
// merged into one kernel with the transpose it took 0.25-0.36% longer at HunyuanVideo 720p (DESIGN.md §5).
template <bool BF16, int D, bool kComplex>
__global__ void __launch_bounds__(kThreads)
qk_rope_kernel(uint4* __restrict__ q, uint4* __restrict__ k, const float* __restrict__ cos_t,
               const float* __restrict__ sin_t, int Hq, int Hk, int S, int row0, int valid) {
  constexpr int LPR = D / 8, RPB = kThreads / LPR;
  const int seg = threadIdx.x % LPR;
  const int t = blockIdx.x * RPB + threadIdx.x / LPR;
  if (t >= valid) return;
  float c8[8], s8[8], c4[4], s4[4];
  load_rope_tables<D>(cos_t, sin_t, t, seg, kComplex, c8, s8, c4, s4);
  const long long hs = static_cast<long long>(S) * LPR;
#pragma unroll 1
  for (int which = 0; which < 2; ++which) {
    const int H = which ? Hk : Hq;
    uint4* p = (which ? k : q) + (static_cast<long long>(blockIdx.y) * H * S + row0 + t) * LPR + seg;
#pragma unroll 1
    for (int h0 = 0; h0 < H; h0 += kUnrollRows) {
      uint4 v[kUnrollRows];
#pragma unroll
      for (int u = 0; u < kUnrollRows; ++u)
        if (h0 + u < H) v[u] = p[(h0 + u) * hs];
#pragma unroll
      for (int u = 0; u < kUnrollRows; ++u) {
        if (h0 + u < H) {
          float f[8];
          unpack8<BF16>(v[u], f);
          if constexpr (kComplex) rope_apply_complex<BF16, false>(f, c4, s4);
          else rope_apply<false>(f, c8, s8);
          p[(h0 + u) * hs] = pack8<BF16>(f);
        }
      }
    }
  }
}

// ---- RoPE backward, out of place: every row of dq [B,Hq,S,D] / dk [B,Hk,S,D]; rows [row0, row0+valid) transposed,
// the others copied
template <bool BF16, int D, bool kComplex>
__global__ void __launch_bounds__(kThreads)
qk_rope_bwd_kernel(const uint4* __restrict__ dq, const uint4* __restrict__ dk, uint4* __restrict__ gq,
                   uint4* __restrict__ gk, const float* __restrict__ cos_t, const float* __restrict__ sin_t, int Hq,
                   int Hk, int S, int row0, int valid) {
  constexpr int LPR = D / 8, RPB = kThreads / LPR;
  const int seg = threadIdx.x % LPR;
  const int t = blockIdx.x * RPB + threadIdx.x / LPR;
  if (t >= S) return;
  const bool rot = t >= row0 && t < row0 + valid;
  float c8[8], s8[8], c4[4], s4[4];
  if (rot) load_rope_tables<D>(cos_t, sin_t, t - row0, seg, kComplex, c8, s8, c4, s4);
  const long long hs = static_cast<long long>(S) * LPR;
#pragma unroll 1
  for (int which = 0; which < 2; ++which) {
    const int H = which ? Hk : Hq;
    const long long o = (static_cast<long long>(blockIdx.y) * H * S + t) * LPR + seg;
    const uint4* src = (which ? dk : dq) + o;
    uint4* dst = (which ? gk : gq) + o;
#pragma unroll 1
    for (int h0 = 0; h0 < H; h0 += kUnrollRows) {
      uint4 v[kUnrollRows];
#pragma unroll
      for (int u = 0; u < kUnrollRows; ++u)
        if (h0 + u < H) v[u] = __ldg(src + (h0 + u) * hs);
#pragma unroll
      for (int u = 0; u < kUnrollRows; ++u) {
        if (h0 + u < H) {
          if (rot) {
            float f[8];
            unpack8<BF16>(v[u], f);
            if constexpr (kComplex) rope_apply_complex<BF16, true>(f, c4, s4);
            else rope_apply<true>(f, c8, s8);
            v[u] = pack8<BF16>(f);
          }
          dst[(h0 + u) * hs] = v[u];
        }
      }
    }
  }
}

// ---- fused transpose + norm + RoPE ----------------------------------------------------------------
// what the fused pass and its backward share: the layout, the norm and the RoPE tables and range
struct PrepGeom {
  const float* cos_t;
  const float* sin_t;
  long long in_token_stride, in_batch_stride, out_head_stride, out_batch_stride;
  int S_in, H, out_row0, norm, rope, rope_lo, rope_n;
  float eps;
};
struct PrepArgs {
  const uint16_t* in[3];   // q, k, v projection outputs [B, S_in, H*D] (token stride / batch stride in geo)
  uint16_t* out[3];        // [B, H, S_out, D]; this call fills rows [out_row0, out_row0 + S_in)
  const uint16_t* gamma[2];
  const uint16_t* beta[2];
  PrepGeom geo;
};

template <bool BF16, int D>
__global__ void __launch_bounds__(kThreads)
qkv_prep_kernel(const PrepArgs a) {
  constexpr int LPR = D / 8, RPB = kThreads / LPR;
  const int seg = threadIdx.x % LPR;
  const int t = blockIdx.x * RPB + threadIdx.x / LPR;
  const int which = blockIdx.z;  // 0 q, 1 k, 2 v
  const bool live = t < a.geo.S_in;
  const int tt = live ? t : a.geo.S_in - 1;  // keep the whole warp in the shuffles; dead lanes never store
  const uint16_t* in = a.in[which] + blockIdx.y * a.geo.in_batch_stride + tt * a.geo.in_token_stride + seg * 8;
  uint16_t* out = a.out[which] + blockIdx.y * a.geo.out_batch_stride + static_cast<long long>(a.geo.out_row0 + tt) * D + seg * 8;
  const int norm = which < 2 ? a.geo.norm : 0;
  const int rp = a.geo.rope;
  const bool rot = which < 2 && rp != 0 && tt >= a.geo.rope_lo && tt < a.geo.rope_lo + a.geo.rope_n;
  float g[8], b[8], c8[8], s8[8], c4[4], s4[4];
  if (norm == 1 || norm == 2) unpack8<BF16>(__ldg(reinterpret_cast<const uint4*>(a.gamma[which]) + seg), g);
  if (norm == 2) unpack8<BF16>(__ldg(reinterpret_cast<const uint4*>(a.beta[which]) + seg), b);
  if (rot) load_rope_tables<D>(a.geo.cos_t, a.geo.sin_t, tt - a.geo.rope_lo, seg, rp == 2, c8, s8, c4, s4);
  float inv_full = 0.f;
  if (norm == 3) {  // RMS over the full hidden row H*D (Wan QK-norm before the head split, wan/attention.py:107-120)
    float ss = 0.f;
#pragma unroll 1
    for (int h0 = 0; h0 < a.geo.H; h0 += kUnrollRows) {
      uint4 v[kUnrollRows];
#pragma unroll
      for (int u = 0; u < kUnrollRows; ++u)
        v[u] = h0 + u < a.geo.H ? *reinterpret_cast<const uint4*>(in + (h0 + u) * D) : make_uint4(0, 0, 0, 0);
#pragma unroll
      for (int u = 0; u < kUnrollRows; ++u) {
        float f[8];
        unpack8<BF16>(v[u], f);
#pragma unroll
        for (int i = 0; i < 8; ++i) ss += f[i] * f[i];
      }
    }
    ss = group_sum<LPR>(ss);
    inv_full = 1.0f / sqrtf(ss / (a.geo.H * D) + a.geo.eps);
  }
#pragma unroll 1
  for (int h0 = 0; h0 < a.geo.H; h0 += kUnrollRows) {
    uint4 v[kUnrollRows];
#pragma unroll
    for (int u = 0; u < kUnrollRows; ++u)
      if (h0 + u < a.geo.H) v[u] = *reinterpret_cast<const uint4*>(in + (h0 + u) * D);
#pragma unroll
    for (int u = 0; u < kUnrollRows; ++u) {
      if (h0 + u < a.geo.H) {  // block-uniform
        if (norm != 0 || rot) {
          float f[8];
          unpack8<BF16>(v[u], f);
          if (norm == 1) rms_apply<D>(f, g, a.geo.eps);
          else if (norm == 2) ln_apply<D>(f, g, b);
          else if (norm == 3) {
            float gw[8];
            unpack8<BF16>(__ldg(reinterpret_cast<const uint4*>(a.gamma[which] + (h0 + u) * D) + seg), gw);
#pragma unroll
            for (int i = 0; i < 8; ++i) f[i] = f[i] * inv_full * gw[i];
          }
          if (rot) {
            if (norm != 0) {
#pragma unroll
              for (int i = 0; i < 8; ++i) f[i] = round16f<BF16>(f[i]);
            }
            if (rp == 2) rope_apply_complex<BF16, false>(f, c4, s4);
            else rope_apply<false>(f, c8, s8);
          }
          v[u] = pack8<BF16>(f);
        }
        if (live) *reinterpret_cast<uint4*>(out + (h0 + u) * a.geo.out_head_stride) = v[u];
      }
    }
  }
}

// ================================= backward (DESIGN.md §5) =====================================================
// Norm backwards on one head row.  x = the saved 16-bit input (f), d = the gradient at the norm output, replaced by
// dx; r and x^ are recomputed exactly as rms_apply / ln_apply compute them.  u = gamma*d:
//   RMS: dx = r*(u - x^*mean(u*x^))          LayerNorm: dx = r*(u - mean(u) - x^*mean(u*x^))
// ag += d*x^ (dgamma), ab += d (dbeta): per-thread fp32 partials of this thread's 8 columns.
// Everything below is pinned bit for bit by tests/test_rowwise_bwd_census_gpu.py (oracle/rowwise_bwd.py).
template <int D>
__device__ __forceinline__ void rms_bwd(const float (&f)[8], float (&d)[8], const float (&g)[8], float eps,
                                        float (&ag)[8]) {
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) ss += f[i] * f[i];
  ss = group_sum<D / 8>(ss);
  const float inv = rsqrtf(ss / D + eps);
  float xh[8], ux = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    xh[i] = f[i] * inv;
    ag[i] += d[i] * xh[i];
    d[i] *= g[i];
    ux += d[i] * xh[i];
  }
  const float m = group_sum<D / 8>(ux) / D;
#pragma unroll
  for (int i = 0; i < 8; ++i) d[i] = inv * (d[i] - xh[i] * m);
}
template <int D>
__device__ __forceinline__ void ln_bwd(const float (&f)[8], float (&d)[8], const float (&g)[8], float (&ag)[8],
                                       float (&ab)[8]) {
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) s += f[i];
  const float mean = group_sum<D / 8>(s) / D;
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) ss += (f[i] - mean) * (f[i] - mean);
  const float inv = rsqrtf(group_sum<D / 8>(ss) / D + 1e-5f);
  float xh[8], su = 0.f, sux = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    xh[i] = (f[i] - mean) * inv;
    ag[i] += d[i] * xh[i];
    ab[i] += d[i];
    d[i] *= g[i];
    su += d[i];
    sux += d[i] * xh[i];
  }
  const float mu = group_sum<D / 8>(su) / D, mux = group_sum<D / 8>(sux) / D;
#pragma unroll
  for (int i = 0; i < 8; ++i) d[i] = inv * (d[i] - mu - xh[i] * mux);
}

// The CTA's per-thread partials of one [N] vector (thread = row group `sub` x 8 columns of segment `seg`) summed over
// the row groups in a fixed order into part[0, N).  No atomics: two runs give the same bits.
template <int N>
__device__ void cta_column_sum(const float (&a)[8], float* __restrict__ part) {
  constexpr int LPR = N / 8, RPB = kThreads / LPR;
  __shared__ float red[kThreads * 8];
  const int seg = threadIdx.x % LPR, sub = threadIdx.x / LPR;
  __syncthreads();  // a previous call may still be reading red
#pragma unroll
  for (int i = 0; i < 8; ++i) red[sub * N + seg * 8 + i] = a[i];
  __syncthreads();
  if (threadIdx.x < N) {
    float s = 0.f;
#pragma unroll 4
    for (int r = 0; r < RPB; ++r) s += red[r * N + threadIdx.x];
    part[threadIdx.x] = s;
  }
}

// Second, small launch of every reduction: out[k][j] = sum over rows r of in[k][r*stride + j], rows in a fixed order
// (each of kColSumY thread rows takes every kColSumY-th partial row, then the kColSumY sums are added in order).
constexpr int kColSumX = 32, kColSumY = 8;
struct ColSumArgs {
  const float* in[4];
  float* out[4];
  long long stride;
  int rows, cols;
};
__global__ void __launch_bounds__(kColSumX* kColSumY) column_sum_kernel(const ColSumArgs a) {
  __shared__ float red[kColSumY][kColSumX];
  const int j = blockIdx.x * kColSumX + threadIdx.x, k = blockIdx.y;
  const float* in = a.in[k];
  float s = 0.f;
  if (j < a.cols && a.out[k]) {
#pragma unroll 4
    for (int r = threadIdx.y; r < a.rows; r += kColSumY) s += in[r * a.stride + j];
  }
  red[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0 && j < a.cols && a.out[k]) {
    float t = 0.f;
#pragma unroll
    for (int y = 0; y < kColSumY; ++y) t += red[y][threadIdx.x];
    a.out[k][j] = t;
  }
}

// ---- row norm backward on [m, N]: dx, and dgamma (dbeta) partials per CTA -------------------------------------
template <bool BF16, int N, bool kLayer>
__global__ void __launch_bounds__(kThreads)
row_norm_bwd_kernel(const uint4* __restrict__ x, const uint4* __restrict__ dy, const uint4* __restrict__ gamma,
                    uint4* __restrict__ dx, float eps, long long m, float* __restrict__ part) {
  constexpr int LPR = N / 8, RPB = kThreads / LPR;
  const int seg = threadIdx.x % LPR, sub = threadIdx.x / LPR;
  float g[8], ag[8] = {}, ab[8] = {};
  unpack8<BF16>(__ldg(gamma + seg), g);
  const long long pass = static_cast<long long>(gridDim.x) * RPB;
  for (long long base = static_cast<long long>(blockIdx.x) * RPB; base < m; base += pass * kUnrollRows) {
    uint4 xv[kUnrollRows], dv[kUnrollRows];
#pragma unroll
    for (int u = 0; u < kUnrollRows; ++u) {
      const long long r = base + u * pass + sub;
      xv[u] = r < m ? x[r * LPR + seg] : make_uint4(0, 0, 0, 0);
      dv[u] = r < m ? dy[r * LPR + seg] : make_uint4(0, 0, 0, 0);  // rows past m add nothing to the partials
    }
#pragma unroll
    for (int u = 0; u < kUnrollRows; ++u) {
      const long long r = base + u * pass + sub;
      float f[8], d[8];
      unpack8<BF16>(xv[u], f);
      unpack8<BF16>(dv[u], d);
      if constexpr (kLayer) ln_bwd<N>(f, d, g, ag, ab);
      else rms_bwd<N>(f, d, g, eps, ag);
      if (r < m) dx[r * LPR + seg] = pack8<BF16>(d);
    }
  }
  cta_column_sum<N>(ag, part + static_cast<long long>(blockIdx.x) * 2 * N);
  if constexpr (kLayer) cta_column_sum<N>(ab, part + static_cast<long long>(blockIdx.x) * 2 * N + N);
}

// ---- fused backward of qkv_prep_kernel -----------------------------------------------------------------------------
struct PrepBwdArgs {
  const uint16_t* dy[3];   // dQ, dK, dV [B, H, S_out, D]: rows [out_row0, out_row0 + S_in) are read, no others
  const uint16_t* x[2];    // the forward's q_in, k_in (token stride / batch stride in geo)
  uint16_t* dx[3];         // dq_in, dk_in, dv_in: contiguous [B, S_in, H*D]
  const uint16_t* gamma[2];
  float* part[2];          // q, k: per-CTA [dgamma | dbeta] partials (NORM_RMS_HIDDEN: per-split dgamma [H*D])
  float2* stats[2];        // NORM_RMS_HIDDEN: per token (r, mean(u*x^) over the hidden row)
  PrepGeom geo;
};

// the gradient at the norm output of one head row: the RoPE transpose, rounded to the 16-bit dtype when a norm
// follows (the forward's own rounding point between norm and RoPE)
template <bool BF16, int D>
__device__ __forceinline__ void prep_dn(float (&f)[8], bool rot, int rope, bool round, const float (&c8)[8],
                                        const float (&s8)[8], const float (&c4)[4], const float (&s4)[4]) {
  if (!rot) return;
  if (rope == 2) {
    rope_apply_complex<BF16, true>(f, c4, s4);
  } else {
    rope_apply<true>(f, c8, s8);
    if (round) {
#pragma unroll
      for (int i = 0; i < 8; ++i) f[i] = round16f<BF16>(f[i]);
    }
  }
}

// grid (token blocks, B, 3), persistent over the tokens.  Per-head norms: dx and the CTA's dgamma / dbeta
// partials.  NORM_RMS_HIDDEN: only the per-token (r, mean(u*x^)) of q and k (hidden_rms_bwd_kernel writes their dx).
template <bool BF16, int D>
__global__ void __launch_bounds__(kThreads)
qkv_prep_bwd_kernel(const PrepBwdArgs a) {
  constexpr int LPR = D / 8, RPB = kThreads / LPR;
  const int seg = threadIdx.x % LPR, sub = threadIdx.x / LPR;
  const int which = blockIdx.z;  // 0 q, 1 k, 2 v
  const int norm = which < 2 ? a.geo.norm : 0;
  const long long HD = static_cast<long long>(a.geo.H) * D;
  float g[8], ag[8] = {}, ab[8] = {}, c8[8], s8[8], c4[4], s4[4];
  if (norm == 1 || norm == 2) unpack8<BF16>(__ldg(reinterpret_cast<const uint4*>(a.gamma[which]) + seg), g);
#pragma unroll 1
  for (int t0 = blockIdx.x * RPB; t0 < a.geo.S_in; t0 += gridDim.x * RPB) {  // block-uniform
    const int t = t0 + sub;
    const bool live = t < a.geo.S_in;
    const int tt = live ? t : a.geo.S_in - 1;  // keep the whole warp in the shuffles; dead lanes add and store nothing
    const uint16_t* dy =
        a.dy[which] + blockIdx.y * a.geo.out_batch_stride + static_cast<long long>(a.geo.out_row0 + tt) * D + seg * 8;
    const uint16_t* x = which < 2 ? a.x[which] + blockIdx.y * a.geo.in_batch_stride + tt * a.geo.in_token_stride + seg * 8
                                  : nullptr;
    uint16_t* dx = a.dx[which] + (static_cast<long long>(blockIdx.y) * a.geo.S_in + tt) * HD + seg * 8;
    const bool rot = which < 2 && a.geo.rope != 0 && tt >= a.geo.rope_lo && tt < a.geo.rope_lo + a.geo.rope_n;
    if (rot) load_rope_tables<D>(a.geo.cos_t, a.geo.sin_t, tt - a.geo.rope_lo, seg, a.geo.rope == 2, c8, s8, c4, s4);
    if (norm == 3) {  // first pass over the hidden row: sum x^2 and (gamma*dn)*x over all H heads
      float ss = 0.f, ux = 0.f;
#pragma unroll 1
      for (int h0 = 0; h0 < a.geo.H; h0 += kUnrollRows) {
        uint4 dv[kUnrollRows], xv[kUnrollRows];
#pragma unroll
        for (int u = 0; u < kUnrollRows; ++u) {
          const bool in = h0 + u < a.geo.H;
          dv[u] = in ? *reinterpret_cast<const uint4*>(dy + (h0 + u) * a.geo.out_head_stride) : make_uint4(0, 0, 0, 0);
          xv[u] = in ? *reinterpret_cast<const uint4*>(x + (h0 + u) * D) : make_uint4(0, 0, 0, 0);
        }
#pragma unroll
        for (int u = 0; u < kUnrollRows; ++u) {
          if (h0 + u < a.geo.H) {
            float f[8], d[8], gw[8];
            unpack8<BF16>(xv[u], f);
            unpack8<BF16>(dv[u], d);
            unpack8<BF16>(__ldg(reinterpret_cast<const uint4*>(a.gamma[which] + (h0 + u) * D) + seg), gw);
            prep_dn<BF16, D>(d, rot, a.geo.rope, true, c8, s8, c4, s4);
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              ss += f[i] * f[i];
              ux += gw[i] * d[i] * f[i];
            }
          }
        }
      }
      ss = group_sum<LPR>(ss);
      ux = group_sum<LPR>(ux);
      const float inv = 1.0f / sqrtf(ss / HD + a.geo.eps);
      if (live && seg == 0)
        a.stats[which][static_cast<long long>(blockIdx.y) * a.geo.S_in + t] = make_float2(inv, inv * ux / HD);
      continue;
    }
#pragma unroll 1
    for (int h0 = 0; h0 < a.geo.H; h0 += kUnrollRows) {
      uint4 dv[kUnrollRows], xv[kUnrollRows];
#pragma unroll
      for (int u = 0; u < kUnrollRows; ++u) {
        if (h0 + u < a.geo.H) {
          dv[u] = *reinterpret_cast<const uint4*>(dy + (h0 + u) * a.geo.out_head_stride);
          if (norm != 0) xv[u] = *reinterpret_cast<const uint4*>(x + (h0 + u) * D);
        }
      }
#pragma unroll
      for (int u = 0; u < kUnrollRows; ++u) {
        if (h0 + u < a.geo.H) {  // block-uniform
          if (norm != 0 || rot) {
            float d[8];
            unpack8<BF16>(dv[u], d);
            prep_dn<BF16, D>(d, rot, a.geo.rope, norm != 0, c8, s8, c4, s4);
            if (norm != 0) {
              float f[8];
              unpack8<BF16>(xv[u], f);
              if (!live) {
#pragma unroll
                for (int i = 0; i < 8; ++i) d[i] = 0.f;
              }
              if (norm == 1) rms_bwd<D>(f, d, g, a.geo.eps, ag);
              else ln_bwd<D>(f, d, g, ag, ab);
            }
            dv[u] = pack8<BF16>(d);
          }
          if (live) *reinterpret_cast<uint4*>(dx + (h0 + u) * D) = dv[u];
        }
      }
    }
  }
  if (norm == 1 || norm == 2) {
    float* p = a.part[which] + (static_cast<long long>(blockIdx.y) * gridDim.x + blockIdx.x) * 2 * D;
    cta_column_sum<D>(ag, p);
    if (norm == 2) cta_column_sum<D>(ab, p + D);
  }
}

// NORM_RMS_HIDDEN, second pass: a thread owns 8 columns of the hidden row (head c / LPR) and walks its split of the
// B*S_in tokens, so its dgamma partial stays in registers: dx = r*(u - x^*m) with (r, m) from the first pass.
constexpr int kHiddenThreads = 128;
template <bool BF16, int D>
__global__ void __launch_bounds__(kHiddenThreads)
hidden_rms_bwd_kernel(const PrepBwdArgs a, int B) {
  constexpr int LPR = D / 8;
  const int which = blockIdx.z;
  const int c = blockIdx.x * kHiddenThreads + threadIdx.x;
  if (c >= a.geo.H * LPR) return;
  const int h = c / LPR, seg = c % LPR;
  const long long HD = static_cast<long long>(a.geo.H) * D;
  const long long T = static_cast<long long>(B) * a.geo.S_in;
  const long long per = (T + gridDim.y - 1) / gridDim.y;
  const long long lo = blockIdx.y * per, hi = lo + per < T ? lo + per : T;
  float g[8], ag[8] = {};
  unpack8<BF16>(__ldg(reinterpret_cast<const uint4*>(a.gamma[which]) + c), g);
#pragma unroll 1
  for (long long i0 = lo; i0 < hi; i0 += kUnrollRows) {
    uint4 dv[kUnrollRows], xv[kUnrollRows];
#pragma unroll
    for (int u = 0; u < kUnrollRows; ++u) {
      const long long i = i0 + u;
      if (i < hi) {
        const long long b = i / a.geo.S_in, t = i % a.geo.S_in;
        dv[u] = *reinterpret_cast<const uint4*>(a.dy[which] + b * a.geo.out_batch_stride + h * a.geo.out_head_stride +
                                                (a.geo.out_row0 + t) * D + seg * 8);
        xv[u] = *reinterpret_cast<const uint4*>(a.x[which] + b * a.geo.in_batch_stride + t * a.geo.in_token_stride + c * 8);
      }
    }
#pragma unroll
    for (int u = 0; u < kUnrollRows; ++u) {
      const long long i = i0 + u;
      if (i < hi) {
        const int t = static_cast<int>(i % a.geo.S_in);
        const bool rot = a.geo.rope != 0 && t >= a.geo.rope_lo && t < a.geo.rope_lo + a.geo.rope_n;
        float c8[8], s8[8], c4[4], s4[4], f[8], d[8];
        if (rot) load_rope_tables<D>(a.geo.cos_t, a.geo.sin_t, t - a.geo.rope_lo, seg, a.geo.rope == 2, c8, s8, c4, s4);
        unpack8<BF16>(xv[u], f);
        unpack8<BF16>(dv[u], d);
        prep_dn<BF16, D>(d, rot, a.geo.rope, true, c8, s8, c4, s4);
        const float2 st = a.stats[which][i];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const float xh = f[k] * st.x;
          ag[k] += d[k] * xh;
          d[k] = st.x * (g[k] * d[k] - xh * st.y);
        }
        *reinterpret_cast<uint4*>(a.dx[which] + i * HD + c * 8) = pack8<BF16>(d);
      }
    }
  }
  float* p = a.part[which] + blockIdx.y * HD + c * 8;
#pragma unroll
  for (int k = 0; k < 8; ++k) p[k] = ag[k];
}


// ================================= host side ===================================================================
// Grid sizes; the backward's workspace sizes are derived from them, so both sides agree.
constexpr int kBwdCtas = 148 * 4;  // persistent grids: a few waves, which bounds the partial rows
// a walk over the rows of [m, n], kUnrollRows rows per thread per pass, on at most cap CTAs
static int row_blocks(long long m, int n, int cap) {
  const long long rpb = kThreads / (n / 8);
  const long long blocks = (m + rpb * kUnrollRows - 1) / (rpb * kUnrollRows);
  return static_cast<int>(blocks < 1 ? 1 : blocks > cap ? cap : blocks);
}
static int prep_bwd_blocks(int B, int S_in, int D) {
  const int rpb = kThreads / (D / 8);
  const int want = (S_in + rpb - 1) / rpb, cap = kBwdCtas / B > 1 ? kBwdCtas / B : 1;
  return want < cap ? want : cap;
}
static int hidden_cols(int H, int D) { return (H * (D / 8) + kHiddenThreads - 1) / kHiddenThreads; }
static int hidden_splits(int B, int S_in, int H, int D) {
  const long long want = kBwdCtas / hidden_cols(H, D), T = static_cast<long long>(B) * S_in;
  return static_cast<int>(want < 1 ? 1 : want > T ? T : want);
}

// The row widths a kernel family is instantiated for.  dispatch() calls f(bf16, n) with both as compile-time
// constants (std::bool_constant, std::integral_constant) and returns its result; check() first.
template <int... Ns>
struct Dims {
  static int check(int n) {
    SVGB_REQUIRE(((n == Ns) || ...), "Unsupported head_dim: %d", n);
    return 0;
  }
};
using NormDims = Dims<32, 64, 128, 256>;  // the row norms: n
using HeadDims = Dims<64, 128, 256>;      // RoPE and the fused prep: D

template <int... Ns, class F>
static int dispatch(Dims<Ns...>, int dtype, int n, F&& f) {
  int rc = 0;
  const auto run = [&](auto N) { rc = dtype == SVGB_BF16 ? f(std::true_type{}, N) : f(std::false_type{}, N); };
  ((n == Ns ? run(std::integral_constant<int, Ns>{}) : void()), ...);
  return rc;
}

static int launch_column_sum(const float* const* in, float* const* out, int n, long long stride, int rows, int cols,
                             cudaStream_t st) {
  ColSumArgs c{};
  for (int k = 0; k < n; ++k) {
    c.in[k] = in[k];
    c.out[k] = out[k];
  }
  c.stride = stride;
  c.rows = rows;
  c.cols = cols;
  column_sum_kernel<<<dim3((cols + kColSumX - 1) / kColSumX, n), dim3(kColSumX, kColSumY), 0, st>>>(c);
  SVGB_LAUNCH_OK();
  return 0;
}

template <bool BF16, int D>
static int launch_prep_bwd(const PrepBwdArgs& a, int B, cudaStream_t st) {
  const int gx = prep_bwd_blocks(B, a.geo.S_in, D);
  qkv_prep_bwd_kernel<BF16, D><<<dim3(gx, B, 3), kThreads, 0, st>>>(a);
  SVGB_LAUNCH_OK();
  if (a.geo.norm == SVGB_NORM_RMS_HIDDEN) {
    const int splits = hidden_splits(B, a.geo.S_in, a.geo.H, D);
    hidden_rms_bwd_kernel<BF16, D><<<dim3(hidden_cols(a.geo.H, D), splits, 2), kHiddenThreads, 0, st>>>(a, B);
    SVGB_LAUNCH_OK();
  }
  return 0;
}

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// svgb_rms_norm / svgb_layer_norm (layer: beta, and eps is LayerNorm's fixed 1e-5)
static int row_norm(void* x, const void* gamma, const void* beta, long long m, int n, float eps, int dtype,
                    bool layer, void* stream) {
  SVGB_REQUIRE(x && gamma && (beta || !layer) && m >= 0, "null pointer");
  if (NormDims::check(n)) return -1;
  SVGB_REQUIRE(dtype == SVGB_BF16 || dtype == SVGB_F16, "dtype %d unsupported", dtype);
  SVGB_REQUIRE(aligned16(x) && aligned16(gamma) && (!layer || aligned16(beta)), "pointers must be 16-byte aligned");
  if (m == 0) return 0;
  const unsigned blocks = row_blocks(m, n, 148 * 32);
  auto X = static_cast<uint4*>(x);
  auto G = static_cast<const uint4*>(gamma);
  auto Bt = static_cast<const uint4*>(beta);
  auto st = static_cast<cudaStream_t>(stream);
  return dispatch(NormDims{}, dtype, n, [&](auto bf, auto N) {
    const auto kernel = layer ? row_norm_kernel<bf, N, true> : row_norm_kernel<bf, N, false>;
    kernel<<<blocks, kThreads, 0, st>>>(X, G, Bt, eps, m);
    SVGB_LAUNCH_OK();
    return 0;
  });
}

// svgb_rms_norm_bwd / svgb_layer_norm_bwd
static int row_norm_bwd(const void* x, const void* dy, const void* gamma, void* dx, float* dgamma, float* dbeta,
                        long long m, int n, float eps, int dtype, bool layer, void* ws, size_t ws_bytes,
                        void* stream) {
  SVGB_REQUIRE(x && dy && gamma && dx && dgamma && (dbeta || !layer) && m >= 0, "null pointer");
  if (NormDims::check(n)) return -1;
  SVGB_REQUIRE(dtype == SVGB_BF16 || dtype == SVGB_F16, "dtype %d unsupported", dtype);
  SVGB_REQUIRE(aligned16(x) && aligned16(dy) && aligned16(gamma) && aligned16(dx), "pointers must be 16-byte aligned");
  size_t need = 0;
  if (svgb_row_norm_bwd_bytes(m, n, &need)) return -1;
  SVGB_REQUIRE(ws && ws_bytes >= need, "backward workspace too small: %zu < %zu", ws_bytes, need);
  auto st = static_cast<cudaStream_t>(stream);
  if (m == 0) {  // no rows: the parameter gradients are zero
    SVGB_CUDA(cudaMemsetAsync(dgamma, 0, sizeof(float) * n, st));
    if (layer) SVGB_CUDA(cudaMemsetAsync(dbeta, 0, sizeof(float) * n, st));
    return 0;
  }
  const int blocks = row_blocks(m, n, kBwdCtas);
  auto X = static_cast<const uint4*>(x);
  auto DY = static_cast<const uint4*>(dy);
  auto G = static_cast<const uint4*>(gamma);
  auto DX = static_cast<uint4*>(dx);
  auto part = static_cast<float*>(ws);
  const int rc = dispatch(NormDims{}, dtype, n, [&](auto bf, auto N) {
    const auto kernel = layer ? row_norm_bwd_kernel<bf, N, true> : row_norm_bwd_kernel<bf, N, false>;
    kernel<<<blocks, kThreads, 0, st>>>(X, DY, G, DX, eps, m, part);
    SVGB_LAUNCH_OK();
    return 0;
  });
  if (rc) return rc;
  const float* in[2] = {part, part + n};
  float* out[2] = {dgamma, dbeta};
  return launch_column_sum(in, out, layer ? 2 : 1, 2LL * n, blocks, n, st);
}

// svgb_qk_rope (in place: q_out = q, k_out = k) / svgb_qk_rope_bwd (transpose: the RoPE transpose, out of place)
static int qk_rope(const void* q, const void* k, void* q_out, void* k_out, const float* cos_t, const float* sin_t,
                   int B, int Hq, int Hk, int S, int D, int len_text, int mode, int dtype, bool transpose,
                   void* stream) {
  SVGB_REQUIRE(q && k && q_out && k_out && cos_t && sin_t, "null pointer");
  SVGB_REQUIRE(B > 0 && Hq > 0 && Hk > 0 && S > 0, "bad sizes");
  if (HeadDims::check(D)) return -1;
  SVGB_REQUIRE(len_text >= 0 && len_text < S, "len_text_prompt must leave at least one rotated row");
  SVGB_REQUIRE(mode >= SVGB_ROPE_TXT_FIRST && mode <= SVGB_ROPE_COMPLEX_TXT_FIRST, "mode %d unknown", mode);
  SVGB_REQUIRE(dtype == SVGB_BF16 || dtype == SVGB_F16, "dtype %d unsupported", dtype);
  SVGB_REQUIRE(aligned16(q) && aligned16(k) && aligned16(q_out) && aligned16(k_out) && aligned16(cos_t) &&
                   aligned16(sin_t),
               "pointers must be 16-byte aligned");
  const int valid = S - len_text;
  const int row0 = mode == SVGB_ROPE_TXT_LAST ? 0 : len_text;
  const bool complex = mode == SVGB_ROPE_COMPLEX_TXT_FIRST;
  const int rpb = kThreads / (D / 8);
  const dim3 grid(((transpose ? S : valid) + rpb - 1) / rpb, B);
  auto Q = static_cast<const uint4*>(q);
  auto K = static_cast<const uint4*>(k);
  auto QO = static_cast<uint4*>(q_out);
  auto KO = static_cast<uint4*>(k_out);
  auto st = static_cast<cudaStream_t>(stream);
  return dispatch(HeadDims{}, dtype, D, [&](auto bf, auto d) {
    if (transpose) {
      const auto kernel = complex ? qk_rope_bwd_kernel<bf, d, true> : qk_rope_bwd_kernel<bf, d, false>;
      kernel<<<grid, kThreads, 0, st>>>(Q, K, QO, KO, cos_t, sin_t, Hq, Hk, S, row0, valid);
    } else {
      const auto kernel = complex ? qk_rope_kernel<bf, d, true> : qk_rope_kernel<bf, d, false>;
      kernel<<<grid, kThreads, 0, st>>>(QO, KO, cos_t, sin_t, Hq, Hk, S, row0, valid);
    }
    SVGB_LAUNCH_OK();
    return 0;
  });
}

// The checks svgb_qkv_prep and svgb_qkv_prep_bwd share, and the geometry they pass to the kernels.
static int prep_geom(PrepGeom& g, long long in_token_stride, long long in_batch_stride, long long out_head_stride,
                     long long out_batch_stride, int B, int S_in, int H, int D, int out_row0, int norm, float eps,
                     int rope, const float* cos_t, const float* sin_t, int rope_lo, int rope_n, int dtype) {
  SVGB_REQUIRE(B > 0 && S_in > 0 && H > 0 && out_row0 >= 0, "bad sizes");
  if (HeadDims::check(D)) return -1;
  SVGB_REQUIRE(dtype == SVGB_BF16 || dtype == SVGB_F16, "dtype %d unsupported", dtype);
  SVGB_REQUIRE(norm >= SVGB_NORM_NONE && norm <= SVGB_NORM_RMS_HIDDEN, "norm %d unknown", norm);
  SVGB_REQUIRE(rope >= 0 && rope <= 2, "rope %d unknown (0 none, 1 cos/sin [n,D], 2 complex [n,D/2])", rope);
  SVGB_REQUIRE(rope == 0 || (cos_t && sin_t && rope_lo >= 0 && rope_n >= 0 && rope_lo + rope_n <= S_in),
               "rope needs tables and a token range inside [0, S_in)");
  SVGB_REQUIRE(in_token_stride % 8 == 0 && in_batch_stride % 8 == 0 && out_head_stride % 8 == 0 &&
                   out_batch_stride % 8 == 0,
               "strides must be multiples of 8 elements (16 bytes)");
  g = PrepGeom{cos_t,    sin_t, in_token_stride, in_batch_stride, out_head_stride, out_batch_stride, S_in, H,
               out_row0, norm,  rope,            rope_lo,         rope_n,          eps};
  return 0;
}

}  // namespace svgb

using namespace svgb;

extern "C" {

int svgb_rms_norm(void* x, const void* gamma, long long m, int n, float eps, int dtype, void* stream) {
  return row_norm(x, gamma, nullptr, m, n, eps, dtype, false, stream);
}

int svgb_layer_norm(void* x, const void* gamma, const void* beta, long long m, int n, int dtype, void* stream) {
  return row_norm(x, gamma, beta, m, n, 0.f, dtype, true, stream);
}

int svgb_qk_rope(void* q, void* k, const float* cos_t, const float* sin_t, int B, int Hq, int Hk, int S, int D,
                 int len_text, int mode, int dtype, void* stream) {
  return qk_rope(q, k, q, k, cos_t, sin_t, B, Hq, Hk, S, D, len_text, mode, dtype, false, stream);
}

int svgb_qkv_prep(const void* q_in, const void* k_in, const void* v_in, long long in_token_stride,
                  long long in_batch_stride, void* q_out, void* k_out, void* v_out, long long out_head_stride,
                  long long out_batch_stride, int B, int S_in, int H, int D, int out_row0, int norm,
                  const void* gamma_q, const void* gamma_k, const void* beta_q, const void* beta_k, float eps,
                  int rope, const float* cos_t, const float* sin_t, int rope_lo, int rope_n, int dtype,
                  void* stream) {
  SVGB_REQUIRE(q_in && k_in && v_in && q_out && k_out && v_out, "null pointer");
  PrepArgs a;
  if (prep_geom(a.geo, in_token_stride, in_batch_stride, out_head_stride, out_batch_stride, B, S_in, H, D, out_row0,
                norm, eps, rope, cos_t, sin_t, rope_lo, rope_n, dtype))
    return -1;
  SVGB_REQUIRE(norm == SVGB_NORM_NONE || (gamma_q && gamma_k), "norm needs gamma_q and gamma_k");
  SVGB_REQUIRE(norm != SVGB_NORM_LAYER || (beta_q && beta_k), "layer norm needs beta_q and beta_k");
  SVGB_REQUIRE(aligned16(q_in) && aligned16(k_in) && aligned16(v_in) && aligned16(q_out) && aligned16(k_out) &&
                   aligned16(v_out),
               "pointers must be 16-byte aligned");
  a.in[0] = static_cast<const uint16_t*>(q_in);
  a.in[1] = static_cast<const uint16_t*>(k_in);
  a.in[2] = static_cast<const uint16_t*>(v_in);
  a.out[0] = static_cast<uint16_t*>(q_out);
  a.out[1] = static_cast<uint16_t*>(k_out);
  a.out[2] = static_cast<uint16_t*>(v_out);
  a.gamma[0] = static_cast<const uint16_t*>(gamma_q);
  a.gamma[1] = static_cast<const uint16_t*>(gamma_k);
  a.beta[0] = static_cast<const uint16_t*>(beta_q);
  a.beta[1] = static_cast<const uint16_t*>(beta_k);
  const int rpb = kThreads / (D / 8);
  const dim3 grid((S_in + rpb - 1) / rpb, B, 3);
  auto st = static_cast<cudaStream_t>(stream);
  return dispatch(HeadDims{}, dtype, D, [&](auto bf, auto d) {
    qkv_prep_kernel<bf, d><<<grid, kThreads, 0, st>>>(a);
    SVGB_LAUNCH_OK();
    return 0;
  });
}

int svgb_row_norm_bwd_bytes(long long m, int n, size_t* bytes) {
  SVGB_REQUIRE(bytes && m >= 0, "bad arguments");
  if (NormDims::check(n)) return -1;
  *bytes = align_up(sizeof(float) * 2 * n * static_cast<size_t>(row_blocks(m, n, kBwdCtas)), 256);
  return 0;
}

int svgb_rms_norm_bwd(const void* x, const void* dy, const void* gamma, void* dx, float* dgamma, long long m, int n,
                      float eps, int dtype, void* ws, size_t ws_bytes, void* stream) {
  return row_norm_bwd(x, dy, gamma, dx, dgamma, nullptr, m, n, eps, dtype, false, ws, ws_bytes, stream);
}

int svgb_layer_norm_bwd(const void* x, const void* dy, const void* gamma, void* dx, float* dgamma, float* dbeta,
                        long long m, int n, int dtype, void* ws, size_t ws_bytes, void* stream) {
  return row_norm_bwd(x, dy, gamma, dx, dgamma, dbeta, m, n, 0.f, dtype, true, ws, ws_bytes, stream);
}

int svgb_qk_rope_bwd(const void* dq, const void* dk, void* dq_out, void* dk_out, const float* cos_t,
                     const float* sin_t, int B, int Hq, int Hk, int S, int D, int len_text, int mode, int dtype,
                     void* stream) {
  return qk_rope(dq, dk, dq_out, dk_out, cos_t, sin_t, B, Hq, Hk, S, D, len_text, mode, dtype, true, stream);
}

int svgb_qkv_prep_bwd_bytes(int B, int S_in, int H, int D, int norm, size_t* bytes) {
  SVGB_REQUIRE(bytes && B > 0 && S_in > 0 && H > 0, "bad arguments");
  if (HeadDims::check(D)) return -1;
  SVGB_REQUIRE(norm >= SVGB_NORM_NONE && norm <= SVGB_NORM_RMS_HIDDEN, "norm %d unknown", norm);
  size_t n = 0;
  if (norm == SVGB_NORM_RMS_HEAD || norm == SVGB_NORM_LAYER)  // q, k: [blocks * B][dgamma | dbeta]
    n = align_up(sizeof(float) * 2 * D * static_cast<size_t>(prep_bwd_blocks(B, S_in, D)) * B, 256) * 2;
  else if (norm == SVGB_NORM_RMS_HIDDEN)  // q, k: [splits][H*D] dgamma, then the per-token (r, m) pairs
    n = align_up(sizeof(float) * static_cast<size_t>(H) * D * hidden_splits(B, S_in, H, D), 256) * 2 +
        align_up(sizeof(float) * 2 * static_cast<size_t>(B) * S_in, 256) * 2;
  *bytes = n;
  return 0;
}

int svgb_qkv_prep_bwd(const void* dq, const void* dk, const void* dv, long long out_head_stride,
                      long long out_batch_stride, const void* q_in, const void* k_in, long long in_token_stride,
                      long long in_batch_stride, void* dq_in, void* dk_in, void* dv_in, int B, int S_in, int H, int D,
                      int out_row0, int norm, const void* gamma_q, const void* gamma_k, float eps, int rope,
                      const float* cos_t, const float* sin_t, int rope_lo, int rope_n, float* dgamma_q,
                      float* dgamma_k, float* dbeta_q, float* dbeta_k, int dtype, void* ws, size_t ws_bytes,
                      void* stream) {
  SVGB_REQUIRE(dq && dk && dv && dq_in && dk_in && dv_in, "null pointer");
  PrepBwdArgs a{};
  if (prep_geom(a.geo, in_token_stride, in_batch_stride, out_head_stride, out_batch_stride, B, S_in, H, D, out_row0,
                norm, eps, rope, cos_t, sin_t, rope_lo, rope_n, dtype))
    return -1;
  SVGB_REQUIRE(norm == SVGB_NORM_NONE || (q_in && k_in && gamma_q && gamma_k && dgamma_q && dgamma_k),
               "norm needs q_in, k_in, gamma_q, gamma_k, dgamma_q and dgamma_k");
  SVGB_REQUIRE(norm != SVGB_NORM_LAYER || (dbeta_q && dbeta_k), "layer norm needs dbeta_q and dbeta_k");
  SVGB_REQUIRE(aligned16(dq) && aligned16(dk) && aligned16(dv) && aligned16(dq_in) && aligned16(dk_in) &&
                   aligned16(dv_in) && (norm == SVGB_NORM_NONE || (aligned16(q_in) && aligned16(k_in))),
               "pointers must be 16-byte aligned");
  size_t need = 0;
  if (svgb_qkv_prep_bwd_bytes(B, S_in, H, D, norm, &need)) return -1;
  SVGB_REQUIRE(need == 0 || (ws && ws_bytes >= need), "backward workspace too small: %zu < %zu", ws_bytes, need);
  a.dy[0] = static_cast<const uint16_t*>(dq);
  a.dy[1] = static_cast<const uint16_t*>(dk);
  a.dy[2] = static_cast<const uint16_t*>(dv);
  a.x[0] = static_cast<const uint16_t*>(q_in);
  a.x[1] = static_cast<const uint16_t*>(k_in);
  a.dx[0] = static_cast<uint16_t*>(dq_in);
  a.dx[1] = static_cast<uint16_t*>(dk_in);
  a.dx[2] = static_cast<uint16_t*>(dv_in);
  a.gamma[0] = static_cast<const uint16_t*>(gamma_q);
  a.gamma[1] = static_cast<const uint16_t*>(gamma_k);
  // workspace: the q then the k partials, each need / 2 (NORM_RMS_HIDDEN: partials, then stats)
  auto base = static_cast<char*>(ws);
  long long rows = 0, stride = 0;
  int cols = 0;
  if (norm == SVGB_NORM_RMS_HEAD || norm == SVGB_NORM_LAYER) {
    rows = static_cast<long long>(prep_bwd_blocks(B, S_in, D)) * B;
    stride = 2 * D;
    cols = D;
    a.part[0] = reinterpret_cast<float*>(base);
    a.part[1] = reinterpret_cast<float*>(base + need / 2);
  } else if (norm == SVGB_NORM_RMS_HIDDEN) {
    rows = hidden_splits(B, S_in, H, D);
    stride = static_cast<long long>(H) * D;
    cols = H * D;
    const size_t pb = align_up(sizeof(float) * static_cast<size_t>(H) * D * rows, 256);
    a.part[0] = reinterpret_cast<float*>(base);
    a.part[1] = reinterpret_cast<float*>(base + pb);
    a.stats[0] = reinterpret_cast<float2*>(base + 2 * pb);
    a.stats[1] = reinterpret_cast<float2*>(base + 2 * pb + align_up(sizeof(float) * 2 * static_cast<size_t>(B) * S_in, 256));
  }
  auto st = static_cast<cudaStream_t>(stream);
  const int rc = dispatch(HeadDims{}, dtype, D, [&](auto bf, auto d) { return launch_prep_bwd<bf, d>(a, B, st); });
  if (rc || norm == SVGB_NORM_NONE) return rc;
  const float* in[4] = {a.part[0], a.part[0] + D, a.part[1], a.part[1] + D};
  float* out[4] = {dgamma_q, norm == SVGB_NORM_LAYER ? dbeta_q : nullptr, dgamma_k,
                   norm == SVGB_NORM_LAYER ? dbeta_k : nullptr};
  if (norm == SVGB_NORM_RMS_HIDDEN) in[1] = in[3] = nullptr;
  return launch_column_sum(in, out, 4, stride, static_cast<int>(rows), cols, st);
}

}  // extern "C"
