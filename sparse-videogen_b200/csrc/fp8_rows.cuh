// Per-row e4m3 quantisation (the FP8 KV cache's per-row format, svgb200.h): a row of D = 128 16-bit values x with
// a = max|x| gets the power-of-two scale s = 2^e, e the smallest integer with a <= 448 * 2^e, clamped to [-126, 127]
// (a = 0: e = 0), and each element is stored as RN(x * 2^-e) in e4m3.  |x * 2^-e| <= 448, so nothing saturates, and
// the product is an exponent shift, exact in fp32.  Shared by the append into a per-row cache (kvcache.cu) and the
// query quantiser (quant_fp8.cu); e4m3_row_exp also builds for the host (tests/test_attention_kvcache_fp8_rows_cpu.py).
#pragma once
#include <stdint.h>
#include <string.h>

namespace svgb {

// e of the scale rule for a row absmax a >= 0.  With a = m 2^k, m in [0.5, 1) (frexp): e = k - 9 if m <= 0.875 (448 =
// 0.875 2^9), else k - 8.  For a normal fp32 a with biased exponent E and mantissa field M: k = E - 126 and
// m <= 0.875 <=> M <= 0x600000.  Subnormal a (E = 0) gives e <= -134, clamped to -126 like every small row.
__host__ __device__ inline int e4m3_row_exp(float a) {
  uint32_t b;
  memcpy(&b, &a, sizeof(b));
  b &= 0x7fffffffu;
  if (b == 0) return 0;
  const int E = static_cast<int>(b >> 23);
  const int e = E - 126 - ((b & 0x7fffffu) <= 0x600000u ? 9 : 8);
  return e < -126 ? -126 : (e > 127 ? 127 : e);
}

#ifdef __CUDACC__
#include <cuda_fp16.h>

// 2^e and 2^-e for e in [-126, 127]: 2^-127 is an fp32 subnormal
__device__ __forceinline__ float e4m3_row_scale(int e) { return __uint_as_float(static_cast<uint32_t>(e + 127) << 23); }
__device__ __forceinline__ float e4m3_row_inv(int e) {
  return e == 127 ? __uint_as_float(0x00400000u) : __uint_as_float(static_cast<uint32_t>(127 - e) << 23);
}

// One thread holds 8 consecutive 16-bit elements x of a 128-element row, and the 16 threads of the row form the
// aligned half-warp `half_mask` (0x0000ffff or 0xffff0000), all of which call this.  Returns the thread's 8 e4m3
// bytes and the row's exponent e in *e.
template <bool BF16>
__device__ __forceinline__ uint2 e4m3_row_quantise(uint4 x, unsigned half_mask, int* e) {
  const uint32_t w[4] = {x.x, x.y, x.z, x.w};
  float f[8];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const uint16_t lo = static_cast<uint16_t>(w[i] & 0xffffu), hi = static_cast<uint16_t>(w[i] >> 16);
    f[2 * i] = BF16 ? __uint_as_float(static_cast<uint32_t>(lo) << 16) : __half2float(__ushort_as_half(lo));
    f[2 * i + 1] = BF16 ? __uint_as_float(static_cast<uint32_t>(hi) << 16) : __half2float(__ushort_as_half(hi));
  }
  float a = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) a = fmaxf(a, fabsf(f[i]));
#pragma unroll
  for (int o = 1; o < 16; o <<= 1) a = fmaxf(a, __shfl_xor_sync(half_mask, a, o));
  *e = e4m3_row_exp(a);
  const float inv = e4m3_row_inv(*e);
  uint32_t out[2];
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    uint16_t p[2];
#pragma unroll
    for (int i = 0; i < 2; ++i)
      asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(p[i]) : "f"(f[4 * j + 2 * i + 1] * inv), "f"(f[4 * j + 2 * i] * inv));
    out[j] = static_cast<uint32_t>(p[0]) | (static_cast<uint32_t>(p[1]) << 16);
  }
  return make_uint2(out[0], out[1]);
}
#endif

}  // namespace svgb
