// Per-head absmax quantisation of a 16-bit [BH, S, D] tensor to fp8 e4m3 (bytes) for the FP8 attention
// path: scale[h] = absmax_h / 448, x8 = round_to_nearest_sat(x / scale[h]).  Two HBM-bound passes.  And the per-row
// quantisation of the queries of the per-row FP8 KV cache (svgb_quantize_e4m3_rows): one pass.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <algorithm>

#include "../../include/svgb200.h"
#include "fp8_rows.cuh"
#include "host_common.h"

namespace svgb {

template <bool BF16>
__device__ __forceinline__ float q_to_f32(uint16_t h) {
  if constexpr (BF16) return __uint_as_float(static_cast<uint32_t>(h) << 16);
  else return __half2float(__ushort_as_half(h));
}

template <bool BF16>
__global__ void __launch_bounds__(256)
absmax_kernel(const uint4* __restrict__ x, long long vec_per_head, unsigned int* __restrict__ amax_bits) {
  const int h = blockIdx.y;
  const uint4* p = x + static_cast<long long>(h) * vec_per_head;
  float m = 0.f;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < vec_per_head;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const uint4 v = p[i];
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      m = fmaxf(m, fabsf(q_to_f32<BF16>(static_cast<uint16_t>(w[j] & 0xffff))));
      m = fmaxf(m, fabsf(q_to_f32<BF16>(static_cast<uint16_t>(w[j] >> 16))));
    }
  }
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMax(amax_bits + h, __float_as_uint(m));  // non-negative floats order as uints
}

__global__ void absmax_to_scale_kernel(float* scale, int BH) {
  const int h = blockIdx.x * blockDim.x + threadIdx.x;
  if (h < BH) {
    const float a = scale[h];
    scale[h] = a > 0.f ? a / 448.f : 1.f;
  }
}

template <bool BF16>
__global__ void __launch_bounds__(256)
quantize_kernel(const uint4* __restrict__ x, const float* __restrict__ scale, uint2* __restrict__ x8,
                long long vec_per_head) {
  const int h = blockIdx.y;
  const float inv = 1.f / scale[h];
  const uint4* p = x + static_cast<long long>(h) * vec_per_head;
  uint2* q = x8 + static_cast<long long>(h) * vec_per_head;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < vec_per_head;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const uint4 v = p[i];
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    uint32_t out[2];
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const float a = q_to_f32<BF16>(static_cast<uint16_t>(w[2 * j] & 0xffff)) * inv;
      const float b = q_to_f32<BF16>(static_cast<uint16_t>(w[2 * j] >> 16)) * inv;
      const float c = q_to_f32<BF16>(static_cast<uint16_t>(w[2 * j + 1] & 0xffff)) * inv;
      const float d = q_to_f32<BF16>(static_cast<uint16_t>(w[2 * j + 1] >> 16)) * inv;
      uint16_t lo, hi;
      asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(lo) : "f"(b), "f"(a));
      asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(hi) : "f"(d), "f"(c));
      out[j] = static_cast<uint32_t>(lo) | (static_cast<uint32_t>(hi) << 16);
    }
    q[i] = make_uint2(out[0], out[1]);
  }
}

// Per-row quantisation of a 16-bit [rows, H, 128] tensor read at its strides: x8 [rows, H, 128] contiguous e4m3 and
// scale [H, rows] (fp8_rows.cuh), one 16-byte vector per thread, 16 threads per (row, head)
template <bool BF16>
__global__ void __launch_bounds__(256)
quantize_rows_kernel(const uint16_t* __restrict__ x, long long row_stride, long long head_stride, int rows, int H,
                     uint2* __restrict__ x8, float* __restrict__ scale) {
  const long long total = static_cast<long long>(rows) * H * 16;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(idx & 15);
    const long long rh = idx >> 4;
    const int h = static_cast<int>(rh % H), r = static_cast<int>(rh / H);
    const uint4 v = *reinterpret_cast<const uint4*>(x + r * row_stride + h * head_stride + 8 * c);
    int e;
    x8[idx] = e4m3_row_quantise<BF16>(v, 0xffffu << (threadIdx.x & 16), &e);  // a (row, head) is an aligned half-warp
    if (c == 0) scale[static_cast<long long>(h) * rows + r] = e4m3_row_scale(e);
  }
}

}  // namespace svgb

using namespace svgb;

extern "C" int svgb_quantize_e4m3_rows(const void* x, int dtype, void* x8, float* scale, int rows, int H, int D,
                                       long long row_stride, long long head_stride, void* stream) {
  const char* who = "svgb_quantize_e4m3_rows";
  SVGB_REQUIRE(x && x8 && scale, "null pointer");
  SVGB_REQUIRE(rows > 0 && H > 0, "%s: bad sizes (rows=%d, H=%d)", who, rows, H);
  SVGB_REQUIRE(D == 128, "%s: per-row scales need head_dim 128 (got %d)", who, D);
  SVGB_REQUIRE(dtype == SVGB_BF16 || dtype == SVGB_F16, "%s takes bf16 or fp16 input (dtype %d)", who, dtype);
  SVGB_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(x8) & 7) == 0,
               "%s: x must be 16-byte and x8 8-byte aligned", who);
  SVGB_REQUIRE(row_stride % 8 == 0 && head_stride % 8 == 0,
               "%s: the row and head strides must be multiples of 8 elements (got %lld, %lld)", who, row_stride,
               head_stride);
  const long long total = static_cast<long long>(rows) * H * 16;
  const unsigned blocks = static_cast<unsigned>(std::min<long long>((total + 255) / 256, 1 << 20));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  auto kern = dtype == SVGB_BF16 ? quantize_rows_kernel<true> : quantize_rows_kernel<false>;
  kern<<<blocks, 256, 0, st>>>(static_cast<const uint16_t*>(x), row_stride, head_stride, rows, H,
                               static_cast<uint2*>(x8), scale);
  SVGB_LAUNCH_OK();
  return 0;
}

extern "C" int svgb_quantize_e4m3(const void* x, int dtype, void* x8, float* scale, int BH, int S, int D,
                                  void* stream) {
  SVGB_REQUIRE(x && x8 && scale && BH > 0 && S > 0 && D > 0 && D % 8 == 0, "bad arguments");
  SVGB_REQUIRE(dtype == SVGB_BF16 || dtype == SVGB_F16, "input dtype %d unsupported", dtype);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long vph = static_cast<long long>(S) * D / 8;
  SVGB_CUDA(cudaMemsetAsync(scale, 0, sizeof(float) * BH, st));
  dim3 grid(static_cast<unsigned>(vph / 1024 > 592 ? 592 : (vph / 1024 > 0 ? vph / 1024 : 1)), BH);
  if (dtype == SVGB_BF16)
    absmax_kernel<true><<<grid, 256, 0, st>>>(static_cast<const uint4*>(x), vph, reinterpret_cast<unsigned int*>(scale));
  else
    absmax_kernel<false><<<grid, 256, 0, st>>>(static_cast<const uint4*>(x), vph, reinterpret_cast<unsigned int*>(scale));
  SVGB_LAUNCH_OK();
  absmax_to_scale_kernel<<<(BH + 127) / 128, 128, 0, st>>>(scale, BH);
  SVGB_LAUNCH_OK();
  if (dtype == SVGB_BF16)
    quantize_kernel<true><<<grid, 256, 0, st>>>(static_cast<const uint4*>(x), scale, static_cast<uint2*>(x8), vph);
  else
    quantize_kernel<false><<<grid, 256, 0, st>>>(static_cast<const uint4*>(x), scale, static_cast<uint2*>(x8), vph);
  SVGB_LAUNCH_OK();
  return 0;
}
