// identify_dynamic_map (svg/kmeans_utils.py:852-896) as one fused kernel: centroid scores, size-weighted
// softmax, stable descending sort, top-p cut, scatter -- one CTA per (head, q-cluster).
//
// Every rounding the reference's torch ops perform on 16-bit tensors is reproduced:
//   scores = round16(round16(qc . kc) / float(sqrt(D)))          (matmul then `/`, :877)
//   prob   = round16(w * exp(s - max) / max(sum, 1e-12))         (weighted_softmax, :852-861, fp32 inside)
//   sort descending (stable radix sort); ties -> lower column first (the reference's torch.sort is unstable; we pin it)
//   cums   = torch.cumsum of the sorted 16-bit tensor AS THE CUDA BACKEND COMPUTES IT (the reference runs on the
//            GPU): blocks of 2*nx elements scanned by a Sklansky network in which every add rounds to 16 bit, block
//            totals carried into element 0 of the next block (ATen/native/cuda/ScanUtils.cuh:
//            tensor_kernel_scan_innermost_dim; nx from get_log_num_threads_x_inner_scan(rows = BH*QC, KC): 16 at
//            24 x 400 x 1000, up to 512 for a few long rows).
//            This is NOT an fp32 running sum: near p = 0.9 (bf16 spacing 2^-8) small probabilities are absorbed and
//            the GPU keeps more clusters.  Reproduced bit for bit at every nx (tests/test_dynmap_exact_gpu.py) and on
//            maps recorded from the reference on a GPU (tests/golden/kmeans_golden.npz, 800 x 1000).
//            Not covered: a single row (BH*QC == 1), where torch.cumsum runs cub::DeviceScan instead, whose 16-bit adds
//            associate differently -- the kernel keeps the block scan, so its map can differ from torch's there.
//   keep[t] = t == 0 || !(cums[t-1] > round16(p)) || t < preserve   (:884-890; scalar compared in 16 bit)
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "../../include/svgb200.h"
#include "host_common.h"

namespace svgb {

template <bool BF16>
__device__ __forceinline__ float h2f(uint16_t h) {
  if constexpr (BF16) return __uint_as_float(static_cast<uint32_t>(h) << 16);
  else return __half2float(__ushort_as_half(h));
}
template <bool BF16>
__device__ __forceinline__ uint16_t f2h(float f) {
  if constexpr (BF16) return __bfloat16_as_ushort(__float2bfloat16_rn(f));
  else return __half_as_ushort(__float2half_rn(f));
}

__device__ __forceinline__ float block_reduce(float v, float* red, bool is_max) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  for (int o = 16; o > 0; o >>= 1) {
    const float other = __shfl_xor_sync(0xffffffffu, v, o);
    v = is_max ? fmaxf(v, other) : v + other;
  }
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float r = red[0];
  for (int w = 1; w < nw; ++w) r = is_max ? fmaxf(r, red[w]) : r + red[w];
  return r;
}

// q-centroid rows per CTA (they share every key-centroid row read).  Measured at 24 x 400 x 1000 with the first
// (bitonic-sort) version (ncu, profiles/r02_dynmap_ncu_summary.json): the kernel is INSTRUCTION-bound (1.06e9 warp
// instructions, issue slots 71 % busy, L2 0.6 %), so sharing the key reads among 8 rows (1.53 ms) lost to one row per
// CTA (1.28 ms), which keeps 8 CTAs per SM resident.  The sort is now a two-pass radix sort (see below).
constexpr int kDynRows = 1;
static_assert(kDynRows == 1, "the tensor-core score stage puts one q row into the A fragment");

template <bool BF16, int NBLK>
__global__ void __launch_bounds__(256)
dynmap_kernel(const uint16_t* __restrict__ qc, const uint16_t* __restrict__ kc, const int* __restrict__ k_sizes,
              int QC, int KC, int KCpad, int D, float top_p, int preserve, int log_nx, uint8_t* __restrict__ map) {
  extern __shared__ uint32_t smem[];
  uint32_t* keys = smem;                                     // KCpad
  float* sc_all = reinterpret_cast<float*>(keys + KCpad);    // kDynRows x KCpad : scores, then weighted exps / cums
  float* qrows = sc_all + kDynRows * KCpad;                  // kDynRows x D
  float* red = qrows + kDynRows * D;                         // 32
  int* rhist = reinterpret_cast<int*>(red + 32);             // 8 warps x 256 radix bins
  uint8_t* keep = reinterpret_cast<uint8_t*>(rhist + 8 * 256);  // KCpad
  const int i0 = blockIdx.x * kDynRows, bh = blockIdx.y;
  const int nr = min(kDynRows, QC - i0);
  for (int e = threadIdx.x; e < kDynRows * D; e += blockDim.x) {
    const int r = e / D, d = e - r * D;
    qrows[e] = r < nr ? h2f<BF16>(qc[(static_cast<size_t>(bh) * QC + i0 + r) * D + d]) : 0.f;
  }
  __syncthreads();
  const float sqrt_d = static_cast<float>(sqrt(static_cast<double>(D)));
  // Scores of the q-centroid against every key centroid on the (legacy) warp-level tensor cores: one
  // mma.sync.m16n8k16 covers 8 key rows x 16 dims with the q row in row 0 of the A fragment (rows 1-15 are zero -- the
  // op is 2.5 GFLOP in total, what matters is the instruction count: the first version spent ~45 warp instructions per
  // key row on FMAs and a 5-step shuffle reduction, this one ~4).  Each lane reads 16 contiguous bytes of "its" key row
  // per 32-dim block (lane = 4 * key + quarter) and feeds them as the B fragments of two k-steps; the q fragment uses
  // the same dim -> k-slot assignment, so the product is the plain dot product with a hardware-defined fp32 summation
  // order (deterministic; the 16-bit roundings that follow are the reference's).
  {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    const int g = lane >> 2, tq = lane & 3;
    constexpr int nblk = NBLK;  // D / 32, D in {64, 128, 192, 256}
    uint32_t qa[NBLK][4];       // q fragment: [32-dim block][a0, a2 of the two k-steps]; zero outside lanes 0-3
#pragma unroll
    for (int sb = 0; sb < NBLK; ++sb)
#pragma unroll
      for (int x = 0; x < 4; ++x) {
        uint32_t v = 0;
        if (g == 0) {
          const int d = 32 * sb + 8 * tq + 2 * x;
          v = static_cast<uint32_t>(f2h<BF16>(qrows[d])) | (static_cast<uint32_t>(f2h<BF16>(qrows[d + 1])) << 16);
        }
        qa[sb][x] = v;
      }
    const int ngroups = (KC + 7) / 8;
    for (int grp = warp; grp < ngroups; grp += nwarps) {
      const int j = min(grp * 8 + g, KC - 1);
      const uint4* kr = reinterpret_cast<const uint4*>(kc + (static_cast<size_t>(bh) * KC + j) * D) + tq;
      uint4 kb[NBLK];
#pragma unroll
      for (int sb = 0; sb < NBLK; ++sb) kb[sb] = __ldg(kr + 4 * sb);
      float c0 = 0.f, c1 = 0.f, c2 = 0.f, c3 = 0.f;
#pragma unroll
      for (int sb = 0; sb < NBLK; ++sb) {
          const uint32_t z = 0u;
          if constexpr (BF16) {
            asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                         : "+f"(c0), "+f"(c1), "+f"(c2), "+f"(c3)
                         : "r"(qa[sb][0]), "r"(z), "r"(qa[sb][1]), "r"(z), "r"(kb[sb].x), "r"(kb[sb].y));
            asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                         : "+f"(c0), "+f"(c1), "+f"(c2), "+f"(c3)
                         : "r"(qa[sb][2]), "r"(z), "r"(qa[sb][3]), "r"(z), "r"(kb[sb].z), "r"(kb[sb].w));
          } else {
            asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                         : "+f"(c0), "+f"(c1), "+f"(c2), "+f"(c3)
                         : "r"(qa[sb][0]), "r"(z), "r"(qa[sb][1]), "r"(z), "r"(kb[sb].x), "r"(kb[sb].y));
            asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                         : "+f"(c0), "+f"(c1), "+f"(c2), "+f"(c3)
                         : "r"(qa[sb][2]), "r"(z), "r"(qa[sb][3]), "r"(z), "r"(kb[sb].z), "r"(kb[sb].w));
          }
        }
      if (g == 0) {  // row 0 of the accumulator tile: lanes 0-3 hold the scores of keys 2*tq, 2*tq + 1 of the group
        const int jo = grp * 8 + 2 * tq;
        if (jo < KC) sc_all[jo] = h2f<BF16>(f2h<BF16>(h2f<BF16>(f2h<BF16>(c0)) / sqrt_d));
        if (jo + 1 < KC) sc_all[jo + 1] = h2f<BF16>(f2h<BF16>(h2f<BF16>(f2h<BF16>(c1)) / sqrt_d));
      }
    }
  }
  __syncthreads();
  for (int rr = 0; rr < nr; ++rr) {
  float* sc = sc_all + rr * KCpad;
  const int i = i0 + rr;
  float mx = -INFINITY;
  for (int j = threadIdx.x; j < KC; j += blockDim.x) mx = fmaxf(mx, sc[j]);
  mx = block_reduce(mx, red, true);
  float part = 0.f;
  for (int j = threadIdx.x; j < KC; j += blockDim.x) {
    const float e = static_cast<float>(k_sizes[static_cast<size_t>(bh) * KC + j]) * expf(sc[j] - mx);
    sc[j] = e;
    part += e;
  }
  const float denom = fmaxf(block_reduce(part, red, false), 1e-12f);
  for (int j = threadIdx.x; j < KCpad; j += blockDim.x) {
    uint32_t key = 0;
    if (j < KC) {
      const uint16_t pb = f2h<BF16>(sc[j] / denom);  // non-negative: bit pattern orders like the value
      key = (static_cast<uint32_t>(pb) << 16) | static_cast<uint32_t>(0xFFFF - j);
    }
    keys[j] = key;
  }
  __syncthreads();
  // Stable LSD radix sort (two 8-bit passes) on the 16-bit probability, descending; equal probabilities keep ascending
  // column order because the input is in column order and both passes are stable.  Each warp owns a contiguous segment,
  // counts / places 32 elements per step with match_any ranks, the (digit, warp) table is scanned once per pass.
  // keys -> alt (low byte) -> keys (high byte).  ~25x fewer instructions than the 55-pass bitonic network it replaces.
  {
    uint32_t* alt = reinterpret_cast<uint32_t*>(sc);  // free between the softmax and the scan
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    const int seg = ((KC + nwarps - 1) / nwarps + 31) & ~31;
    const int e0 = warp * seg, e1 = min(KC, e0 + seg);
    const unsigned lt = (1u << lane) - 1u;
    for (int pass = 0; pass < 2; ++pass) {
      const uint32_t* src = pass == 0 ? keys : alt;
      uint32_t* dst = pass == 0 ? alt : keys;
      const int shift = pass * 8;
      for (int x = threadIdx.x; x < nwarps * 256; x += blockDim.x) rhist[x] = 0;
      __syncthreads();
      int* mine = rhist + warp * 256;
      for (int e = e0 + lane; e - lane < e1; e += 32) {
        const bool valid = e < e1;
        const int digit = valid ? static_cast<int>(((0xFFFFu - (src[e] >> 16)) >> shift) & 0xFFu) : 256 + lane;
        const unsigned peers = __match_any_sync(0xffffffffu, digit);
        if (valid && (peers & lt) == 0) mine[digit] += __popc(peers);
        __syncwarp();
      }
      __syncthreads();
      {  // thread d: exclusive prefix over the warps for digit d, then a block-wide exclusive scan over the digit totals
        const int d = threadIdx.x;  // blockDim.x == 256
        int tot = 0;
        for (int w = 0; w < nwarps; ++w) {
          const int v = rhist[w * 256 + d];
          rhist[w * 256 + d] = tot;
          tot += v;
        }
        int incl = tot;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const int n = __shfl_up_sync(0xffffffffu, incl, o);
          if (lane >= o) incl += n;
        }
        __shared__ int wtot[8];
        if (lane == 31) wtot[warp] = incl;
        __syncthreads();
        int basew = 0;
        for (int w = 0; w < warp; ++w) basew += wtot[w];
        const int excl = basew + incl - tot;
        for (int w = 0; w < nwarps; ++w) rhist[w * 256 + d] += excl;
      }
      __syncthreads();
      for (int e = e0 + lane; e - lane < e1; e += 32) {
        const bool valid = e < e1;
        const uint32_t key = valid ? src[e] : 0u;
        const int digit = valid ? static_cast<int>(((0xFFFFu - (key >> 16)) >> shift) & 0xFFu) : 256 + lane;
        const unsigned peers = __match_any_sync(0xffffffffu, digit);
        const int rank = __popc(peers & lt);
        int pos = 0;
        if (valid) pos = mine[digit] + rank;
        __syncwarp();
        if (valid && rank == 0) mine[digit] += __popc(peers);
        __syncwarp();
        if (valid) dst[pos] = key;
      }
      __syncthreads();
    }
  }
  // ---- cumsum exactly as torch's CUDA scan does it on a 16-bit tensor (see the header comment); cums -> sc[]
  auto r16 = [](float f) { return h2f<BF16>(f2h<BF16>(f)); };
  if (log_nx == 4) {
    // 32-element blocks: one warp, lane = element, Sklansky steps through shuffles; blocks are a serial chain
    if (threadIdx.x < 32) {
      const int lane = threadIdx.x;
      float total = 0.f;
      for (int b0 = 0; b0 < KC; b0 += 32) {
        const int t = b0 + lane;
        float v = t < KC ? h2f<BF16>(static_cast<uint16_t>(keys[t] >> 16)) : 0.f;
        if (lane == 0) v = r16(v + total);
#pragma unroll
        for (int m = 0; m < 5; ++m) {
          const int sft = 1 << m;
          const float o = __shfl_sync(0xffffffffu, v, (lane & ~(2 * sft - 1)) | (sft - 1));
          if (lane & sft) v = r16(v + o);
        }
        if (t < KC) sc[t] = v;
        total = __shfl_sync(0xffffffffu, v, 31);
      }
    }
  } else {
    // general block size 2 * nx (64 .. 1024): the same network in shared memory
    const int nx = 1 << log_nx, blk = 2 * nx;
    float* buf = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(keep + KCpad) + 15) & ~uintptr_t(15));
    float total = 0.f;
    for (int b0 = 0; b0 < KC; b0 += blk) {
      for (int e = threadIdx.x; e < blk; e += blockDim.x) {
        float v = (b0 + e) < KC ? h2f<BF16>(static_cast<uint16_t>(keys[b0 + e] >> 16)) : 0.f;
        if (e == 0) v = r16(v + total);
        buf[e] = v;
      }
      __syncthreads();
      for (int m = 0; m <= log_nx; ++m) {
        const int sft = 1 << m;
        for (int tt = threadIdx.x; tt < nx; tt += blockDim.x) {
          const int a = ((tt >> m) << (m + 1)) | sft;
          const int ti = a + (tt % sft), si = a - 1;
          buf[ti] = r16(buf[ti] + buf[si]);
        }
        __syncthreads();
      }
      for (int e = threadIdx.x; e < blk; e += blockDim.x)
        if (b0 + e < KC) sc[b0 + e] = buf[e];
      total = buf[blk - 1];
      __syncthreads();
    }
  }
  __syncthreads();
  {
    const float p16 = r16(top_p);
    for (int t = threadIdx.x; t < KC; t += blockDim.x)
      keep[t] = (t == 0) || !(sc[t - (t > 0)] > p16) || (t < preserve);
  }
  __syncthreads();
  uint8_t* out = map + (static_cast<size_t>(bh) * QC + i) * KC;
  for (int t = threadIdx.x; t < KC; t += blockDim.x) out[0xFFFF - (keys[t] & 0xFFFF)] = keep[t];
  __syncthreads();  // keys / keep are reused by the next row
  }
}

}  // namespace svgb

using namespace svgb;

extern "C" int svgb_dynamic_map(const void* qc, const void* kc, const int32_t* k_sizes, int BH, int QC,
                                int KC, int D, int dtype, float top_p, int preserve, uint8_t* map,
                                void* stream) {
  SVGB_REQUIRE(qc && kc && k_sizes && map, "null pointer");
  SVGB_REQUIRE(BH > 0 && QC > 0 && KC > 0 && KC <= 4096 && D > 0 && D % 64 == 0 && D <= 256, "bad sizes (KC <= 4096, D in {64,128,192,256})");
  SVGB_REQUIRE(dtype == SVGB_BF16 || dtype == SVGB_F16, "dtype %d unsupported", dtype);
  SVGB_REQUIRE(reinterpret_cast<uintptr_t>(kc) % 16 == 0, "kc must be 16-byte aligned");
  int KCpad = 2;
  while (KCpad < KC) KCpad <<= 1;
  // block size of torch's CUDA scan for a [BH*QC, KC] tensor: get_log_num_threads_x_inner_scan (ScanUtils.cuh:19-41,
  // uint32 arithmetic) -- 4 (32-element blocks) at 24 x 400 rows of 1000, up to 9 (1024-element blocks) for a few rows
  uint32_t lx = 0, ly = 0;
  while ((1u << lx) < static_cast<uint32_t>(KC)) ++lx;
  while ((1ull << ly) < static_cast<unsigned long long>(BH) * QC) ++ly;
  uint32_t log_nx = (9u + lx - ly) / 2u;
  log_nx = log_nx < 4u ? 4u : (log_nx > 9u ? 9u : log_nx);
  const size_t smem = sizeof(uint32_t) * KCpad + sizeof(float) * (kDynRows * (KCpad + D) + 32) + 8 * 256 * sizeof(int) + KCpad +
                      (log_nx == 4 ? 0 : sizeof(float) * (2u << log_nx) + 16);
  SVGB_REQUIRE(smem <= 200 * 1024, "KC too large for the dynamic-map kernel (%zu B smem)", smem);
  dim3 grid((QC + kDynRows - 1) / kDynRows, BH);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  auto launch = [&](auto kern) -> int {
    SVGB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
    kern<<<grid, 256, smem, st>>>(static_cast<const uint16_t*>(qc), static_cast<const uint16_t*>(kc), k_sizes, QC, KC,
                                  KCpad, D, top_p, preserve, static_cast<int>(log_nx), map);
    return 0;
  };
  const bool bf = dtype == SVGB_BF16;
  int rc = 0;
  switch (D / 32) {
    case 2: rc = bf ? launch(dynmap_kernel<true, 2>) : launch(dynmap_kernel<false, 2>); break;
    case 4: rc = bf ? launch(dynmap_kernel<true, 4>) : launch(dynmap_kernel<false, 4>); break;
    case 6: rc = bf ? launch(dynmap_kernel<true, 6>) : launch(dynmap_kernel<false, 6>); break;
    default: rc = bf ? launch(dynmap_kernel<true, 8>) : launch(dynmap_kernel<false, 8>); break;
  }
  if (rc) return rc;
  SVGB_LAUNCH_OK();
  return 0;
}
