// sample_mse (svg/models/hyvideo/attention.py:375-399; wan/attention.py:211-233): the SVG1 online
// profiling step.  For `n_rows` sampled query rows per head compute attention over ALL keys three
// times -- unmasked, under the spatial profiling mask, under the temporal one -- and return the mean
// squared error of each masked result against the unmasked one.
//
// Design: the sampled rows are gathered into a [BH, nsplit*128, D] query tensor (the same rows
// repeated per KV split) and pushed through the attention kernel three times with split-KV
// items (fp32 partial outputs + LSE), the profiling masks being evaluated analytically on the fly
// (MASK_PROF_*; the reference materialises two [10000, S] fp32 masks = 2 x 4.76 GB at HY 720p).
// A combine kernel merges the splits and reduces the MSE.  K and V are read three times out of L2/HBM
// (3 x 1.46 GB at HY 720p); everything else is a few MB.
#include "../../include/svgb200.h"
#include "attn_common.cuh"
#include "host_common.h"

namespace svgb {

__global__ void smse_gather_kernel(const uint4* __restrict__ q, const int* __restrict__ rows, int n_rows,
                                   int nsplit, int S, int vec_per_row, uint4* __restrict__ qg,
                                   int* __restrict__ q_index) {
  // qg[bh, s*128 + r, :] = q[bh, rows[r], :] (zero rows for r >= n_rows)
  const int bh = blockIdx.y;
  const int total = nsplit * 128 * vec_per_row;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int row = i / vec_per_row, vc = i - row * vec_per_row;
    const int r = row & 127;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (r < n_rows) v = q[(static_cast<size_t>(bh) * S + rows[r]) * vec_per_row + vc];
    qg[(static_cast<size_t>(bh) * nsplit * 128 + row) * vec_per_row + vc] = v;
    if (bh == 0 && vc == 0) q_index[row] = r < n_rows ? rows[r] : 0;
  }
}

__global__ void smse_plan_kernel(int S, int nsplit, int n_chunks, int* counts, int4* items, int2* chunks_plain,
                                 int2* chunks_elem) {
  const int cps = (n_chunks + nsplit - 1) / nsplit;
  for (int c = threadIdx.x; c < n_chunks; c += blockDim.x) {
    const int valid = min(kChunkCols, S - c * kChunkCols);
    chunks_plain[c] = make_int2(c * kChunkCols, chunk_meta(valid, false));
    chunks_elem[c] = make_int2(c * kChunkCols, chunk_meta(valid, true));
  }
  for (int s = threadIdx.x; s < nsplit; s += blockDim.x) {
    const int c0 = min(n_chunks, s * cps), c1 = min(n_chunks, c0 + cps);
    put_item(items + 2 * s, s * 128, 128, c0, c1 - c0);
  }
  if (threadIdx.x == 0) counts[0] = nsplit;
}

// merge split-KV partials and reduce the squared error.  grid (BH, kCombineParts): block (bh, p) handles
// the sampled rows r with r % kCombineParts == p and writes one partial sum per mask; a second tiny kernel
// adds the partials in a fixed order (deterministic).
constexpr int kCombineParts = 8;

__global__ void __launch_bounds__(256)
smse_combine_kernel(const float* __restrict__ o_part, const float* __restrict__ lse_part, int nsplit,
                    int n_rows, int D, int BH, float* __restrict__ partial) {
  // o_part: [3][BH][nsplit*128][D]; lse_part: [3][BH][nsplit*128]; partial: [2][BH][kCombineParts]
  const int bh = blockIdx.x, part = blockIdx.y;
  const size_t rows_per_head = static_cast<size_t>(nsplit) * 128;
  const size_t var_stride_o = static_cast<size_t>(BH) * rows_per_head * D;
  const size_t var_stride_l = static_cast<size_t>(BH) * rows_per_head;
  __shared__ float red[2][8];
  float acc0 = 0.f, acc1 = 0.f;
  const int my_rows = (n_rows - part + kCombineParts - 1) / kCombineParts;
  for (int e = threadIdx.x; e < my_rows * D; e += blockDim.x) {
    const int r = part + (e / D) * kCombineParts, d = e % D;
    float outv[3];
#pragma unroll
    for (int var = 0; var < 3; ++var) {
      const float* lp = lse_part + var * var_stride_l + bh * rows_per_head;
      const float* op = o_part + var * var_stride_o + (bh * rows_per_head) * D;
      float m = -INFINITY;
      for (int s = 0; s < nsplit; ++s) m = fmaxf(m, lp[s * 128 + r]);
      float num = 0.f, den = 0.f;
      for (int s = 0; s < nsplit; ++s) {
        const float l = lp[s * 128 + r];
        const float w = (l == -INFINITY) ? 0.f : __expf(l - m);
        num += w * op[(static_cast<size_t>(s) * 128 + r) * D + d];
        den += w;
      }
      outv[var] = den > 0.f ? num / den : 0.f;
    }
    const float d0 = outv[1] - outv[0], d1 = outv[2] - outv[0];
    acc0 += d0 * d0;
    acc1 += d1 * d1;
  }
  for (int o = 16; o > 0; o >>= 1) {
    acc0 += __shfl_xor_sync(0xffffffffu, acc0, o);
    acc1 += __shfl_xor_sync(0xffffffffu, acc1, o);
  }
  if ((threadIdx.x & 31) == 0) {
    red[0][threadIdx.x >> 5] = acc0;
    red[1][threadIdx.x >> 5] = acc1;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = 0.f, b = 0.f;
    for (int w = 0; w < 8; ++w) {
      a += red[0][w];
      b += red[1][w];
    }
    partial[(0 * BH + bh) * kCombineParts + part] = a;
    partial[(1 * BH + bh) * kCombineParts + part] = b;
  }
}

__global__ void smse_final_kernel(const float* __restrict__ partial, int BH, int n_rows, int D, float* __restrict__ mse) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;  // (mask, bh)
  if (i >= 2 * BH) return;
  float s = 0.f;
  for (int p = 0; p < kCombineParts; ++p) s += partial[i * kCombineParts + p];
  mse[i] = s / (static_cast<float>(n_rows) * D);
}

struct SmseLayout {
  int nsplit, n_chunks;
  size_t qg, qidx, counts, items, chunks_plain, chunks_elem, o_part, lse_part, partial, total;
};
// n_sms: SM count of the current device.  The attention kernel fits one CTA per SM (its shared memory), so
// BH * nsplit <= n_sms keeps each pass to one wave; one CTA more would run as a second wave and double the pass.
static SmseLayout smse_layout(int BH, int S, int D, int n_sms) {
  SmseLayout L;
  L.n_chunks = (S + kChunkCols - 1) / kChunkCols;
  L.nsplit = n_sms / BH;
  if (L.nsplit > 32) L.nsplit = 32;  // few heads (per-head pipelines): keep the merge cheap
  if (L.nsplit > L.n_chunks) L.nsplit = L.n_chunks;
  if (L.nsplit < 1) L.nsplit = 1;
  size_t o = 0;
  auto take = [&](size_t b) {
    size_t at = o;
    o += align_up(b, 256);
    return at;
  };
  const size_t rows = static_cast<size_t>(L.nsplit) * 128;
  L.qg = take(2ull * BH * rows * D);
  L.qidx = take(4 * rows);
  L.counts = take(256);
  L.items = take(2 * sizeof(int4) * L.nsplit);
  L.chunks_plain = take(sizeof(int2) * L.n_chunks);
  L.chunks_elem = take(sizeof(int2) * L.n_chunks);
  L.o_part = take(4ull * 3 * BH * rows * D);
  L.lse_part = take(4ull * 3 * BH * rows);
  L.partial = take(4ull * 2 * BH * kCombineParts);
  L.total = o;
  return L;
}

static int device_sms(int* n_sms) {
  int dev = 0;
  SVGB_CUDA(cudaGetDevice(&dev));
  SVGB_CUDA(cudaDeviceGetAttribute(n_sms, cudaDevAttrMultiProcessorCount, dev));
  return 0;
}

}  // namespace svgb

using namespace svgb;

extern "C" {

int svgb_sample_mse_bytes(int BH, int S, int D, int n_rows, size_t* bytes) {
  SVGB_REQUIRE(BH > 0 && S > 0 && (D == 64 || D == 128) && n_rows > 0 && n_rows <= 128 && bytes,
               "bad arguments (n_rows <= 128, D in {64,128})");
  int n_sms = 0;
  if (device_sms(&n_sms)) return -1;
  *bytes = smse_layout(BH, S, D, n_sms).total;
  return 0;
}

int svgb_sample_mse(const void* q, const void* k, const void* v, const int32_t* rows, int n_rows,
                    int BH, int S, int D, int dtype, int layout, int ctx, int F, int P, float* mse,
                    void* ws, size_t ws_bytes, void* stream) {
  // every check on the arguments alone comes before the device query and the first launch
  SVGB_REQUIRE(q && k && v && rows && mse && ws, "null pointer");
  // the gather moves 2-byte elements and the attention passes run without fp8 scales
  SVGB_REQUIRE(dtype == SVGB_BF16 || dtype == SVGB_F16,
               "sample_mse takes 16-bit q/k/v only: SVGB_BF16 or SVGB_F16, not dtype %d", dtype);
  SVGB_REQUIRE(layout >= 0 && layout <= 2, "layout %d unsupported (0 = HY text-last, 1 = WAN, 2 = COG text-first)", layout);
  SVGB_REQUIRE(ctx >= 0 && F > 0 && P > 0, "bad sequence layout ctx %d, F %d, P %d", ctx, F, P);
  SVGB_REQUIRE(static_cast<long long>(S) == ctx + static_cast<long long>(F) * P, "seq_len %d != ctx %d + F %d * P %d",
               S, ctx, F, P);
  SVGB_REQUIRE(layout != 1 || ctx == 0, "WAN layout has no text tokens");
  SVGB_REQUIRE(layout != 2 || ctx < (1 << 19), "COG layout: context length %d too large", ctx);
  // reference thresholds: block_thres // block_size with block_thres = 1.5*P (HY, COG) or 2*P (WAN)
  const int thres = layout == 1 ? static_cast<int>((2LL * P) / 128) : static_cast<int>((1.5 * P) / 128.0);
  SVGB_REQUIRE(thres < (1 << 12), "profiling band threshold %d too large", thres);
  size_t need = 0;
  if (svgb_sample_mse_bytes(BH, S, D, n_rows, &need)) return -1;
  SVGB_REQUIRE(ws_bytes >= need, "workspace too small: %zu < %zu", ws_bytes, need);
  int n_sms = 0;
  if (device_sms(&n_sms)) return -1;
  const SmseLayout L = smse_layout(BH, S, D, n_sms);  // the same device, so the same layout as the byte count
  char* w = static_cast<char*>(ws);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int vpr = D * 2 / 16;
  const int rows_per_head = L.nsplit * 128;
  smse_gather_kernel<<<dim3(8, BH), 256, 0, st>>>(static_cast<const uint4*>(q), rows, n_rows, L.nsplit, S, vpr,
                                                   reinterpret_cast<uint4*>(w + L.qg),
                                                   reinterpret_cast<int*>(w + L.qidx));
  SVGB_LAUNCH_OK();
  smse_plan_kernel<<<1, 256, 0, st>>>(S, L.nsplit, L.n_chunks, reinterpret_cast<int*>(w + L.counts),
                                      reinterpret_cast<int4*>(w + L.items),
                                      reinterpret_cast<int2*>(w + L.chunks_plain),
                                      reinterpret_cast<int2*>(w + L.chunks_elem));
  SVGB_LAUNCH_OK();
  static const int kModes[3][2] = {{MASK_PROF_HY_S, MASK_PROF_HY_T}, {MASK_PROF_WAN_S, MASK_PROF_WAN_T},
                                   {MASK_PROF_COG_S, MASK_PROF_COG_T}};
  for (int var = 0; var < 3; ++var) {
    AttnArgs a;
    a.items = reinterpret_cast<const int4*>(w + L.items);
    a.item_count = reinterpret_cast<const int*>(w + L.counts);
    a.chunks = reinterpret_cast<const int2*>(w + (var == 0 ? L.chunks_plain : L.chunks_elem));
    a.o = w + L.o_part + 4ull * var * BH * rows_per_head * D;
    a.o_row_stride = D;
    a.o_head_stride = static_cast<long long>(rows_per_head) * D;
    a.lse = reinterpret_cast<float*>(w + L.lse_part) + static_cast<size_t>(var) * BH * rows_per_head;
    a.scale_log2 = 1.4426950408889634f / sqrtf(static_cast<float>(D));
    a.S = rows_per_head;
    a.mask_mode = var == 0 ? MASK_NONE : kModes[layout][var - 1];
    a.m0 = F;
    a.m1 = P;
    a.m2 = layout == 2 ? (thres | (ctx << 12)) : thres;
    a.q_index = reinterpret_cast<const int*>(w + L.qidx);
    a.out_f32 = 1;
    const Strides kv = flat_strides(D, static_cast<long long>(S) * D, BH);
    if (attn_fwd_impl(w + L.qg, flat_strides(D, static_cast<long long>(rows_per_head) * D, BH), rows_per_head, k, kv,
                      v, kv, S, dtype, 1, BH, D, a, false, L.nsplit, st))
      return -1;
  }
  smse_combine_kernel<<<dim3(BH, kCombineParts), 256, 0, st>>>(
      reinterpret_cast<const float*>(w + L.o_part), reinterpret_cast<const float*>(w + L.lse_part), L.nsplit,
      n_rows, D, BH, reinterpret_cast<float*>(w + L.partial));
  SVGB_LAUNCH_OK();
  smse_final_kernel<<<(2 * BH + 127) / 128, 128, 0, st>>>(reinterpret_cast<const float*>(w + L.partial), BH, n_rows,
                                                           D, mse);
  SVGB_LAUNCH_OK();
  return 0;
}

}  // extern "C"
