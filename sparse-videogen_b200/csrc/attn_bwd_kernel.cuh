// Block-sparse flash attention backward for sm_90a (Hopper wgmma).  DESIGN.md §5 has the derivation, the FLOP count
// and the shared-memory budget.
//
// Two launches of one kernel template, neither with atomics, so the gradients are deterministic:
//   query-major (kKeyMajor = false), over the forward plan : one CTA per query item, dQ      += dS  K
//   key-major   (kKeyMajor = true),  over the key-major plan: one CTA per key item,   dK      += dS^T Q,  dV += P^T dO
// Every query row lives in exactly one stream of the forward plan and every key in exactly one stream of the key-major
// plan, so each gradient row is summed by one warpgroup in a fixed order and stored once.
//
// The two directions are the same computation with the roles of the tiles swapped.  A stream holds the STATIONARY
// tiles X, Y (128 rows each) and walks the chunk list, loading the STREAMED tiles U, W (128 rows each) per chunk:
//   query-major: X = Q, Y = dO, U = K, W = V        key-major: X = K, Y = V, U = Q, W = dO
// Per chunk, in two halves of 64 columns (m64n64 score tiles keep the key-major kernel's four accumulator sets inside
// the register file), each consumer warpgroup (64 rows of X) computes
//   S  = X U^T, dP = Y W^T                      wgmma m64n64k16, SS (both K-major)
//   P  = exp2(S * scale_log2 - lse * log2 e)    lse of the query (row or column), from the forward
//   dS = P * (dP - delta)                       delta = rowsum(dO * O) of the query
//   A1 += dS U  (dQ or dK),  A2 += P W (dV)     wgmma m64nDk16, RS (dS, P from registers, U / W MN-major)
// Masked entries and columns past the chunk's valid count get P = dS = 0.  ELEM chunks evaluate mask_allowed with the
// query position first in both directions (segment plans: relative to the stream's segment, seg_origin).  A row without
// any allowed key has lse = -inf and gets P = 0 on every column, so its dQ is exactly 0; a key that no query reaches
// gets an empty list and dK = dV = 0.
//
// 256 threads, two warpgroups, no producer warpgroup: thread 0 issues the TMA loads, the stationary pair once per
// stream and the streamed pair of chunk j + 2 into the stage chunk j leaves, after a block barrier that follows the
// last wgmma reading it.  The tiles, their 128-byte swizzle, the descriptors and the wgmma wrappers are the forward's.
#pragma once
#include "attn_kernel.cuh"

namespace svgb {

struct AttnBwdArgs {
  const int4* items = nullptr;      // the plan's two stream descriptors per item (attn_common.cuh)
  const int* item_count = nullptr;  // [BH] when items_stride != 0, else [1]
  const int2* chunks = nullptr;     // chunk lists
  int items_stride = 0;
  // query heads per key/value head (grouped-query attention).  Query-major: CTA head bh is a query head, its plan and
  // K / V are at bh / kv_group.  Key-major: bh is a key/value head with its own plan, and each stream walks its chunk
  // list once for every query head bh * kv_group + g of the group.
  int kv_group = 1;
  // heads of the stationary tiles per batch element (query-major: Hq, key-major: Hkv): CTA head bh is head bh % Hx of
  // batch element bh / Hx in the tensor maps (d, row, head, batch) and the gradient stores; the plan, LSE and delta
  // index the flat head
  int Hx = 1;
  const float* lse = nullptr;    // [BH, S] natural-log LSE of the forward (query rows)
  const float* delta = nullptr;  // [BH, S] rowsum(dO * O)
  void* g0 = nullptr;            // query-major: dQ; key-major: dK
  void* g1 = nullptr;            // key-major: dV
  long long g0_bs = 0, g0_hs = 0, g0_rs = 0;  // element strides (batch, head, row) of g0
  long long g1_bs = 0, g1_hs = 0, g1_rs = 0;  // and of g1
  float scale_log2 = 0, sm_scale = 0;
  int S = 0;
  int mask_mode = 0, m0 = 0, m1 = 0, m2 = 0;
  // segment plans: the plan's copy of the bounds {nseg, cq[0..nseg], ck[0..nseg]} (seg_origin); nullptr otherwise
  const int* segs = nullptr;
};

template <int D>
struct AttnBwdCfg {
  static constexpr int kTileBytes = AttnCfg<D, DT_BF16>::kTileBytes;
  // X, Y, and two stages of (U, W); + 1 KB for the alignment of the dynamic window, + 1 KB for the mbarriers
  static constexpr int kSmemBytes = 1024 + 6 * kTileBytes + 1024;
  static constexpr int kThreads = 256;
  static_assert(kSmemBytes <= 227 * 1024, "exceeds the 227 KB per-CTA shared memory of sm_90");
};

// S[64 x 64] = A[64 rows, K-major] B[64 rows, K-major]^T over the head dimension, one warpgroup, one wgmma group
template <int D, bool kBF16>
__device__ __forceinline__ void bwd_score_issue(float (&s)[32], uint32_t sA, uint32_t sB) {
  using Cfg = AttnCfg<D, DT_BF16>;
#pragma unroll
  for (int i = 0; i < 32; ++i) s[i] = 0.f;
  wg_fence();
#pragma unroll
  for (int kk = 0; kk < Cfg::kKSteps; ++kk) {
    const uint32_t off = (kk >> 2) * Cfg::kPanelBytes + (kk & 3) * 32;
    wgmma_m64n64k16_ss<kBF16>(s, wg_desc_kmajor(sA + off), wg_desc_kmajor(sB + off), kk > 0);
  }
}

// acc[64 x D] += A[64 x 64, registers] B[64 rows x D, MN-major] (issued into the open wgmma group)
template <int D, bool kBF16>
__device__ __forceinline__ void bwd_acc_issue(float (&acc)[D / 2], const uint32_t (&a)[4][4], uint32_t sB) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    const uint64_t b = wg_desc_mnmajor(sB + kk * 2048, 128 * 128);
    if constexpr (D == 128) wgmma_m64n128k16_rs<kBF16>(acc, a[kk], b, 1);
    else wgmma_m64n64k16_rs<kBF16>(acc, a[kk], b, 1);
  }
}

template <bool kBF16>
__device__ __forceinline__ void bwd_pack(uint32_t (&a)[4][4], const float (&x)[32]) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk)
#pragma unroll
    for (int r = 0; r < 4; ++r) a[kk][r] = pack2<kBF16>(x[8 * kk + 2 * r], x[8 * kk + 2 * r + 1]);
}

// log2-domain LSE of a query: +inf for a query without keys (lse = -inf), so that exp2(s - lse2) = 0
__device__ __forceinline__ float bwd_lse2(float lse) {
  return lse == -INFINITY ? INFINITY : lse * 1.4426950408889634f;
}

template <int D, int DT, bool kKeyMajor>
__global__ void __launch_bounds__(256, 1)
attn_bwd_kernel(const __grid_constant__ CUtensorMap xmap, const __grid_constant__ CUtensorMap ymap,
                const __grid_constant__ CUtensorMap umap, const __grid_constant__ CUtensorMap wmap,
                const AttnBwdArgs args) {
  static_assert(DT == DT_BF16 || DT == DT_F16, "the backward takes 16-bit inputs");
  using Cfg = AttnCfg<D, DT>;
  constexpr bool BF16 = DT == DT_BF16;
  constexpr int kTile = Cfg::kTileBytes;
  const int bh = blockIdx.y;  // head of the stationary tiles X, Y and of the gradients this CTA stores
  const int G = args.kv_group;
  const int ph = kKeyMajor ? bh : bh / G;  // head of the plan (a key/value head)
  // batch element and head within it of the stationary tiles; the streamed tiles are in the same batch element
  const int batch = bh / args.Hx, xh = bh - batch * args.Hx;
  const int n_items = args.item_count[args.items_stride ? ph : 0];
  if (static_cast<int>(blockIdx.x) >= n_items) return;
  const int4* desc = args.items + 2 * (static_cast<size_t>(ph) * args.items_stride + blockIdx.x);

  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_u32 = smem_u32(smem_raw);
  const uint32_t base = (raw_u32 + 1023u) & ~1023u;
  uint8_t* smem_al = smem_raw + (base - raw_u32);
  const uint32_t sX = base, sY = sX + kTile;
  const uint32_t sU0 = sY + kTile;  // stage b: U at sU0 + 2b * tile, W right after it
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem_al + 6 * kTile);  // [0] X and Y, [1 + b] U and W of stage b
  const uint32_t bar_xy = smem_u32(&bar[0]);

  const int tid = threadIdx.x;
  const int wg = tid >> 7, lane = tid & 31, wq = (tid >> 5) & 3;
  if (tid == 0) {
    for (int i = 0; i < 3; ++i) mbar_init(smem_u32(&bar[i]), 1);
    mbar_fence_init();
    tma_prefetch_desc(&xmap);
    tma_prefetch_desc(&ymap);
    tma_prefetch_desc(&umap);
    tma_prefetch_desc(&wmap);
  }
  __syncthreads();

  // thread 0: the two tiles of `row` (rows row .. row + 127 of head `head` of this CTA's batch element) into dst0 /
  // dst1, on one barrier
  auto load_pair = [&](uint32_t b, uint32_t dst0, const CUtensorMap* m0, uint32_t dst1, const CUtensorMap* m1, int row,
                       int head) {
    mbar_expect_tx(b, 2 * kTile);
    for (int h = 0; h < Cfg::kHalves; ++h) {
      tma_load_4d(dst0 + h * Cfg::kPanelBytes, m0, b, h * Cfg::kPanelElems, row, head, batch);
      tma_load_4d(dst1 + h * Cfg::kPanelBytes, m1, b, h * Cfg::kPanelElems, row, head, batch);
    }
  };
  auto stage_u = [&](int n) { return sU0 + 2 * (n & 1) * kTile; };
  auto bar_u = [&](int n) { return smem_u32(&bar[1 + (n & 1)]); };

  const float c = args.scale_log2;
  const int mode = args.mask_mode, m0 = args.m0, m1 = args.m1, m2 = args.m2;
  // this thread's accumulator rows: rloc and rloc + 8 of the stream's 128; columns 8j + 2 * (lane % 4) (+1)
  const int rloc = 64 * wg + 16 * wq + (lane >> 2);
  const uint32_t sXw = sX + 64 * wg * 128, sYw = sY + 64 * wg * 128;

  const int nstreams = __ldg(&desc[1].y) > 0 ? 2 : 1;
  int n = 0;   // chunks of the earlier streams (stage n & 1, phase (n >> 1) & 1)
  int nx = 0;  // stationary tile pairs loaded so far (phase of bar[0])
  for (int st = 0; st < nstreams; ++st) {
    const int4 d = __ldg(&desc[st]);
    const int r0 = d.x, nr = d.y, nch = d.w;
    const int2* __restrict__ chunks = args.chunks + d.z;
    // segment plans: the stream's segment shifts the query positions (the rows, key-major the columns), and the mask
    // sees both positions relative to the segment's first key, where its block grid is anchored (seg_origin)
    SegOrigin so{0, m0};
    if (args.segs) so = seg_origin(args.segs, r0, kKeyMajor, m0);
    const int q_off = so.shift + so.key0, sink_rel = so.sink_end - so.key0;
    // step t of the stream takes chunk t % nch of the streamed tiles' head uhead(t): the query-major kernel walks the
    // list once (K / V of head bh / G), the key-major kernel once per query head of the group, g = t / nch in order
    const int steps = kKeyMajor ? G * nch : nch;
    auto uhead = [&](int t) { return kKeyMajor ? xh * G + t / nch : xh / G; };
    if (tid == 0 && nch > 0) {
      load_pair(bar_xy, sX, &xmap, sY, &ymap, r0, xh);
      for (int t = 0; t < 2 && t < steps; ++t) {
        const uint32_t su = stage_u(n + t);
        load_pair(bar_u(n + t), su, &umap, su + kTile, &wmap, __ldg(&chunks[t % nch].x), uhead(t));
      }
    }
    // query-major: the rows are queries, their lse / delta are fixed for the stream (rows past nr: P = 0)
    float lse_r[2] = {0.f, 0.f}, dl_r[2] = {0.f, 0.f};
    if constexpr (!kKeyMajor) {
      const size_t qbase = static_cast<size_t>(bh) * args.S;
#pragma unroll
      for (int v1 = 0; v1 < 2; ++v1) {
        const int row = rloc + 8 * v1;
        lse_r[v1] = row < nr ? bwd_lse2(__ldg(&args.lse[qbase + r0 + row])) : INFINITY;
        dl_r[v1] = row < nr ? __ldg(&args.delta[qbase + r0 + row]) : 0.f;
      }
    }
    float acc1[D / 2], acc2[kKeyMajor ? D / 2 : 1];
#pragma unroll
    for (int i = 0; i < D / 2; ++i) acc1[i] = 0.f;
#pragma unroll
    for (int i = 0; i < (kKeyMajor ? D / 2 : 1); ++i) acc2[i] = 0.f;

    if (nch > 0) mbar_wait(bar_xy, nx & 1, 21);
    // key-major: lse / delta of the step's query head (the columns are its queries)
    const float* lse_h = args.lse + static_cast<size_t>(bh) * G * args.S;
    const float* dl_h = args.delta + static_cast<size_t>(bh) * G * args.S;
    for (int t = 0, j = 0; t < steps; ++t) {
      const int nn = n + t;
      const int2 ch = __ldg(&chunks[j]);
      const int c0 = ch.x, valid = chunk_valid(ch.y);
      const bool elem = (ch.y & kChunkElem) != 0;
      const uint32_t sU = stage_u(nn), sW = sU + kTile;
      mbar_wait(bar_u(nn), (nn >> 1) & 1, 22);
#pragma unroll 1
      for (int h = 0; h < 2 && 64 * h < valid; ++h) {
        float s[32], dp[32];
        bwd_score_issue<D, BF16>(s, sXw, sU + h * 64 * 128);
        bwd_score_issue<D, BF16>(dp, sYw, sW + h * 64 * 128);
        wg_commit();
        attn_wait<0>(s);
        wg_fence_regs(dp);
#pragma unroll
        for (int jj = 0; jj < 8; ++jj)
#pragma unroll
          for (int v0 = 0; v0 < 2; ++v0) {
            const int col = 64 * h + 8 * jj + 2 * (lane & 3) + v0;
            const bool in = col < valid;
            float lse_c = INFINITY, dl_c = 0.f;
            if constexpr (kKeyMajor) {  // the columns are queries
              if (in) {
                lse_c = bwd_lse2(__ldg(&lse_h[c0 + col]));
                dl_c = __ldg(&dl_h[c0 + col]);
              }
            }
#pragma unroll
            for (int v1 = 0; v1 < 2; ++v1) {
              const int i = 4 * jj + 2 * v1 + v0;
              bool ok = in;
              if (elem && ok) {
                const int rp = r0 + rloc + 8 * v1, cp = c0 + col;
                ok = kKeyMajor ? mask_allowed(mode, cp - q_off, rp - so.key0, sink_rel, m1, m2)
                               : mask_allowed(mode, rp - q_off, cp - so.key0, sink_rel, m1, m2);
              }
              const float l2 = kKeyMajor ? lse_c : lse_r[v1];
              const float dl = kKeyMajor ? dl_c : dl_r[v1];
              const float p = ok ? ex2_approx(fmaf(s[i], c, -l2)) : 0.f;
              s[i] = p;
              dp[i] = p * (dp[i] - dl);
            }
          }
        uint32_t ds_a[4][4], p_a[4][4];
        bwd_pack<BF16>(ds_a, dp);
        if constexpr (kKeyMajor) bwd_pack<BF16>(p_a, s);
        wg_fence();
        bwd_acc_issue<D, BF16>(acc1, ds_a, sU + h * 64 * 128);
        if constexpr (kKeyMajor) bwd_acc_issue<D, BF16>(acc2, p_a, sW + h * 64 * 128);
        wg_commit();
        attn_wait<0>(acc1);
        wg_fence_regs(acc2);
      }
      __syncthreads();  // both warpgroups' wgmma on this stage have retired: refill it with step t + 2
      if (tid == 0 && t + 2 < steps) {
        load_pair(bar_u(nn + 2), sU, &umap, sW, &wmap, __ldg(&chunks[(t + 2) % nch].x), uhead(t + 2));
      }
      if (++j == nch) {  // key-major: on to the next query head of the group
        j = 0;
        lse_h += args.S;
        dl_h += args.S;
      }
    }
    n += steps;
    nx += nch > 0;

    // ---- epilogue: A1 * sm_scale (dQ or dK), A2 (dV); rows past nr belong to other streams
#pragma unroll
    for (int v1 = 0; v1 < 2; ++v1) {
      const int row = rloc + 8 * v1;
      if (row >= nr) continue;
      const long long r = r0 + row, c0 = 2 * (lane & 3);
      uint16_t* g0 = reinterpret_cast<uint16_t*>(args.g0) + batch * args.g0_bs + xh * args.g0_hs + r * args.g0_rs + c0;
#pragma unroll
      for (int jj = 0; jj < D / 8; ++jj)
        *reinterpret_cast<uint32_t*>(g0 + 8 * jj) =
            pack2<BF16>(acc1[4 * jj + 2 * v1] * args.sm_scale, acc1[4 * jj + 2 * v1 + 1] * args.sm_scale);
      if constexpr (kKeyMajor) {
        uint16_t* g1 = reinterpret_cast<uint16_t*>(args.g1) + batch * args.g1_bs + xh * args.g1_hs + r * args.g1_rs + c0;
#pragma unroll
        for (int jj = 0; jj < D / 8; ++jj)
          *reinterpret_cast<uint32_t*>(g1 + 8 * jj) = pack2<BF16>(acc2[4 * jj + 2 * v1], acc2[4 * jj + 2 * v1 + 1]);
      }
    }
  }
}

// delta[bh, s] = sum_d dO[bh, s, d] * O[bh, s, d] in fp32: one warp per row; head bh is head bh % H of batch element
// bh / H in o and dO, each at its own element strides (batch, head, row)
template <bool kBF16>
__global__ void __launch_bounds__(256)
attn_bwd_delta_kernel(const uint16_t* __restrict__ o, const uint16_t* __restrict__ dout, long long o_bs, long long o_hs,
                      long long o_rs, long long do_bs, long long do_hs, long long do_rs, int BH, int H, int S, int D,
                      float* __restrict__ delta) {
  const long long r = static_cast<long long>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  if (r >= static_cast<long long>(BH) * S) return;
  const int lane = threadIdx.x & 31;
  const long long bh = r / S, s = r - bh * S, b = bh / H, h = bh - b * H;
  const uint16_t* orow = o + b * o_bs + h * o_hs + s * o_rs;
  const uint16_t* drow = dout + b * do_bs + h * do_hs + s * do_rs;
  float acc = 0.f;
  for (int d = 2 * lane; d < D; d += 64) {
    const uint32_t x = *reinterpret_cast<const uint32_t*>(orow + d);
    const uint32_t y = *reinterpret_cast<const uint32_t*>(drow + d);
    float2 fa, fb;
    if constexpr (kBF16) {
      fa = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&x));
      fb = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&y));
    } else {
      fa = __half22float2(*reinterpret_cast<const __half2*>(&x));
      fb = __half22float2(*reinterpret_cast<const __half2*>(&y));
    }
    acc = fmaf(fa.x, fb.x, fmaf(fa.y, fb.y, acc));
  }
#pragma unroll
  for (int m = 16; m > 0; m >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, m);
  if (lane == 0) delta[r] = acc;
}

}  // namespace svgb
