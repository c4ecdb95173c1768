// Block-sparse flash attention forward for sm_90a (Hopper wgmma).
//
// One CTA per work item, 256 threads = two consumer warpgroups; warpgroup w owns query rows 64w .. 64w+63 of a
// 128-row tile.  A work item is one or two 128-row STREAMS (a two-tile item: rows 0-127 and 128-255 over the same
// chunk list; a dual item: two independent tails, each with its own chunk list), run one after the other.
//   Q tile          : TMA (or cp.async row gather), 128-byte swizzle, stays in shared memory for the stream
//   K(j), V(j)      : double-buffered; chunk j+1 is loaded while chunk j is computed
//   S = Q K^T       : wgmma m64n128 (SS, both operands K-major), fp32 accumulators in registers
//   softmax         : online, in registers (each row is spread over the 4 lanes of a quad)
//   O += P V        : wgmma m64nD (RS: P from registers in the accumulator layout of S, V MN-major)
// FP8 (e4m3) inputs: Q K^T runs on e4m3 wgmma (k32); wgmma has no MN-major 8-bit B operand, so each V tile is
// widened to fp16 in shared memory and P V runs in fp16.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>

#include "attn_common.cuh"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace svgb {

// element type of Q/K/V: 0 = bf16, 1 = fp16, 2 = fp8 e4m3 (output bf16)
constexpr int DT_BF16 = 0, DT_F16 = 1, DT_E4M3 = 2;

template <int D, int DT = DT_BF16>
struct AttnCfg {
  static_assert(D == 64 || D == 128, "head_dim must be 64 or 128");
  static_assert(DT != DT_E4M3 || D == 128, "the e4m3 path is built for head_dim 128 (128-byte rows)");
  static constexpr int kElemBytes = DT == DT_E4M3 ? 1 : 2;
  static constexpr int kRowBytes = D * kElemBytes;
  static constexpr int kHalves = kRowBytes / 128;        // 128-byte swizzle panels per row
  static constexpr int kPanelElems = 128 / kElemBytes;   // elements per panel row (TMA box width)
  static constexpr int kPanelBytes = 128 * 128;          // 128 rows x 128 B
  static constexpr int kTileBytes = kPanelBytes * kHalves;
  static constexpr int kKSteps = kRowBytes / 32;         // wgmma K steps of Q K^T (32 bytes each)
  static constexpr int kVhBytes = DT == DT_E4M3 ? 2 * kPanelBytes : 0;  // fp16 copy of the e4m3 V tile
  static constexpr int kMaxRunsSmem = kTileBytes / 8 - 1;
  static constexpr int kBarBytes = 1024;                 // mbarriers + gather row table
  // + 1 KB: the kernel aligns the dynamic window to 1024 bytes itself
  static constexpr int kSmemBytes = 1024 + kTileBytes + 4 * kTileBytes + kVhBytes + kBarBytes;
  static constexpr int kThreads = 256;
  static_assert(kSmemBytes <= 227 * 1024, "exceeds the 227 KB per-CTA shared memory of sm_90");
};

// S[64 x 128] = Q[64 rows of the tile] K^T for one warpgroup
template <int D, int DT>
__device__ __forceinline__ void attn_qk(float (&s)[64], uint32_t sQw, uint32_t sK) {
  using Cfg = AttnCfg<D, DT>;
#pragma unroll
  for (int i = 0; i < 64; ++i) s[i] = 0.f;
  wg_fence();
#pragma unroll
  for (int kk = 0; kk < Cfg::kKSteps; ++kk) {
    const uint32_t off = (kk >> 2) * Cfg::kPanelBytes + (kk & 3) * 32;
    const uint64_t a = wg_desc_kmajor(sQw + off), b = wg_desc_kmajor(sK + off);
    if constexpr (DT == DT_E4M3) wgmma_m64n128k32_e4m3_ss(s, a, b, kk > 0);
    else wgmma_m64n128k16_ss<DT == DT_BF16>(s, a, b, kk > 0);
  }
  wg_commit();
  wg_wait<0>();
  wg_fence_regs(s);
}

// O[64 x D] += P[64 x 128] V[128 x D]; P in the accumulator layout of S, packed to 16 bit (kBF16: bf16, else fp16)
template <int D, bool kBF16>
__device__ __forceinline__ void attn_pv(float (&o)[D / 2], const float (&p)[64], uint32_t sV) {
  uint32_t a[8][4];
#pragma unroll
  for (int kk = 0; kk < 8; ++kk)
#pragma unroll
    for (int r = 0; r < 4; ++r) a[kk][r] = pack2<kBF16>(p[8 * kk + 2 * r], p[8 * kk + 2 * r + 1]);
  wg_fence();
#pragma unroll
  for (int kk = 0; kk < 8; ++kk) {
    const uint64_t b = wg_desc_mnmajor(sV + kk * 2048, 128 * 128);
    if constexpr (D == 128) wgmma_m64n128k16_rs<kBF16>(o, a[kk], b, 1);
    else wgmma_m64n64k16_rs<kBF16>(o, a[kk], b, 1);
  }
  wg_commit();
  wg_wait<0>();
  wg_fence_regs(o);
}

struct AttnSmemCtl {
  uint64_t q_full;
  uint64_t kv_full[2];
  int src[128];  // gather: source row of each of the 128 rows being loaded (-1: zero fill)
};

// kGather selects the loader: false = TMA boxes over contiguous key ranges (chunk list), true = cp.async
// row gathers over a run list.
template <int D, int DT, bool kGather>
__global__ void __launch_bounds__(256, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap qmap, const __grid_constant__ CUtensorMap kmap,
                const __grid_constant__ CUtensorMap vmap, const AttnArgs args) {
  using Cfg = AttnCfg<D, DT>;
  constexpr bool BF16 = DT != DT_F16;  // output format (fp8 inputs produce bf16 output)
  constexpr bool FP8 = DT == DT_E4M3;
  constexpr bool kPBF16 = DT == DT_BF16;  // format of P and V in the P V product (fp8: fp16)
  static_assert(!(FP8 && kGather), "row-gather loads are 16-bit only");
  const int bh = blockIdx.y;
  const int n_items = args.item_count[bh * args.counts_stride];
  if (static_cast<int>(blockIdx.x) >= n_items) return;
  const size_t item_idx = static_cast<size_t>(bh) * args.items_stride + blockIdx.x;
  const int4 item = args.items[item_idx];
  int4 item2 = make_int4(0, 0, 0, 0);
  if (!kGather && args.items2) item2 = args.items2[item_idx];
  const bool dual = item2.y > 0;
  // gather mode: item.w = number of runs, chunks are implicit (128 selected keys each, last one partial)
  const int total_kv = kGather ? args.item_total[item_idx] : 0;

  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_u32 = smem_u32(smem_raw);
  const uint32_t base = (raw_u32 + 1023u) & ~1023u;
  uint8_t* smem_al = smem_raw + (base - raw_u32);
  const uint32_t sQ = base;
  const uint32_t sK0 = sQ + Cfg::kTileBytes;  // stage s: K at sK0 + 2s*tile, V at sK0 + (2s+1)*tile
  const uint32_t sVh = sK0 + 4 * Cfg::kTileBytes;
  AttnSmemCtl* ctl = reinterpret_cast<AttnSmemCtl*>(smem_al + Cfg::kTileBytes * 5 + Cfg::kVhBytes);

  const int tid = threadIdx.x;
  const int wg = tid >> 7, wt = tid & 127, lane = tid & 31, wq = wt >> 5;
  if (tid == 0) {
    mbar_init(smem_u32(&ctl->q_full), 1);
    mbar_init(smem_u32(&ctl->kv_full[0]), 1);
    mbar_init(smem_u32(&ctl->kv_full[1]), 1);
    mbar_fence_init();
    if constexpr (!kGather) {
      tma_prefetch_desc(&qmap);
      tma_prefetch_desc(&kmap);
      tma_prefetch_desc(&vmap);
    }
  }
  __syncthreads();

  const float c = args.scale_log2 * (args.q_scale ? __ldg(&args.q_scale[bh]) * __ldg(&args.k_scale[bh]) : 1.f);
  const float vs = args.v_scale ? __ldg(&args.v_scale[bh]) : 1.f;
  const int mode = args.mask_mode, m0 = args.m0, m1 = args.m1, m2 = args.m2;
  const uint16_t* kp = static_cast<const uint16_t*>(args.k_ptr) + bh * args.in_head_stride;
  const uint16_t* vp = static_cast<const uint16_t*>(args.v_ptr) + bh * args.in_head_stride;
  const int* kv_rows = (kGather && args.kv_rows) ? args.kv_rows + static_cast<size_t>(bh) * args.S : nullptr;
  const int2* __restrict__ runs = args.chunks + item.z;
  const int nruns = item.w;

  // gather: piece p (16 B) of row r -> panel p/8, byte r*128 + ((p%8) ^ (r%8))*16
  auto gather_rows = [&](uint32_t dst, const uint16_t* src_base, bool two, const uint16_t* src2, uint32_t dst2) {
    constexpr int kPieces = D / 8;
#pragma unroll 4
    for (int i = tid; i < 128 * kPieces; i += 256) {
      const int r = i / kPieces, pc = i % kPieces;
      const int src = ctl->src[r];
      const uint32_t off = (pc >> 3) * Cfg::kPanelBytes + r * 128 + (((pc & 7) ^ (r & 7)) << 4);
      const long long so = static_cast<long long>(src < 0 ? 0 : src) * args.in_row_stride + pc * 8;
      cp_async16(dst + off, src_base + so, src >= 0 ? 16u : 0u);
      if (two) cp_async16(dst2 + off, src2 + so, src >= 0 ? 16u : 0u);
    }
  };
  // gather: source rows of keys j*128 .. j*128+127 of this item -> ctl->src (threads 0..127)
  auto resolve_chunk = [&](int j) {
    if (tid < 128) {
      const int pos = j * kChunkCols + tid;
      int src = -1;
      if (pos < total_kv) {
        int lo = 0, hi = nruns - 1;  // largest run with keys_before <= pos
        while (lo < hi) {
          const int mid = (lo + hi + 1) >> 1;
          if (__ldg(&runs[mid].y) <= pos) lo = mid;
          else hi = mid - 1;
        }
        const int2 rr = __ldg(&runs[lo]);
        const int prow = rr.x + (pos - rr.y);
        src = kv_rows ? __ldg(&kv_rows[prow]) : prow;
      }
      ctl->src[tid] = src;
    }
  };

  int g = 0;       // chunks loaded so far (stage = g & 1, mbarrier phase = (g >> 1) & 1)
  int nq = 0;      // Q tiles loaded so far (q_full phase)
  const int nstreams = (dual || item.y > kTileRows) ? 2 : 1;
  for (int st = 0; st < nstreams; ++st) {
    const bool second = st == 1;
    const int q0 = second ? (dual ? item2.x : item.x + kTileRows) : item.x;
    const int nr = second ? (dual ? item2.y : item.y - kTileRows) : (dual ? item.y : min(item.y, kTileRows));
    const int2* __restrict__ chunks = args.chunks + ((second && dual) ? item2.z : item.z);
    const int nch = kGather ? (total_kv + kChunkCols - 1) / kChunkCols : ((second && dual) ? item2.w : item.w);

    // issue the loads of chunk j into stage `stage`
    auto load_chunk = [&](int j, int stage) {
      const uint32_t sK = sK0 + 2 * stage * Cfg::kTileBytes, sV = sK + Cfg::kTileBytes;
      if constexpr (kGather) {
        resolve_chunk(j);
        __syncthreads();
        gather_rows(sK, kp, true, vp, sV);
        cp_async_commit();
        __syncthreads();  // ctl->src is reused by the next resolve
      } else if (tid == 0) {
        const int kv0 = __ldg(&chunks[j].x);
        const uint32_t fb = smem_u32(&ctl->kv_full[stage]);
        mbar_expect_tx(fb, 2 * Cfg::kTileBytes);
        for (int h = 0; h < Cfg::kHalves; ++h) {
          tma_load_3d(sK + h * Cfg::kPanelBytes, &kmap, fb, h * Cfg::kPanelElems, kv0, bh);
          tma_load_3d(sV + h * Cfg::kPanelBytes, &vmap, fb, h * Cfg::kPanelElems, kv0, bh);
        }
      }
    };

    if (nch > 0) {
      // ---- Q (rows past nr: zero filled by the gather, other rows' data by TMA -- never stored)
      if constexpr (kGather) {
        if (tid < 128) {
          const int* q_rows = args.q_rows ? args.q_rows + static_cast<size_t>(bh) * args.S : nullptr;
          const int qr = q0 + tid;
          ctl->src[tid] = tid < nr ? (q_rows ? __ldg(&q_rows[qr]) : qr) : -1;
        }
        __syncthreads();
        gather_rows(sQ, static_cast<const uint16_t*>(args.q_ptr) + bh * args.in_head_stride, false, nullptr, 0);
        __syncthreads();
      } else if (tid == 0) {
        const uint32_t qb = smem_u32(&ctl->q_full);
        mbar_expect_tx(qb, Cfg::kTileBytes);
        for (int h = 0; h < Cfg::kHalves; ++h) tma_load_3d(sQ + h * Cfg::kPanelBytes, &qmap, qb, h * Cfg::kPanelElems, q0, bh);
      }
      load_chunk(0, g & 1);  // gather: Q and chunk 0 share one cp.async group
    }

    // per thread: rows r0 = 16*wq + lane/4 and r0 + 8 of this warpgroup's 64; columns 8j + 2*(lane%4) (+1)
    const int rloc = 64 * wg + 16 * wq + (lane >> 2);
    ElemMask em;
    if constexpr (!kGather) {  // gather plans carry no element masks
      int qm[2];
#pragma unroll
      for (int v1 = 0; v1 < 2; ++v1) {
        const int q = q0 + rloc + 8 * v1;
        qm[v1] = (args.q_index && q < args.S) ? __ldg(&args.q_index[q]) : q;  // position seen by the mask
      }
      em.init(mode, qm, m0, m1, m2);
    }
    float o[D / 2];
#pragma unroll
    for (int i = 0; i < D / 2; ++i) o[i] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};

    for (int j = 0; j < nch; ++j, ++g) {
      const int stage = g & 1;
      if (j + 1 < nch) load_chunk(j + 1, stage ^ 1);
      if constexpr (kGather) {
        if (j + 1 < nch) cp_async_wait<1>();
        else cp_async_wait<0>();
        fence_proxy_async_smem();
        __syncthreads();
      } else {
        if (j == 0) mbar_wait(smem_u32(&ctl->q_full), nq & 1, 1);
        mbar_wait(smem_u32(&ctl->kv_full[stage]), (g >> 1) & 1, 2);
      }
      const uint32_t sK = sK0 + 2 * stage * Cfg::kTileBytes, sV = sK + Cfg::kTileBytes;
      if constexpr (FP8) {
        // widen V (e4m3, one 128-byte panel) to fp16 (two panels) in the same swizzled image
#pragma unroll
        for (int i = tid; i < 128 * 8; i += 256) {
          const int r = i >> 3, pc = i & 7;
          const uint4 w = *reinterpret_cast<const uint4*>(smem_al + (sV - base) + r * 128 + ((pc ^ (r & 7)) << 4));
          const uint32_t in[4] = {w.x, w.y, w.z, w.w};
          uint32_t out[8];
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const __half2_raw lo = __nv_cvt_fp8x2_to_halfraw2(static_cast<__nv_fp8x2_storage_t>(in[k] & 0xffffu), __NV_E4M3);
            const __half2_raw hi = __nv_cvt_fp8x2_to_halfraw2(static_cast<__nv_fp8x2_storage_t>(in[k] >> 16), __NV_E4M3);
            out[2 * k] = static_cast<uint32_t>(lo.x) | (static_cast<uint32_t>(lo.y) << 16);
            out[2 * k + 1] = static_cast<uint32_t>(hi.x) | (static_cast<uint32_t>(hi.y) << 16);
          }
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            const int p16 = 2 * pc + hh;  // 16-byte piece of the fp16 row
            *reinterpret_cast<uint4*>(smem_al + (sVh - base) + (p16 >> 3) * Cfg::kPanelBytes + r * 128 +
                                      (((p16 & 7) ^ (r & 7)) << 4)) =
                make_uint4(out[4 * hh], out[4 * hh + 1], out[4 * hh + 2], out[4 * hh + 3]);
          }
        }
        fence_proxy_async_smem();
        __syncthreads();
      }

      float s[64];
      attn_qk<D, DT>(s, sQ + 64 * wg * 128, sK);

      // ---- mask: partial chunks and element-mask chunks
      int kv0 = 0, valid = kChunkCols;
      bool elem = false;
      if constexpr (kGather) {
        valid = min(kChunkCols, total_kv - j * kChunkCols);
      } else {
        const int2 ch = __ldg(&chunks[j]);
        kv0 = ch.x;
        valid = chunk_valid(ch.y);
        elem = (ch.y & kChunkElem) != 0;
      }
      if (valid < kChunkCols || elem) {
        // keep[v1] bit 2*jj + v0: column 8*jj + 2*(lane%4) + v0 of row v1 is an allowed key
        uint32_t keep[2] = {~0u, ~0u};
        if (elem) em.bits(kv0 + 2 * (lane & 3), keep);
#pragma unroll
        for (int jj = 0; jj < 16; ++jj)
#pragma unroll
          for (int v1 = 0; v1 < 2; ++v1)
#pragma unroll
            for (int v0 = 0; v0 < 2; ++v0) {
              const int col = 8 * jj + 2 * (lane & 3) + v0;
              const bool ok = col < valid && ((keep[v1] >> (2 * jj + v0)) & 1u);
              if (!ok) s[4 * jj + 2 * v1 + v0] = -INFINITY;
            }
      }

      // ---- online softmax (scores in log2 units: x * c)
#pragma unroll
      for (int v1 = 0; v1 < 2; ++v1) {
        float mx = -INFINITY;
#pragma unroll
        for (int jj = 0; jj < 16; ++jj) mx = fmaxf(mx, fmaxf(s[4 * jj + 2 * v1], s[4 * jj + 2 * v1 + 1]));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
        const float m_new = fmaxf(m_run[v1], mx);
        const float mc = m_new == -INFINITY ? 0.f : m_new * c;
        const float alpha = ex2_approx(m_run[v1] == -INFINITY ? -INFINITY : m_run[v1] * c - mc);
        m_run[v1] = m_new;
        float ls = 0.f;
#pragma unroll
        for (int jj = 0; jj < 16; ++jj)
#pragma unroll
          for (int v0 = 0; v0 < 2; ++v0) {
            const float p = ex2_approx(fmaf(s[4 * jj + 2 * v1 + v0], c, -mc));
            s[4 * jj + 2 * v1 + v0] = p;
            ls += p;
          }
        l_run[v1] = l_run[v1] * alpha + ls;
#pragma unroll
        for (int jj = 0; jj < D / 8; ++jj) {
          o[4 * jj + 2 * v1] *= alpha;
          o[4 * jj + 2 * v1 + 1] *= alpha;
        }
      }
      attn_pv<D, kPBF16>(o, s, FP8 ? sVh : sV);
      __syncthreads();  // stage `stage` (and the fp16 V copy) may be overwritten from here on
    }
    if (nch > 0) ++nq;

    // ---------------- epilogue: O / l -> global (optionally scattered rows), LSE
#pragma unroll
    for (int v1 = 0; v1 < 2; ++v1) {
      float l = l_run[v1];
      l += __shfl_xor_sync(0xffffffffu, l, 1);
      l += __shfl_xor_sync(0xffffffffu, l, 2);
      const int row = rloc + 8 * v1;
      if (row >= nr) continue;
      const int q = q0 + row;
      const float inv_l = (l > 0.f ? 1.f / l : 0.f) * vs;
      long long out_row = q;
      if (args.o_rows) out_row = __ldg(&args.o_rows[static_cast<size_t>(bh) * args.S + q]);
      const int col0 = 2 * (lane & 3);
      if (args.out_f32) {
        float* optr = reinterpret_cast<float*>(args.o) + bh * args.o_head_stride + out_row * args.o_row_stride;
#pragma unroll
        for (int jj = 0; jj < D / 8; ++jj)
          *reinterpret_cast<float2*>(optr + 8 * jj + col0) =
              make_float2(o[4 * jj + 2 * v1] * inv_l, o[4 * jj + 2 * v1 + 1] * inv_l);
      } else {
        uint16_t* optr = reinterpret_cast<uint16_t*>(args.o) + bh * args.o_head_stride + out_row * args.o_row_stride;
#pragma unroll
        for (int jj = 0; jj < D / 8; ++jj)
          *reinterpret_cast<uint32_t*>(optr + 8 * jj + col0) =
              pack2<BF16>(o[4 * jj + 2 * v1] * inv_l, o[4 * jj + 2 * v1 + 1] * inv_l);
      }
      if (args.lse && (lane & 3) == 0) {
        // natural-log LSE of the scaled scores; -inf for rows that saw no key
        const float lse = l > 0.f ? (m_run[v1] * c + log2f(l)) * 0.6931471805599453f : -INFINITY;
        args.lse[static_cast<size_t>(bh) * args.S + out_row] = lse;
      }
    }
  }
}

}  // namespace svgb
