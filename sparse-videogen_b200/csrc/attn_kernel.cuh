// Block-sparse flash attention forward for sm_90a (Hopper wgmma).
//
// One CTA per work item, 384 threads in three warpgroups.  Warpgroup 0 is the PRODUCER: it does every load.
// Warpgroups 1 and 2 are the CONSUMERS: consumer c owns query rows 64c .. 64c+63 of a 128-row tile.  A work item is
// one or two 128-row STREAMS, each a descriptor {q_row0, nrows, list_off, list_len} (attn_common.cuh), run one after
// the other.
//   Q tile          : TMA (or cp.async row gather), 128-byte swizzle, stays in shared memory for the stream
//   K(j), V(j)      : three stages, each half with its own full and empty mbarrier
//   S = Q K^T       : wgmma m64n128 (SS, both operands K-major), fp32 accumulators in registers
//   softmax         : online, in registers (each row is spread over the 4 lanes of a quad)
//   O += P V        : wgmma m64nD (RS: P from registers in the accumulator layout of S, V MN-major)
// The producer and the consumers meet only at mbarriers (the protocol table is in DESIGN.md §1); after the role
// split there is no block-wide barrier.  The chunk loop is software-pipelined inside each consumer: iteration j
// issues S = Q K(j+1)^T and then O += P(j) V(j) as two wgmma groups, waits for the first only, and runs the mask
// and softmax of chunk j+1 while P V(j) is still on the tensor cores.  The two consumers take turns issuing their
// groups (two named barriers), so one consumer's softmax also runs under the other's MMAs.  Every row still sees
// the same operations in the same order as a one-chunk-at-a-time loop (rescale O by alpha(j+1), then accumulate
// P(j+1) V(j+1)).
// FP8 (e4m3) inputs: Q K^T runs on e4m3 wgmma (k32); wgmma has no MN-major 8-bit B operand, so the producer widens
// each V tile to fp16 in shared memory (two buffers, with their own full and empty barriers) and P V runs in fp16.
// Both loaders serve e4m3: the row gather copies 128-byte e4m3 rows into the same swizzled image TMA writes, and
// the widening step that follows is shared.
// Per-row FP8 (DT_E4M3_ROWS, KV-cache plans only): every q, k and v row has its own power-of-two scale (fp8_rows.cuh).
// The K and V scales of a chunk (128 floats each) land with its K and V tiles, in the same TMA transactions; the
// consumers multiply each S column by its K scale before the row max, each row's c carries its q scale, and the
// producer's widening multiplies every V row by its scale and writes bf16, so P V runs in bf16 (DESIGN.md).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>

#include <type_traits>

#include "attn_common.cuh"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace svgb {

// element type of Q/K/V: 0 = bf16, 1 = fp16, 2 = fp8 e4m3 with per-head scales, 3 = fp8 e4m3 with per-row scales
// (both output bf16)
constexpr int DT_BF16 = 0, DT_F16 = 1, DT_E4M3 = 2, DT_E4M3_ROWS = 3;
// K/V stages: with P V(j) still running when Q K(j+1)^T is issued, V(j) frees late in iteration j, so the load of
// chunk j+3 into its stage gets about two chunks of lead time
constexpr int kKvStages = 3;

template <int D, int DT = DT_BF16>
struct AttnCfg {
  static_assert(D == 64 || D == 128, "head_dim must be 64 or 128");
  static_assert(DT < DT_E4M3 || D == 128, "the e4m3 path is built for head_dim 128 (128-byte rows)");
  static constexpr int kElemBytes = DT >= DT_E4M3 ? 1 : 2;
  static constexpr int kRowBytes = D * kElemBytes;
  static constexpr int kHalves = kRowBytes / 128;        // 128-byte swizzle panels per row
  static constexpr int kPanelElems = 128 / kElemBytes;   // elements per panel row (TMA box width)
  static constexpr int kPanelBytes = 128 * 128;          // 128 rows x 128 B
  static constexpr int kTileBytes = kPanelBytes * kHalves;
  static constexpr int kKSteps = kRowBytes / 32;         // wgmma K steps of Q K^T (32 bytes each)
  static constexpr int kVhBytes = DT >= DT_E4M3 ? 2 * kPanelBytes : 0;  // 16-bit copy of one e4m3 V tile
  // per-row FP8 (KV-cache plans, TMA loader only).  The kernel reads these here rather than from locals of its own:
  // extra local constants in attn_fwd_kernel change the register allocation of the per-head e4m3 instantiation.
  static constexpr bool kRows = DT == DT_E4M3_ROWS;
  static constexpr int kScaleRowBytes = 128 * 4;                             // one chunk's K (or V) row scales
  static constexpr int kScaleBytes = kRows ? kKvStages * 2 * kScaleRowBytes : 0;  // per stage: K, V row scales
  static constexpr int kBarBytes = 1024;                 // mbarriers + gather row table
  // + 1 KB: the kernel aligns the dynamic window to 1024 bytes itself
  static constexpr int kSmemBytes =
      1024 + kTileBytes + 2 * kKvStages * kTileBytes + 2 * kVhBytes + kScaleBytes + kBarBytes;
  static constexpr int kThreads = 384;  // producer warpgroup + two consumer warpgroups
  static_assert(kSmemBytes <= 227 * 1024, "exceeds the 227 KB per-CTA shared memory of sm_90");
};

// The wgmma products are issued and committed as one group each; their accumulators (and the P fragments of
// P V) may not be touched until attn_wait has retired the group.

// S[64 x 128] = Q[64 rows of the tile] K^T for one warpgroup
template <int D, int DT>
__device__ __forceinline__ void attn_qk_issue(float (&s)[64], uint32_t sQw, uint32_t sK) {
  using Cfg = AttnCfg<D, DT>;
#pragma unroll
  for (int i = 0; i < 64; ++i) s[i] = 0.f;
  wg_fence();
#pragma unroll
  for (int kk = 0; kk < Cfg::kKSteps; ++kk) {
    const uint32_t off = (kk >> 2) * Cfg::kPanelBytes + (kk & 3) * 32;
    const uint64_t a = wg_desc_kmajor(sQw + off), b = wg_desc_kmajor(sK + off);
    if constexpr (DT >= DT_E4M3) wgmma_m64n128k32_e4m3_ss(s, a, b, kk > 0);
    else wgmma_m64n128k16_ss<DT == DT_BF16>(s, a, b, kk > 0);
  }
  wg_commit();
}

// P[64 x 128] in the accumulator layout of S -> the A fragments of P V, packed to 16 bit (kBF16: bf16, else fp16)
template <bool kBF16>
__device__ __forceinline__ void attn_pack_p(uint32_t (&a)[8][4], const float (&p)[64]) {
#pragma unroll
  for (int kk = 0; kk < 8; ++kk)
#pragma unroll
    for (int r = 0; r < 4; ++r) a[kk][r] = pack2<kBF16>(p[8 * kk + 2 * r], p[8 * kk + 2 * r + 1]);
}

// O[64 x D] += P[64 x 128] V[128 x D]
template <int D, bool kBF16>
__device__ __forceinline__ void attn_pv_issue(float (&o)[D / 2], const uint32_t (&a)[8][4], uint32_t sV) {
  wg_fence();
#pragma unroll
  for (int kk = 0; kk < 8; ++kk) {
    const uint64_t b = wg_desc_mnmajor(sV + kk * 2048, 128 * 128);
    if constexpr (D == 128) wgmma_m64n128k16_rs<kBF16>(o, a[kk], b, 1);
    else wgmma_m64n64k16_rs<kBF16>(o, a[kk], b, 1);
  }
  wg_commit();
}

// wait until at most N of this warpgroup's wgmma groups are pending (groups retire in issue order), then let the
// accumulators `d` of a retired group be read
template <int N, int M>
__device__ __forceinline__ void attn_wait(float (&d)[M]) {
  wg_wait<N>();
  wg_fence_regs(d);
}

// Per-row FP8: 16 e4m3 values of one V row -> bf16(v8 * sv), sv = 2^e its scale.  e4m3 -> fp16 -> fp32 are exact, the
// product is an exponent shift, and the bf16 rounding is exact wherever the result lies in bf16's range (DESIGN.md).
__device__ __forceinline__ void widen_rows(const uint32_t (&in)[4], uint32_t (&out)[8], float sv) {
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const __half2_raw h2 =
        __nv_cvt_fp8x2_to_halfraw2(static_cast<__nv_fp8x2_storage_t>((in[k >> 1] >> (16 * (k & 1))) & 0xffffu), __NV_E4M3);
    const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&h2));
    const __nv_bfloat162 b2 = __floats2bfloat162_rn(f.x * sv, f.y * sv);
    out[k] = *reinterpret_cast<const uint32_t*>(&b2);
  }
}

// mbarriers of the producer / consumer protocol.  A full barrier completes once its data has landed: one arrival
// with the transaction bytes from the TMA-issuing thread, or (row gather) one cp.async arrival from each of the
// producer's 128 threads.  An empty barrier completes once both consumers are done with the buffer: one arrival
// from thread 0 of each consumer warpgroup.  vh_full: one arrival from each producer thread after widening.
struct AttnSmemCtl {
  uint64_t q_full, q_empty;
  uint64_t k_full[kKvStages], k_empty[kKvStages];
  uint64_t v_full[kKvStages], v_empty[kKvStages];
  uint64_t vh_full[2], vh_empty[2];  // FP8: the two fp16 copies of V
  int src[128];  // gather: source row of each of the 128 rows being loaded (-1: zero fill)
  float pin[8];  // one word per consumer warp, written and never read (see the chunk loop)
};

// named barriers (0 is __syncthreads): the producer's own 128 threads, and the two consumers' turns
constexpr int kBarProducer = 1, kBarTurn = 2;  // consumer c waits for its turn on kBarTurn + c
// register split of the 64 K registers: 128 x 24 (producer) + 256 x 240 (consumers) = 64,512
constexpr int kProducerRegs = 24, kConsumerRegs = 240;

// kGather selects the loader: false = TMA boxes over contiguous key ranges (chunk list), true = cp.async
// row gathers over a run list.  ksmap, vsmap: DT_E4M3_ROWS only, the K and V row scales [num_blocks, Hkv, block_rows]
// as (row, head, block), box 128 x 1 x 1 fp32.
template <int D, int DT, bool kGather>
__global__ void __launch_bounds__(384, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap qmap, const __grid_constant__ CUtensorMap kmap,
                const __grid_constant__ CUtensorMap vmap, const AttnArgs args,
                const __grid_constant__ CUtensorMap ksmap, const __grid_constant__ CUtensorMap vsmap) {
  using Cfg = AttnCfg<D, DT>;
  constexpr bool BF16 = DT != DT_F16;  // output format (fp8 inputs produce bf16 output)
  constexpr bool FP8 = DT >= DT_E4M3;
  // format of P and V in the P V product (fp8: fp16 with per-head scales, bf16 with per-row scales)
  constexpr bool kPBF16 = DT == DT_BF16 || Cfg::kRows;
  using Elem = typename std::conditional<FP8, uint8_t, uint16_t>::type;  // storage element of Q / K / V
  const int bh = blockIdx.y;  // query head: Q, O, LSE
  // key/value head: K, V and the plan's work list.  Gather plans take no groups (their kv_rows are per query head; the
  // host refuses them with kv_group > 1), so the row-gather kernel keeps bh and its code of kv_group = 1.
  const int kvh = kGather ? bh : bh / args.kv_group;
  const int n_items = args.item_count[args.items_stride ? kvh : 0];
  if (static_cast<int>(blockIdx.x) >= n_items) return;
  const int4* desc = args.items + 2 * (static_cast<size_t>(kvh) * args.items_stride + blockIdx.x);

  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_u32 = smem_u32(smem_raw);
  const uint32_t base = (raw_u32 + 1023u) & ~1023u;
  uint8_t* smem_al = smem_raw + (base - raw_u32);
  const uint32_t sQ = base;
  const uint32_t sK0 = sQ + Cfg::kTileBytes;  // stage s: K at sK0 + 2s*tile, V at sK0 + (2s+1)*tile
  const uint32_t sVh = sK0 + 2 * kKvStages * Cfg::kTileBytes;  // FP8: buffer b at sVh + b*kVhBytes
  // ROWS: stage s's K row scales at sSc + 2s * 512, its V row scales 512 bytes after them
  const uint32_t sSc = sVh + 2 * Cfg::kVhBytes;
  AttnSmemCtl* ctl = reinterpret_cast<AttnSmemCtl*>(smem_al + Cfg::kTileBytes * (1 + 2 * kKvStages) +
                                                    2 * Cfg::kVhBytes + Cfg::kScaleBytes);

  const int tid = threadIdx.x;
  // the warpgroup index through a shuffle, so that ptxas sees it is warp-uniform and splits the register allocation
  // at the setmaxnreg of each role
  const int wg = __shfl_sync(0xffffffffu, tid >> 7, 0);
  const int wt = tid & 127, lane = tid & 31, wq = wt >> 5;
  if (tid == 0) {
    const uint32_t full_count = kGather ? 128 : 1;
    mbar_init(smem_u32(&ctl->q_full), full_count);
    mbar_init(smem_u32(&ctl->q_empty), 2);
    for (int i = 0; i < kKvStages; ++i) {
      mbar_init(smem_u32(&ctl->k_full[i]), full_count);
      // ROWS: the consumers also read the stage's K scales, so each of their 8 warps releases it
      mbar_init(smem_u32(&ctl->k_empty[i]), Cfg::kRows ? 8 : 2);
      mbar_init(smem_u32(&ctl->v_full[i]), full_count);
      mbar_init(smem_u32(&ctl->v_empty[i]), 2);
    }
    for (int b = 0; b < 2; ++b) {
      mbar_init(smem_u32(&ctl->vh_full[b]), 128);
      mbar_init(smem_u32(&ctl->vh_empty[b]), 2);
    }
    mbar_fence_init();
    if constexpr (!kGather) {
      tma_prefetch_desc(&qmap);
      tma_prefetch_desc(&kmap);
      tma_prefetch_desc(&vmap);
    }
    if constexpr (Cfg::kRows) {
      tma_prefetch_desc(&ksmap);
      tma_prefetch_desc(&vsmap);
    }
  }
  __syncthreads();  // the barriers are initialised; the last block-wide barrier of the kernel

  const int nstreams = __ldg(&desc[1].y) > 0 ? 2 : 1;
  // stream st of the item: first query row, rows, list, list length, chunk count and (gather) selected keys.  A
  // gather stream's chunks are implicit: 128 selected keys each, the last one partial.
  struct Stream {
    int q0, nr, nlist, nch, total;
    const int2* list;
  };
  auto stream = [&](int st) {
    const int4 d = __ldg(&desc[st]);
    Stream sm;
    sm.q0 = d.x;
    sm.nr = d.y;
    sm.list = args.chunks + d.z;
    sm.nlist = d.w;
    sm.total = kGather ? __ldg(&sm.list[d.w].y) : 0;  // the run list's sentinel
    sm.nch = kGather ? (sm.total + kChunkCols - 1) / kChunkCols : d.w;
    return sm;
  };
  // Both roles count chunks over the whole CTA: chunk n (the stream's chunk j is n = g + j, g = chunks of the earlier
  // streams) lives in K/V stage n % 3, phase (n / 3) & 1 of that stage's barriers; FP8: its fp16 V copy in buffer
  // n & 1, phase (n / 2) & 1.  An empty barrier's wait for round r is on parity (r & 1) ^ 1: round 0 passes at once.
  auto stage_k = [&](int n) { return sK0 + 2 * (n % kKvStages) * Cfg::kTileBytes; };
  auto stage_ks = [&](int n) { return sSc + 2 * (n % kKvStages) * Cfg::kScaleRowBytes; };  // ROWS: K scales; V: + 512
  auto vh_buf = [&](int n) { return sVh + (n & 1) * Cfg::kVhBytes; };

  if (wg == 0) {
    // ======================= producer: every load, and the FP8 widening of V
    setmaxnreg_dec<kProducerRegs>();
    const Elem* kp = static_cast<const Elem*>(args.k_ptr) + kvh * args.in_head_stride;
    const Elem* vp = static_cast<const Elem*>(args.v_ptr) + kvh * args.in_head_stride;
    const int* kv_rows = (kGather && args.kv_rows) ? args.kv_rows + static_cast<size_t>(bh) * args.S : nullptr;

    // gather: piece p (16 B) of row r -> panel p/8, byte r*128 + ((p%8) ^ (r%8))*16; a row is kRowBytes bytes
    // (e4m3 at D = 128: 8 pieces, one panel)
    auto gather_rows = [&](uint32_t dst, const Elem* src_base) {
      constexpr int kPieces = Cfg::kRowBytes / 16;
      constexpr int kPieceElems = 16 / Cfg::kElemBytes;
#pragma unroll 4
      for (int i = wt; i < 128 * kPieces; i += 128) {
        const int r = i / kPieces, pc = i % kPieces;
        const int src = ctl->src[r];
        const uint32_t off = (pc >> 3) * Cfg::kPanelBytes + r * 128 + (((pc & 7) ^ (r & 7)) << 4);
        const long long so = static_cast<long long>(src < 0 ? 0 : src) * args.in_row_stride + pc * kPieceElems;
        cp_async16(dst + off, src_base + so, src >= 0 ? 16u : 0u);
      }
    };
    // gather: source rows of keys j*128 .. j*128+127 of stream sm -> ctl->src
    auto resolve_chunk = [&](const Stream& sm, int j) {
      const int2* __restrict__ runs = sm.list;
      const int pos = j * kChunkCols + wt;
      int src = -1;
      if (pos < sm.total) {
        int lo = 0, hi = sm.nlist - 1;  // largest run with keys_before <= pos
        while (lo < hi) {
          const int mid = (lo + hi + 1) >> 1;
          if (__ldg(&runs[mid].y) <= pos) lo = mid;
          else hi = mid - 1;
        }
        const int2 rr = __ldg(&runs[lo]);
        const int prow = rr.x + (pos - rr.y);
        src = kv_rows ? __ldg(&kv_rows[prow]) : prow;
      }
      ctl->src[wt] = src;
    };
    // FP8: widen V (e4m3, one 128-byte panel) of chunk n to fp16 (two panels) in the same swizzled image.  The
    // copy is written through the generic proxy and read by wgmma (async proxy): each writer fences before its
    // arrival on vh_full, and the consumers' acquire of vh_full orders their wgmma after it.
    auto widen_v = [&](int n) {
      mbar_wait(smem_u32(&ctl->v_full[n % kKvStages]), (n / kKvStages) & 1, 9);
      mbar_wait(smem_u32(&ctl->vh_empty[n & 1]), ((n >> 1) & 1) ^ 1, 8);
      const uint32_t sV = stage_k(n) + Cfg::kTileBytes, dst = vh_buf(n);
#pragma unroll 1
      for (int i = wt; i < 128 * 8; i += 128) {
        const int r = i >> 3, pc = i & 7;
        const uint4 w = *reinterpret_cast<const uint4*>(smem_al + (sV - base) + r * 128 + ((pc ^ (r & 7)) << 4));
        const uint32_t in[4] = {w.x, w.y, w.z, w.w};
        uint32_t out[8];
        if constexpr (Cfg::kRows) widen_rows(in, out, *reinterpret_cast<const float*>(smem_al + (stage_ks(n) - base) +
                                                                                 Cfg::kScaleRowBytes + 4 * r));
        else {
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const __half2_raw lo = __nv_cvt_fp8x2_to_halfraw2(static_cast<__nv_fp8x2_storage_t>(in[k] & 0xffffu), __NV_E4M3);
          const __half2_raw hi = __nv_cvt_fp8x2_to_halfraw2(static_cast<__nv_fp8x2_storage_t>(in[k] >> 16), __NV_E4M3);
          out[2 * k] = static_cast<uint32_t>(lo.x) | (static_cast<uint32_t>(lo.y) << 16);
          out[2 * k + 1] = static_cast<uint32_t>(hi.x) | (static_cast<uint32_t>(hi.y) << 16);
        }
        }
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int p16 = 2 * pc + hh;  // 16-byte piece of the fp16 row
          *reinterpret_cast<uint4*>(smem_al + (dst - base) + (p16 >> 3) * Cfg::kPanelBytes + r * 128 +
                                    (((p16 & 7) ^ (r & 7)) << 4)) =
              make_uint4(out[4 * hh], out[4 * hh + 1], out[4 * hh + 2], out[4 * hh + 3]);
        }
      }
      fence_proxy_async_smem();
      mbar_arrive(smem_u32(&ctl->vh_full[n & 1]));
    };

    // TMA: thread 0 issues every box.  Gather: all 128 threads resolve and copy rows; each one's cp.async arrival
    // (.noinc: counted by the barrier's 128) fires once its own copies have landed.  Those copies are generic-proxy
    // writes that wgmma reads through the async proxy; the writer cannot fence after an asynchronous copy, so each
    // consumer thread fences (fence.proxy.async) after its full-barrier wait, before its warpgroup's wgmma.
    const bool leader = wt == 0;
    // the tensor maps' (head, batch) coordinates: query head hq and key/value head hkv of batch element `batch`
    const int batch = bh / args.Hq, hq = bh - batch * args.Hq, hkv = hq / args.kv_group;
    int g = 0, nq = 0;  // chunks and Q tiles of the earlier streams
    for (int st = 0; st < nstreams; ++st) {
      const Stream sm = stream(st);
      if (sm.nch == 0) continue;
      // Q (rows past nr: zero filled by the gather, other rows' data by TMA -- never stored); the previous stream's
      // Q is free once both consumers have retired its last Q K^T
      if constexpr (kGather) {
        const int* q_rows = args.q_rows ? args.q_rows + static_cast<size_t>(bh) * args.S : nullptr;
        ctl->src[wt] = wt < sm.nr ? (q_rows ? __ldg(&q_rows[sm.q0 + wt]) : sm.q0 + wt) : -1;
        mbar_wait(smem_u32(&ctl->q_empty), (nq & 1) ^ 1, 5);
        named_bar_sync(kBarProducer, 128);
        gather_rows(sQ, static_cast<const Elem*>(args.q_ptr) + bh * args.in_head_stride);
        cp_async_arrive_noinc(smem_u32(&ctl->q_full));
        named_bar_sync(kBarProducer, 128);  // ctl->src is reused by the next resolve
      } else if (leader) {
        const uint32_t qb = smem_u32(&ctl->q_full);
        mbar_wait(smem_u32(&ctl->q_empty), (nq & 1) ^ 1, 5);
        mbar_expect_tx(qb, Cfg::kTileBytes);
        for (int x = 0; x < Cfg::kHalves; ++x) tma_load_4d(sQ + x * Cfg::kPanelBytes, &qmap, qb, x * Cfg::kPanelElems, sm.q0, hq, batch);
      }
      for (int j = 0; j < sm.nch; ++j) {
        const int n = g + j, s = n % kKvStages, par = ((n / kKvStages) & 1) ^ 1;
        const uint32_t sK = stage_k(n), sV = sK + Cfg::kTileBytes;
        const uint32_t kf = smem_u32(&ctl->k_full[s]), vf = smem_u32(&ctl->v_full[s]);
        if constexpr (kGather) {
          resolve_chunk(sm, j);
          mbar_wait(smem_u32(&ctl->k_empty[s]), par, 6);
          named_bar_sync(kBarProducer, 128);
          gather_rows(sK, kp);
          cp_async_arrive_noinc(kf);
          mbar_wait(smem_u32(&ctl->v_empty[s]), par, 7);
          gather_rows(sV, vp);
          cp_async_arrive_noinc(vf);
          named_bar_sync(kBarProducer, 128);  // ctl->src is reused by the next resolve
        } else if (leader) {
          const int kv0 = __ldg(&sm.list[j].x);
          // ROWS: the chunk's scales at (row, head, block) of its physical row kv0; rows past the block's end are
          // outside the scale map and TMA fills them with zeros
          int srow = 0, sblk = 0;
          if constexpr (Cfg::kRows) {
            sblk = kv0 / args.scale_block_rows;
            srow = kv0 - sblk * args.scale_block_rows;
          }
          mbar_wait(smem_u32(&ctl->k_empty[s]), par, 6);
          mbar_expect_tx(kf, Cfg::kTileBytes + (Cfg::kRows ? Cfg::kScaleRowBytes : 0));
          for (int x = 0; x < Cfg::kHalves; ++x) tma_load_4d(sK + x * Cfg::kPanelBytes, &kmap, kf, x * Cfg::kPanelElems, kv0, hkv, batch);
          if constexpr (Cfg::kRows) tma_load_3d(stage_ks(n), &ksmap, kf, srow, hkv, sblk);
          mbar_wait(smem_u32(&ctl->v_empty[s]), par, 7);
          mbar_expect_tx(vf, Cfg::kTileBytes + (Cfg::kRows ? Cfg::kScaleRowBytes : 0));
          for (int x = 0; x < Cfg::kHalves; ++x) tma_load_4d(sV + x * Cfg::kPanelBytes, &vmap, vf, x * Cfg::kPanelElems, kv0, hkv, batch);
          if constexpr (Cfg::kRows) tma_load_3d(stage_ks(n) + Cfg::kScaleRowBytes, &vsmap, vf, srow, hkv, sblk);
        }
        // FP8: widen the previous chunk's V, requested one chunk earlier, rather than wait here for V(j) to land
        if constexpr (FP8) {
          if (j > 0) widen_v(n - 1);
        }
      }
      if constexpr (FP8) widen_v(g + sm.nch - 1);
      g += sm.nch;
      ++nq;
    }
    return;
  }

  // ======================= consumers
  setmaxnreg_inc<kConsumerRegs>();
  const int cw = wg - 1;                    // this consumer's 64 rows of the tile: 64cw .. 64cw+63
  const uint32_t sQw = sQ + 64 * cw * 128;
  // FP8: q_scale per query head, k_scale and v_scale per key/value head (a group's query heads share its K and V).
  // 16-bit inputs take no scales; their instantiations keep indexing by bh, so their code does not depend on kvh.
  // ROWS: the row scales take their place (c_row below, the K scales on S, the V scales in the widening).
  const int sh = FP8 ? kvh : bh;
  const float c = args.scale_log2 * ((!Cfg::kRows && args.q_scale) ? __ldg(&args.q_scale[bh]) * __ldg(&args.k_scale[sh]) : 1.f);
  const float vs = (!Cfg::kRows && args.v_scale) ? __ldg(&args.v_scale[sh]) : 1.f;
  const int mode = args.mask_mode, m0 = args.m0, m1 = args.m1, m2 = args.m2;

  // Turns on the tensor cores: each consumer issues its wgmma groups between turn_wait and turn_pass, so the two
  // consumers' groups alternate and one's softmax runs under the other's MMAs.  Consumer 0 takes the first turn.
  auto turn_wait = [&]() { named_bar_sync(kBarTurn + cw, 256); };
  auto turn_pass = [&]() { named_bar_arrive(kBarTurn + (cw ^ 1), 256); };
  // thread 0 of the warpgroup arrives for it, after the warpgroup's wgmma reading the buffer has retired
  auto release = [&](uint64_t& bar) {
    if (wt == 0) mbar_arrive(smem_u32(&bar));
  };
  // a K stage is free once the warpgroup's Q K^T has retired and (ROWS) each warp has read the stage's K scales
  auto release_k = [&](int n) {
    if constexpr (Cfg::kRows) {
      __syncwarp();
      if (lane == 0) mbar_arrive(smem_u32(&ctl->k_empty[n % kKvStages]));
    } else {
      release(ctl->k_empty[n % kKvStages]);
    }
  };
  if (cw == 1) turn_pass();

  int g = 0;   // chunks of this CTA before the current stream (the stream's chunk j is the CTA's chunk g + j)
  int nq = 0;  // Q tiles loaded so far (q_full phase)
  for (int st = 0; st < nstreams; ++st) {
    const Stream sm = stream(st);
    const int q0 = sm.q0, nr = sm.nr, nch = sm.nch, total = sm.total;
    const int2* __restrict__ chunks = sm.list;

    auto wait_k = [&](int n) { mbar_wait(smem_u32(&ctl->k_full[n % kKvStages]), (n / kKvStages) & 1, 2); };
    auto wait_v = [&](int n) {
      if constexpr (FP8) mbar_wait(smem_u32(&ctl->vh_full[n & 1]), (n >> 1) & 1, 4);
      else mbar_wait(smem_u32(&ctl->v_full[n % kKvStages]), (n / kKvStages) & 1, 3);
    };
    // FP8: the e4m3 V stage was read by the producer's widening, which the wait on vh_full ordered before P V
    auto release_v = [&](int n) {
      release(ctl->v_empty[n % kKvStages]);
      if constexpr (FP8) release(ctl->vh_empty[n & 1]);
    };
    auto pv_b = [&](int n) { return FP8 ? vh_buf(n) : stage_k(n) + Cfg::kTileBytes; };

    // per thread: rows r0 = 16*wq + lane/4 and r0 + 8 of this warpgroup's 64; columns 8j + 2*(lane%4) (+1)
    const int rloc = 64 * cw + 16 * wq + (lane >> 2);
    ElemMask em;
    if constexpr (!kGather) {  // gather plans carry no element masks
      // segment plans: the stream's segment shifts the query positions, moves the sink bound and anchors the block grid
      // (seg_origin); KV-cache plans: the stream's length shifts them to logical positions (kv_origin)
      SegOrigin so{0, m0};
      if (args.segs) so = args.kv_logical ? kv_stream_origin(args.segs, q0, m0) : seg_origin(args.segs, q0, false, m0);
      int qm[2];
#pragma unroll
      for (int v1 = 0; v1 < 2; ++v1) {
        const int q = q0 + rloc + 8 * v1;
        qm[v1] = ((args.q_index && q < args.S) ? __ldg(&args.q_index[q]) : q) - so.shift;  // position seen by the mask
      }
      em.init(mode, qm, so.sink_end, m1, m2, so.key0);
    }
    // ROWS: c of each of the thread's two rows carries the row's q scale, q_scale [Hq, S] (rows past nr: never stored)
    float c_row[2] = {0.f, 0.f};
    if constexpr (Cfg::kRows) {
#pragma unroll
      for (int v1 = 0; v1 < 2; ++v1) {
        const int row = rloc + 8 * v1;
        c_row[v1] = c * (row < nr ? __ldg(&args.q_scale[static_cast<size_t>(bh) * args.S + q0 + row]) : 1.f);
      }
    }
    auto crow = [&](int v1) {
      if constexpr (Cfg::kRows) return c_row[v1];
      else return c;
    };
    float o[D / 2];
#pragma unroll
    for (int i = 0; i < D / 2; ++i) o[i] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f}, alpha[2];
    float s[64];        // S of the chunk being scored, then its P
    uint32_t pa[8][4];  // P of the chunk whose P V is next, packed to 16 bit

    // ROWS: S column 8 jj + 2 (lane % 4) + v0 times the K scale of its key row (chunk n's stage)
    auto scale_k = [&](int n) {
      if constexpr (Cfg::kRows) {
        const float* ks = reinterpret_cast<const float*>(smem_al + (stage_ks(n) - base)) + 2 * (lane & 3);
#pragma unroll
        for (int jj = 0; jj < 16; ++jj) {
          const float2 k2 = *reinterpret_cast<const float2*>(ks + 8 * jj);
#pragma unroll
          for (int v1 = 0; v1 < 2; ++v1) {
            s[4 * jj + 2 * v1] *= k2.x;
            s[4 * jj + 2 * v1 + 1] *= k2.y;
          }
        }
      }
    };
    // mask and online softmax of chunk j (scores in log2 units: x * c): S -> P, running max and sum, alpha = the
    // factor O still has to be scaled by before P(j) V(j) is accumulated
    auto softmax = [&](int j) {
      // ---- mask: partial chunks and element-mask chunks
      int kv0 = 0, meta = 0, valid = kChunkCols;
      bool elem = false;
      if constexpr (kGather) {
        valid = min(kChunkCols, total - j * kChunkCols);
      } else {
        const int2 ch = __ldg(&chunks[j]);
        kv0 = ch.x;
        meta = ch.y;
        valid = chunk_valid(ch.y);
        elem = (ch.y & kChunkElem) != 0;
      }
      if (valid < kChunkCols || elem) {
        // keep[v1] bit 2*jj + v0: column 8*jj + 2*(lane%4) + v0 of row v1 is an allowed key
        uint32_t keep[2] = {~0u, ~0u};
        // KV-cache plans: the mask sees the chunk's logical position, the TMA box loaded its physical row kv0
        if (elem) em.bits((args.kv_logical ? chunk_logical_kv0(meta) : kv0) + 2 * (lane & 3), keep);
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
#pragma unroll
      for (int v1 = 0; v1 < 2; ++v1) {
        float mx = -INFINITY;
#pragma unroll
        for (int jj = 0; jj < 16; ++jj) mx = fmaxf(mx, fmaxf(s[4 * jj + 2 * v1], s[4 * jj + 2 * v1 + 1]));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
        const float m_new = fmaxf(m_run[v1], mx);
        const float mc = m_new == -INFINITY ? 0.f : m_new * crow(v1);
        alpha[v1] = ex2_approx(m_run[v1] == -INFINITY ? -INFINITY : m_run[v1] * crow(v1) - mc);
        m_run[v1] = m_new;
        float ls = 0.f;
#pragma unroll
        for (int jj = 0; jj < 16; ++jj)
#pragma unroll
          for (int v0 = 0; v0 < 2; ++v0) {
            const float p = ex2_approx(fmaf(s[4 * jj + 2 * v1 + v0], crow(v1), -mc));
            s[4 * jj + 2 * v1 + v0] = p;
            ls += p;
          }
        l_run[v1] = l_run[v1] * alpha[v1] + ls;
      }
    };
    // O *= alpha and P -> fragments: only once P V of the previous chunk has retired
    auto rescale_pack = [&]() {
#pragma unroll
      for (int v1 = 0; v1 < 2; ++v1)
#pragma unroll
        for (int jj = 0; jj < D / 8; ++jj) {
          o[4 * jj + 2 * v1] *= alpha[v1];
          o[4 * jj + 2 * v1 + 1] *= alpha[v1];
        }
      attn_pack_p<kPBF16>(pa, s);
    };

    if (nch > 0) {
      mbar_wait(smem_u32(&ctl->q_full), nq & 1, 1);
      wait_k(g);
      if constexpr (kGather) fence_proxy_async_smem();  // cp.async rows -> wgmma (see the producer)
      turn_wait();
      attn_qk_issue<D, DT>(s, sQw, stage_k(g));
      turn_pass();
      attn_wait<0>(s);
      scale_k(g);
      release_k(g);
      if (nch == 1) release(ctl->q_empty);
      softmax(0);
      rescale_pack();

      for (int j = 0; j + 1 < nch; ++j) {
        const int n = g + j;
        wait_k(n + 1);
        wait_v(n);
        if constexpr (kGather) fence_proxy_async_smem();
        turn_wait();
        attn_qk_issue<D, DT>(s, sQw, stage_k(n + 1));  // group A
        attn_pv_issue<D, kPBF16>(o, pa, pv_b(n));      // group B: O and pa stay in flight
        turn_pass();
        attn_wait<1>(s);                               // A has retired, B may still be running
        scale_k(n + 1);
        release_k(n + 1);
        if (j + 2 == nch) release(ctl->q_empty);       // the stream's last Q K^T has retired
        softmax(j + 1);                                // runs under P V(j)
        // ptxas schedules wgmma.wait_group ahead of register math that does not depend on it, which would move
        // the exps below the wait and out from under P V(j).  Shared-memory stores stay ahead of the wait, so
        // storing the running sums (they depend on every exp of the chunk) keeps the softmax in front of it.
        if (lane == 0) ctl->pin[4 * cw + wq] = l_run[0] + l_run[1];
        attn_wait<0>(o);
        wg_fence_regs(s);  // P(j+1) is packed into pa only after P V(j) has read it
        release_v(n);
        rescale_pack();
      }
      wait_v(g + nch - 1);
      if constexpr (kGather) fence_proxy_async_smem();
      turn_wait();
      attn_pv_issue<D, kPBF16>(o, pa, pv_b(g + nch - 1));
      turn_pass();
      attn_wait<0>(o);
      release_v(g + nch - 1);
      g += nch;
      ++nq;
    }

    // ---------------- epilogue: O / l -> global (optionally scattered rows), LSE
    // batch element and head of the o store (the row gather: its one batch element), derived per stream rather than
    // kept live through the chunk loop, since the consumers are register-bound
    long long o_base = bh * args.o_head_stride;
    float* lse_out = args.lse;
    if constexpr (!kGather) {
      const int bhe = ctaid_y_here(), batch = bhe / args.Hq;
      o_base = batch * args.o_batch_stride + (bhe - batch * args.Hq) * args.o_head_stride;
      if (args.split_items) {  // split KV-cache plans: the fp32 partial o and LSE of this CTA's split
        const int sp = static_cast<int>(blockIdx.x) / args.split_items;
        o_base += sp * args.o_split_stride;
        lse_out += static_cast<size_t>(sp) * gridDim.y * args.S;
      }
    }
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
        float* optr = reinterpret_cast<float*>(args.o) + o_base + out_row * args.o_row_stride;
#pragma unroll
        for (int jj = 0; jj < D / 8; ++jj)
          *reinterpret_cast<float2*>(optr + 8 * jj + col0) =
              make_float2(o[4 * jj + 2 * v1] * inv_l, o[4 * jj + 2 * v1 + 1] * inv_l);
      } else {
        uint16_t* optr = reinterpret_cast<uint16_t*>(args.o) + o_base + out_row * args.o_row_stride;
#pragma unroll
        for (int jj = 0; jj < D / 8; ++jj)
          *reinterpret_cast<uint32_t*>(optr + 8 * jj + col0) =
              pack2<BF16>(o[4 * jj + 2 * v1] * inv_l, o[4 * jj + 2 * v1 + 1] * inv_l);
      }
      if (args.lse && (lane & 3) == 0) {
        // natural-log LSE of the scaled scores; -inf for rows that saw no key
        const float lse = l > 0.f ? (m_run[v1] * crow(v1) + log2f(l)) * 0.6931471805599453f : -INFINITY;
        lse_out[static_cast<size_t>(bh) * args.S + out_row] = lse;
      }
    }
  }
  if (cw == 0) turn_wait();  // consumer 1's hand-over after its last turn, so no named barrier is left pending
}

}  // namespace svgb
