// Shared definitions for the block-sparse attention path: the device-resident "plan" (work items +
// KV chunk lists) that every mask family (SVG2 variable blocks, SVG1 band masks, BSR, dense) is
// lowered to, and the element-mask predicates used on partial tiles.
#pragma once
#include <cuda_runtime.h>
#include <limits.h>
#include <stdint.h>

namespace svgb {

// One work item = one CTA = two STREAM descriptors, items[2 * item + st] (st = 0, 1), run one after the other:
//   stream = {q_row0, nrows (0..128; 0 = no stream), list_off, list_len}
// A stream is up to 128 consecutive query rows of one head (one MMA tile) over the list at chunks + list_off.
// Stream 0 always has rows; stream 1 has nrows == 0 when the CTA runs one stream.  The planners cut query rows into
// items of up to kItemRows rows (put_item); a variable-block TMA plan also pairs two tails of different q-blocks,
// each with its own list.  The list is
//   TMA plans   : list_len chunks {kv_start, meta}; meta bits [0,8) = valid columns - 1 (0..127), bit 8 = ELEM
//                 (evaluate the element mask predicate on this chunk), bit 9 = reserved; KV-cache plans only: bits
//                 [10,32) = the chunk's logical index j (keys 128 j .. of its stream), the position the mask sees, while
//                 kv_start is the physical row its TMA box loads from.
//   gather plans: list_len runs {src_start, keys before the run} of the selected key ranges and a sentinel
//                 {0, total}; the kernel gathers exactly-full 128-key chunks across run boundaries.
constexpr int kItemRows = 256;
constexpr int kTileRows = 128;
constexpr int kChunkCols = 128;
constexpr int kChunkElem = 1 << 8;

__host__ __device__ inline int chunk_meta(int valid, bool elem) {
  return ((valid - 1) & 0xff) | (elem ? kChunkElem : 0);
}
__host__ __device__ inline int chunk_valid(int meta) { return (meta & 0xff) + 1; }
constexpr int kChunkLogicalShift = 10;
// first logical key of a KV-cache chunk (128 j); j < 2^22, so the shift never reaches the sign bit
__host__ __device__ inline int chunk_logical_kv0(int meta) {
  return static_cast<int>(static_cast<unsigned>(meta) >> kChunkLogicalShift) * kChunkCols;
}

// the two streams of an item of nrows (1..kItemRows) consecutive query rows from q0, both over one list
__device__ inline void put_item(int4* item, int q0, int nrows, int list_off, int list_len) {
  item[0] = make_int4(q0, min(nrows, kTileRows), list_off, list_len);
  item[1] = make_int4(q0 + kTileRows, max(nrows - kTileRows, 0), list_off, list_len);
}

// Element mask families (SURVEY §8 a5): parameters m0,m1,m2.
enum MaskMode : int {
  MASK_NONE = 0,
  // HunyuanVideo (text last), reference svg/models/hyvideo/utils.py:20-44
  //   m0 = V = F*P, m1 = R = V + prompt_len, m2 = W
  MASK_HY = 1,
  // Wan / Cosmos (no text, first-frame sink), reference svg/models/wan/utils.py:25-41
  //   m0 = P (tokens per frame), m2 = W   : kv < P | |q-kv| <= W
  MASK_WAN = 2,
  // CogVideoX (text first), reference svg/models/cog/utils.py:30-46
  //   m0 = first-column limit (prompt_len or prompt_len + P), m1 = prompt_len, m2 = W
  MASK_COG = 3,
  // SVG1 profiling masks of get_attention_mask (hyvideo/utils.py:47-93, wan/utils.py:63-110),
  // evaluated analytically: 128-token-block band |bq - bk| < thres in frame-major (spatial) or
  // token-major (temporal) order.  m0 = F, m1 = P, m2 = thres (blocks).  HY: text rows / columns
  // (index >= F*P) always attend; WAN: first-frame sink painted before the token-major permutation.
  MASK_PROF_HY_S = 4,
  MASK_PROF_HY_T = 5,
  MASK_PROF_WAN_S = 6,
  MASK_PROF_WAN_T = 7,
  // CogVideoX (text FIRST) profiling masks, svg/models/cog/utils.py:61-88.  m2 = thres | ctx << 12.
  //   spatial : text rows / columns all-ones; the 128-token block band is painted in ABSOLUTE sequence
  //             coordinates (blocks 0 .. ceil(F*P/128)-1 from row / column 0, cog/utils.py:68-74)
  //   temporal: band in token-major order on the video x video part only; text rows and columns stay zero
  //             (cog/utils.py:76-86) -- a sampled text row has no allowed key at all
  MASK_PROF_COG_S = 8,
  MASK_PROF_COG_T = 9,
  // Local band with attention sinks (causal, sliding window, StreamingLLM):
  //   m0 = sink, m1 = left, m2 = right (all >= 0)   : kv < sink | (q - kv <= left & kv - q <= right)
  // MASK_WAN(P, W) is MASK_LOCAL(P, W, W).
  MASK_LOCAL = 10,
  // Block-causal mask of autoregressive video (chunk-wise causal, CausVid / Self-Forcing): positions form blocks of C
  // with ends at F, F + C, F + 2C, ... (1 <= F <= C), e(q) the first end past q, and
  //   m0 = sink, m1 = C | (C - F) << 16, m2 = W >= C   : kv < sink | (e(q) - W <= kv < e(q))
  // With q rounded to its block's last position e(q) - 1 (block_last) it is MASK_LOCAL(sink, W - 1, 0); W >= C keeps
  // every row's own block.  Mode 11 is unassigned.
  MASK_BLOCK_CAUSAL = 12,
};

// MASK_BLOCK_CAUSAL: the last position e(p) - 1 of p's block, m1 = C | (C - F) << 16.  Positions before the first
// block end (negative ones too: KV-cache queries ahead of their keys) belong to the first block.
__host__ __device__ inline int block_last(int p, int m1) {
  const int C = m1 & 0xffff, F = C - (m1 >> 16);
  return p < F ? F - 1 : p + (C - 1) - (p - F) % C;
}

// the same inside a segment whose block grid is anchored at key position key0 (SegOrigin::key0; 0 for other plans)
__host__ __device__ inline int seg_block_last(int p, int key0, int m1) { return key0 + block_last(p - key0, m1); }

__host__ __device__ inline bool mask_allowed(int mode, int q, int kv, int m0, int m1, int m2) {
  // reference semantics, written branch-free (bitwise) so warps do not diverge on it
  int d = q - kv;
  d = d < 0 ? -d : d;
  switch (mode) {
    case MASK_HY: {
      const bool real = (q < m1) & (kv < m1);
      const bool fake = (q >= m1) & (kv >= m1);
      const bool vid = (d < m2) | (kv >= m0) | (q >= m0);
      return (real & vid) | fake;
    }
    case MASK_WAN:  // MASK_LOCAL(m0, m2, m2), kept as |q - kv| (DESIGN §1: fewer instructions in the ELEM chunks)
      return (kv < m0) | (d <= m2);
    case MASK_LOCAL:
      return (kv < m0) | ((q - kv <= m1) & (kv - q <= m2));
    case MASK_BLOCK_CAUSAL: {
      const int e = block_last(q, m1);
      return (kv < m0) | ((kv <= e) & (e - kv <= m2 - 1));
    }
    case MASK_COG:
      return (kv < m0) | (q < m1) | (d < m2);
    case MASK_PROF_COG_S: {
      const int thres = m2 & 0xfff, ctx = m2 >> 12;
      const int lim = ((m0 * m1 + 127) / 128) * 128;
      int bd = q / 128 - kv / 128;
      bd = bd < 0 ? -bd : bd;
      return (q < ctx) | (kv < ctx) | ((q < lim) & (kv < lim) & (bd < thres));
    }
    case MASK_PROF_COG_T: {
      const int thres = m2 & 0xfff, ctx = m2 >> 12;
      if (q < ctx || kv < ctx) return false;
      const int F = m0, P = m1;
      const int qv = q - ctx, kvv = kv - ctx;
      int bd = ((qv % P) * F + qv / P) / 128 - ((kvv % P) * F + kvv / P) / 128;
      bd = bd < 0 ? -bd : bd;
      return bd < thres;
    }
    case MASK_PROF_HY_S:
    case MASK_PROF_HY_T:
    case MASK_PROF_WAN_S:
    case MASK_PROF_WAN_T: {
      const int F = m0, P = m1, V = m0 * m1;
      const bool hy = mode <= MASK_PROF_HY_T;
      const bool temporal = (mode == MASK_PROF_HY_T) || (mode == MASK_PROF_WAN_T);
      if (q >= V || kv >= V) return hy;  // text rows / columns (HY); cannot occur for WAN (S == V)
      const int qi = temporal ? (q % P) * F + q / P : q;
      const int ki = temporal ? (kv % P) * F + kv / P : kv;
      int bd = qi / 128 - ki / 128;
      bd = bd < 0 ? -bd : bd;
      return (bd < m2) | (!hy & (ki < P));
    }
    default:
      return true;
  }
}

// Packed variable-length segments (SVGB_PLAN_SEG / SVGB_PLAN_SEG_T).  The plan keeps its own copy of the bounds at byte
// SVGB_PLAN_SEG_BOUNDS_OFF of its workspace, seg = {nseg, cq_0 .. cq_nseg, ck_0 .. ck_nseg}: query segment i is rows
// [cq_i, cq_i+1), key segment i keys [ck_i, ck_i+1).
// Every stream lies in one segment, so the local mask of segment i is MASK_LOCAL(sink, left, right) with two per-stream
// constants: query positions shifted by delta_i = cq_i+1 - ck_i+1 (query qi of the segment sits at key position
// ck_i + qi + Lk_i - Lq_i, FlashAttention's bottom-right alignment) and the sink bound ck_i + sink in place of m0.
// The same segment is implicit: a stream's chunks are keys (key-major: queries) of its own segment only.
struct SegOrigin {
  int shift;     // subtract from a query position
  int sink_end;  // m0 of the stream: keys below it are sinks
  int key0 = 0;  // the segment's first key ck_i, where its block grid is anchored; 0 for every other plan
};
// origin of the stream whose first row is `row`: a query row (key_major = false) or a key row (true).  Its segment is
// the last one that starts at or before it, so empty segments are skipped.
__host__ __device__ inline SegOrigin seg_origin(const int* seg, int row, bool key_major, int sink) {
  const int nseg = seg[0];
  const int* segs = seg + 1;
  const int* b = segs + (key_major ? nseg + 1 : 0);
  int lo = 0, hi = nseg - 1;  // largest i < nseg with b[i] <= row
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (b[mid] <= row) lo = mid;
    else hi = mid - 1;
  }
  const int* ck = segs + nseg + 1;
  SegOrigin o;
  o.shift = segs[lo + 1] - ck[lo + 1];
  o.sink_end = ck[lo] + sink;
  o.key0 = ck[lo];
  return o;
}

// KV-cache plans (SVGB_PLAN_KVCACHE, and SVGB_PLAN_KVCACHE_SPLIT with the same header).  The plan keeps at byte SVGB_PLAN_SEG_BOUNDS_OFF of its workspace
// kv = {B, Sq, L_0 .. L_B-1}: stream b has its queries at packed rows [b Sq, (b+1) Sq) and L_b keys at logical positions
// 0 .. L_b - 1 (clamped to its capacity).  Query row q of stream b sits at logical position L_b - Sq + (q - b Sq), so the
// mask is MASK_LOCAL(sink, left, right) on logical positions with shift (b+1) Sq - L_b and the sink bound `sink`; the
// key positions come from each chunk's logical index (chunk_logical_kv0), not from its physical row.
__host__ __device__ inline SegOrigin kv_origin(const int* kv, int row, int sink) {
  const int Sq = kv[1], b = row / Sq;
  SegOrigin o;
  o.shift = (b + 1) * Sq - kv[2 + b];
  o.sink_end = sink;
  return o;
}

// Variable-length KV-cache plans (svgb_attn_plan_kvcache_varlen) keep kv = {B, kKvVarlen, L_0 .. L_B-1, cu_0 .. cu_B}:
// stream b has its queries at packed rows [cu_b, cu_b+1) and query row q sits at logical position L_b - (cu_b+1 - q), so
// the shift is cu_b+1 - L_b.  The marker in the Sq slot tells the header from a uniform one; the stream of a row is the
// last one that starts at or before it (empty streams are skipped), found by binary search as seg_origin does.
constexpr int kKvVarlen = -1;
__host__ __device__ inline SegOrigin kv_origin_varlen(const int* kv, int row, int sink) {
  const int B = kv[0];
  const int* cu = kv + 2 + B;
  int lo = 0, hi = B - 1;  // largest b < B with cu[b] <= row
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (cu[mid] <= row) lo = mid;
    else hi = mid - 1;
  }
  SegOrigin o;
  o.shift = cu[lo + 1] - kv[2 + lo];
  o.sink_end = sink;
  return o;
}
// the origin of the stream of `row` under either KV-cache header
__host__ __device__ inline SegOrigin kv_stream_origin(const int* kv, int row, int sink) {
  return kv[1] == kKvVarlen ? kv_origin_varlen(kv, row, sink) : kv_origin(kv, row, sink);
}

// Kind of a chunk of a segment plan, from the mask's interval form: 0 = omitted (no allowed pair), 1 = FULL (every pair
// allowed), 2 = ELEM.  Query-major: rows r0..r1 are queries at positions p = q - shift, columns c0..c1 keys.  Key-major:
// rows are keys, columns queries.  Pairs (p, kv) are allowed when kv < sink_end or p - left <= kv <= p + right; every
// key of the chunk and of the item lies in the segment (kv >= sink_end - sink).  64-bit: left / right may be large.
__host__ __device__ inline int seg_chunk_kind(bool key_major, int r0, int r1, int c0, int c1, SegOrigin o, int left,
                                              int right) {
  const long long L = left, R = right;
  if (!key_major) {
    const long long p0 = static_cast<long long>(r0) - o.shift, p1 = static_cast<long long>(r1) - o.shift;
    const bool any = c0 < o.sink_end || (c0 <= p1 + R && c1 >= p0 - L);
    const long long k = c0 > o.sink_end ? c0 : o.sink_end;  // first key past the sinks
    const bool all = k > c1 || (k >= p1 - L && c1 <= p0 + R);
    return any ? (all ? 1 : 2) : 0;
  }
  // key kv is reached by positions kv - right .. kv + left, i.e. queries kv + shift - right .. kv + shift + left
  const long long k0 = r0 > o.sink_end ? r0 : o.sink_end;  // first key of the item past the sinks
  const bool any = r0 < o.sink_end || (c0 <= r1 + o.shift + L && c1 >= r0 + o.shift - R);
  const bool all = k0 > r1 || (c0 >= r1 + o.shift - R && c1 <= k0 + o.shift + L);
  return any ? (all ? 1 : 2) : 0;
}

// MASK_BLOCK_CAUSAL, key-major: the positions p that reach key k >= 0 (both relative to the segment's first key, k not
// a sink) are those with k + 1 <= e(p) <= k + W, the interval [lo, hi]: lo is the first position of k's block (none
// for k < F, where negative positions share the first block) and hi is one less than the last block end <= k + W
// (k + W >= W >= C >= F, so there is one).  Both bounds are nondecreasing in k.
struct PosSpan {
  long long lo, hi;
};
__host__ __device__ inline PosSpan block_reach(int k, int m1, int W) {
  const int C = m1 & 0xffff, F = C - (m1 >> 16);
  const long long x = static_cast<long long>(k) + W;
  PosSpan s;
  s.lo = k < F ? LLONG_MIN / 2 : k - (k - F) % C;
  s.hi = x - (x - F) % C - 1;
  return s;
}

// Kind of a chunk of a key-major block-causal segment plan (0 / 1 / 2 as seg_chunk_kind): rows r0..r1 are keys, columns
// c0..c1 queries at positions c - shift, of the segment of o.  The keys past the sinks, k0..r1, are reached by the union
// [lo(k0), hi(r1)] of their intervals (consecutive ones touch: hi(k) >= k + W - C >= k) and, all of them, by the
// intersection [lo(r1), hi(k0)]; the sink keys by every query of the segment.
__host__ __device__ inline int seg_block_chunk_kind_t(int r0, int r1, int c0, int c1, SegOrigin o, int m1, int W) {
  const int k0 = r0 > o.sink_end ? r0 : o.sink_end;  // first key of the item past the sinks
  const long long p0 = static_cast<long long>(c0) - o.shift - o.key0, p1 = static_cast<long long>(c1) - o.shift - o.key0;
  const PosSpan a = block_reach(k0 - o.key0, m1, W), b = block_reach(r1 - o.key0, m1, W);
  const bool any = r0 < o.sink_end || (k0 <= r1 && p0 <= b.hi && p1 >= a.lo);
  const bool all = k0 > r1 || (p0 >= b.lo && p1 <= a.hi);
  return any ? (all ? 1 : 2) : 0;
}

// Element masks inside the attention kernel.  A thread holds the scores of two query rows at positions q[0], q[1]
// and key columns kvb + 8*jj + v0 (jj < 16, v0 < 2; kvb = chunk start + 2*(lane % 4)), the wgmma accumulator
// layout.  ElemMask::bits returns them as two 32-bit masks: bit 2*jj + v0 of keep[v1] <=> mask_allowed(mode, q[v1],
// kvb + 8*jj + v0).
// The mask family is dispatched once per chunk, never per element.  The band families and the CogVideoX spatial
// profiling mask inline mask_allowed with the mode as a compile-time constant (comparisons and shifts only).  The
// banded profiling masks (HY / WAN spatial and temporal, COG temporal) hoist the query's 128-token block to init
// (once per stream) and, in temporal order, step the key's (frame, token) pair across the columns: one division
// per chunk instead of two per element.
struct ElemMask {
  int mode, m0, m1, m2;
  // per query row, one register (the kernel is register-bound):
  //   direct families: the query position (block-causal: its block's last position, evaluated as MASK_LOCAL)
  //   banded profiling masks: band_lo = qblk - thres + 1, the first key block of the row's band, so that
  //   |qblk - kblk| < thres <=> (unsigned)(kblk - band_lo) < 2*thres - 1; or kRowOut when the query lies outside
  //   the banded part (every key then gives Prof::outside_val)
  int row[2];
  static constexpr int kRowOut = INT_MIN;  // band_lo >= INT_MIN + 2 for 0 < thres <= INT_MAX, and 0 for thres <= 0

  // parameters of the banded profiling masks, in the form the evaluator uses
  struct Prof {
    int F, P, off, lim, thres;  // token index r = position - off; r < 0 or r >= lim is outside the band
    bool temporal, outside_val, sink;  // sink: WAN first frame (token-major index < P) always attends
  };
  __device__ __forceinline__ static bool banded(int mode) {
    return (mode >= MASK_PROF_HY_S && mode <= MASK_PROF_WAN_T) || mode == MASK_PROF_COG_T;
  }
  __device__ __forceinline__ Prof prof() const {
    Prof p;
    p.F = m0;
    p.P = m1;
    const bool cog = mode == MASK_PROF_COG_T;
    // HY / WAN: text rows and columns (index >= F*P) give `hy`.  COG temporal: text comes first (index < ctx)
    // and gives false; there is no upper limit (mask_allowed bands every index >= ctx)
    p.off = cog ? m2 >> 12 : 0;
    p.lim = cog ? INT_MAX : m0 * m1;
    p.thres = cog ? m2 & 0xfff : m2;
    p.temporal = cog || mode == MASK_PROF_HY_T || mode == MASK_PROF_WAN_T;
    p.outside_val = mode == MASK_PROF_HY_S || mode == MASK_PROF_HY_T;
    p.sink = mode == MASK_PROF_WAN_S || mode == MASK_PROF_WAN_T;
    return p;
  }

  // key0: where the block grid is anchored (SegOrigin::key0), so a block-causal row rounds inside its segment
  __device__ __forceinline__ void init(int mode_, const int (&qm)[2], int m0_, int m1_, int m2_, int key0) {
    mode = mode_; m0 = m0_; m1 = m1_; m2 = m2_;
    const bool block = mode == MASK_BLOCK_CAUSAL;
#pragma unroll
    for (int v1 = 0; v1 < 2; ++v1) row[v1] = block ? seg_block_last(qm[v1], key0, m1_) : qm[v1];
    if (block) {  // rows rounded to their block ends: the local band (sink, W - 1, 0), no division per element
      mode = MASK_LOCAL;
      m1 = m2_ - 1;
      m2 = 0;
    }
    if (!banded(mode)) return;
    const Prof p = prof();
#pragma unroll
    for (int v1 = 0; v1 < 2; ++v1) {
      const int r = qm[v1] - p.off;
      if (r < 0 || r >= p.lim) {
        row[v1] = kRowOut;
      } else {
        const int qi = p.temporal ? (r % p.P) * p.F + r / p.P : r;
        row[v1] = p.thres > 0 ? static_cast<int>(static_cast<uint32_t>(qi >> 7) - static_cast<uint32_t>(p.thres) + 1u) : 0;
      }
    }
  }

  template <int kMode>
  __device__ __forceinline__ void bits_direct(int kvb, uint32_t (&keep)[2]) const {
#pragma unroll 1
    for (int jj = 0; jj < 16; ++jj)
#pragma unroll
      for (int v0 = 0; v0 < 2; ++v0) {
        const int kv = kvb + 8 * jj + v0;
#pragma unroll
        for (int v1 = 0; v1 < 2; ++v1)
          keep[v1] |= (mask_allowed(kMode, row[v1], kv, m0, m1, m2) ? 1u : 0u) << (2 * jj + v0);
      }
  }

  template <bool kTemporal>
  __device__ __forceinline__ void bits_banded(int kvb, uint32_t (&keep)[2]) const {
    const Prof pr = prof();
    const int F = pr.F, P = pr.P;
    const uint32_t width = pr.thres > 0 ? 2u * static_cast<uint32_t>(pr.thres) - 1u : 0u;
    const int r0 = kvb - pr.off;
    // temporal: (f, p) = floor division of the token index by P, stepped by 1 within a column pair and by 8
    // (= f8 frames + p8 tokens) from one pair to the next
    int f = 0, p = 0, f8 = 0, p8 = 0;
    if (kTemporal) {
      f = r0 >= 0 ? r0 / P : -((P - 1 - r0) / P);
      p = r0 - f * P;
      f8 = 8 / P;
      p8 = 8 - f8 * P;
    }
#pragma unroll 1
    for (int jj = 0; jj < 16; ++jj) {
      int fc = f, pc = p;
#pragma unroll
      for (int v0 = 0; v0 < 2; ++v0) {
        const int r = r0 + 8 * jj + v0;
        const int ki = kTemporal ? pc * F + fc : r;
        const bool col_out = r < 0 || r >= pr.lim;
        const bool sink = pr.sink & (ki < P);
        const uint32_t kb = static_cast<uint32_t>(ki >> 7);
#pragma unroll
        for (int v1 = 0; v1 < 2; ++v1) {
          const bool out = row[v1] == kRowOut || col_out;
          const bool a = out ? pr.outside_val : ((kb - static_cast<uint32_t>(row[v1]) < width) | sink);
          keep[v1] |= (a ? 1u : 0u) << (2 * jj + v0);
        }
        if (kTemporal && v0 == 0) {
          ++pc;
          if (pc == P) {
            pc = 0;
            ++fc;
          }
        }
      }
      if (kTemporal) {
        p += p8;
        f += f8;
        if (p >= P) {
          p -= P;
          ++f;
        }
      }
    }
  }

  __device__ __forceinline__ void bits(int kvb, uint32_t (&keep)[2]) const {
    keep[0] = keep[1] = 0;
    if (mode == MASK_HY) bits_direct<MASK_HY>(kvb, keep);
    else if (mode == MASK_WAN) bits_direct<MASK_WAN>(kvb, keep);
    else if (mode == MASK_COG) bits_direct<MASK_COG>(kvb, keep);
    else if (mode == MASK_LOCAL) bits_direct<MASK_LOCAL>(kvb, keep);
    else if (mode == MASK_PROF_COG_S) bits_direct<MASK_PROF_COG_S>(kvb, keep);
    else if (mode == MASK_PROF_HY_S || mode == MASK_PROF_WAN_S) bits_banded<false>(kvb, keep);
    else if (banded(mode)) bits_banded<true>(kvb, keep);
    else keep[0] = keep[1] = ~0u;  // MASK_NONE (mask_allowed's default)
  }
};

struct AttnArgs {
  const int4* items = nullptr;      // two stream descriptors per item
  const int* item_count = nullptr;  // [BH] when items_stride != 0, else [1]
  const int2* chunks = nullptr;     // chunk or run lists
  int items_stride = 0;             // 0: one plan shared by all heads (band masks); else items per head
  // query heads per key/value head (grouped-query attention): query head bh reads K / V head bh / kv_group, and so
  // does the plan (built over the key/value heads); Q, O and LSE stay at bh
  int kv_group = 1;
  // query heads per batch element: CTA head bh is query head bh % Hq of batch element bh / Hq, which the tensor maps
  // (d, row, head, batch) and the o store address; the plan, LSE and the row vectors index the flat bh
  int Hq = 1;
  void* o = nullptr;
  long long o_row_stride = 0;    // elements
  long long o_head_stride = 0;   // elements
  long long o_batch_stride = 0;  // elements
  const int* o_rows = nullptr;  // optional [BH, S]: output row for query row q (fused inverse permutation)
  float* lse = nullptr;         // optional [BH, S] (natural log), indexed like o rows
  float scale_log2 = 0;         // softmax scale * log2(e)
  int S = 0;                    // query rows per head (indexing of o_rows / lse / q_index)
  int mask_mode = 0, m0 = 0, m1 = 0, m2 = 0;
  const int* q_index = nullptr;  // optional [S]: query position used by the element mask (sampled rows)
  // segment plans: the plan's copy of the bounds {nseg, cq[0..nseg], ck[0..nseg]} (seg_origin); nullptr otherwise
  const int* segs = nullptr;
  // KV-cache plans: segs is the plan's {B, Sq, L_b} (kv_origin) or its varlen header (kv_origin_varlen), and element
  // masks see each chunk's logical position
  int kv_logical = 0;
  int out_f32 = 0;               // 1: o is fp32 (used for split-KV partials)
  // split KV-cache plans (SVGB_PLAN_KVCACHE_SPLIT): the plan's items per split, so that CTA x runs split
  // x / split_items, whose fp32 partial o starts o_split_stride elements and whose partial LSE gridDim.y * S floats
  // after the previous split's.  0: no split
  int split_items = 0;
  long long o_split_stride = 0;
  // FP8 (e4m3) inputs: per-head dequantisation scales, q_scale [BH] by query head, k_scale and v_scale [BH / kv_group]
  // by key/value head; s_q * s_k multiplies the logits, s_v the output.  NULL for 16-bit inputs.
  const float* q_scale = nullptr;
  const float* k_scale = nullptr;
  const float* v_scale = nullptr;
  // ---- gather mode (SVG2; attn_fwd_kernel<..., kGather = true>, run lists): K/V rows are gathered with cp.async,
  // optionally through row-index vectors so the cluster permutation of Q, K, V never materialises in HBM.
  const int* q_rows = nullptr;      // optional [BH, S]: source row of (permuted) query row
  const int* kv_rows = nullptr;     // optional [BH, S]: source row of (permuted) key/value row
  const void* q_ptr = nullptr;      // raw tensors for the gather path ([BH,S,D] with the strides below)
  const void* k_ptr = nullptr;
  const void* v_ptr = nullptr;
  long long in_row_stride = 0, in_head_stride = 0;  // elements
  // ---- per-row FP8 (attn_fwd_kernel<128, DT_E4M3_ROWS, false>, KV-cache plans): block_rows of the cache, which splits a
  // chunk's physical row into (block, row) for its scale boxes; q_scale is then [BH, S] like the LSE and the K / V row
  // scales come through their own tensor maps.  0 otherwise.
  int scale_block_rows = 0;
};

}  // namespace svgb
