// Attention plans (device-built work lists), the attention launcher, density, and the tile
// self-test.  See attn_kernel.cuh for the kernel itself.
#include <algorithm>

#include "../../include/svgb200.h"
#include "attn_kernel.cuh"
#include "host_common.h"

namespace svgb {

// =============================================================================================
// Plan: variable blocks (SVG2 dynamic map / BSR / dense)
//   one CTA per head; thread per q-block walks its map row, merges selected k-blocks that are
//   adjacent in token space into runs and cuts runs into <=128-column chunks.
// =============================================================================================
// Two kernels.  (1) plan_lists_kernel -- grid (ceil(QC/8), BH), one WARP per q-block: the map row is read with
// coalesced byte loads 32 columns at a time, a ballot gives the selected non-empty k-blocks, the (warp-uniform) run
// walk visits only the set bits and the chunks of a finished run are written by the lanes in parallel;
// (2) plan_items_kernel -- one CTA per head: work items from the row sizes and list lengths.
// (The first version walked each row byte by byte with one thread: 0.37 ms at 24 x 400 x 1000; this one ~0.02 ms.)
constexpr int kPlanWarps = 8;
__global__ void __launch_bounds__(kPlanWarps * 32)
plan_lists_kernel(const uint8_t* __restrict__ map, const int* __restrict__ row_sz, const int* __restrict__ col_sz,
                  int QC, int KC, int chunk_cap, int gather, int2* __restrict__ chunks, int* __restrict__ nch_of) {
  // gather form: the list holds RUNS {start, keys before this run} plus a sentinel {0, total}; the kernel then
  // gathers exactly-full 128-key chunks across run boundaries.
  extern __shared__ int sm[];
  int* coloff = sm;  // KC + 1
  __shared__ int wsum[kPlanWarps];
  const int bh = blockIdx.y;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  row_sz += static_cast<size_t>(bh) * QC;
  col_sz += static_cast<size_t>(bh) * KC;
  // exclusive prefix sum of the key-block sizes: a contiguous slice per thread, warp scan, serial pass over 8 warp sums
  {
    const int nthr = kPlanWarps * 32;
    const int per = (KC + nthr - 1) / nthr;
    const int j0 = min(KC, static_cast<int>(threadIdx.x) * per), j1 = min(KC, j0 + per);
    int acc = 0;
    for (int j = j0; j < j1; ++j) acc += col_sz[j];
    int incl = acc;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int n = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += n;
    }
    if (lane == 31) wsum[warp] = incl;
    __syncthreads();
    int base = incl - acc;
    for (int w = 0; w < warp; ++w) base += wsum[w];
    for (int j = j0; j < j1; ++j) {
      coloff[j] = base;
      base += col_sz[j];
    }
    if (threadIdx.x == nthr - 1) coloff[KC] = base;  // the last thread's slice ends at KC (possibly empty)
  }
  __syncthreads();
  const int qb = blockIdx.x * kPlanWarps + warp;
  if (qb >= QC) return;
  const size_t list = (static_cast<size_t>(bh) * QC + qb) * chunk_cap;
  int2* out = chunks + list;
  const uint8_t* mrow = map + (static_cast<size_t>(bh) * QC + qb) * KC;
  int n = 0, total = 0;  // warp-uniform
  if (row_sz[qb] > 0) {
    int run_s = -1, run_e = -1;
    auto flush = [&]() {
      if (gather) {
        if (n < chunk_cap - 1) {
          if (lane == 0) out[n] = make_int2(run_s, total);
          ++n;
        }
        total += run_e - run_s;
      } else {
        const int cnt = min((run_e - run_s + kChunkCols - 1) / kChunkCols, chunk_cap - n);
        for (int c = lane; c < cnt; c += 32) {
          const int p = run_s + c * kChunkCols;
          out[n + c] = make_int2(p, chunk_meta(min(kChunkCols, run_e - p), false));
        }
        n += cnt;
      }
    };
    for (int j0 = 0; j0 < KC; j0 += 32) {
      const int j = j0 + lane;
      const bool sel = j < KC && mrow[j] != 0 && coloff[j + 1] > coloff[j];
      unsigned m = __ballot_sync(0xffffffffu, sel);
      while (m) {
        const int jj = j0 + __ffs(m) - 1;
        m &= m - 1;
        const int s = coloff[jj], e = coloff[jj + 1];
        if (run_s >= 0 && s == run_e) {
          run_e = e;  // contiguous in token space (only empty k-blocks in between): extend
        } else {
          if (run_s >= 0) flush();
          run_s = s;
          run_e = e;
        }
      }
    }
    if (run_s >= 0) flush();
    if (gather && lane == 0) out[n] = make_int2(0, total);  // sentinel: ends the last run
  }
  if (lane == 0) nch_of[static_cast<size_t>(bh) * QC + qb] = n;
}

__global__ void plan_items_kernel(const int* __restrict__ row_sz, const int* __restrict__ nch_all, int QC,
                                  int max_items, int chunk_cap, int gather, int* __restrict__ counts,
                                  int4* __restrict__ items) {
  // TMA form: a q-block of r rows becomes r/256 two-tile items (+ one more when r % 256 > 128, its second tile
  // partial) and, when 0 < r % 256 <= 128, a single-tile TAIL.  Tails are where k-means clusters lose tensor-core
  // rows (a 297-row cluster = 256 + 41) and a lone single-tile CTA leaves half of the softmax warps idle, so the
  // tails of a head are sorted by chunk count and packed two per CTA, one per stream, each with its own list.
  // Launch order: two-tile items in q-block order, then the paired tails from long to short.  Gather form: every
  // q-block is cut into items of up to 256 rows; tails are not paired.
  extern __shared__ int sm[];
  int* rowoff = sm;                 // QC + 1
  int* itembase = rowoff + QC + 1;  // QC + 1 : first two-tile item of the q-block (gather: first item)
  int* long_of = itembase + QC + 1; // QC     : rows of the q-block's tail (1..128; 0 = none) -> paired
  int* nch_of = long_of + QC;       // QC
  __shared__ int s_total2, s_nlong;
  const int bh = blockIdx.x;
  row_sz += static_cast<size_t>(bh) * QC;
  const bool pair = !gather;
  for (int i = threadIdx.x; i < QC; i += blockDim.x) {
    nch_of[i] = nch_all[static_cast<size_t>(bh) * QC + i];
    rowoff[i] = row_sz[i];  // staged: the serial pass below turns the sizes into offsets in place
  }
  __syncthreads();
  // the last r % 256 rows of a q-block (pair == true): a tail when there are at most 128 of them, otherwise one
  // more two-tile item (second tile partial)
  if (threadIdx.x == 32) {
    int acc = 0, it = 0, nl = 0;
    for (int i = 0; i < QC; ++i) {
      const int r = rowoff[i];
      rowoff[i] = acc;
      itembase[i] = it;
      acc += r;
      const int rem = r % kItemRows;
      int lg = 0, n2 = (r + kItemRows - 1) / kItemRows;
      if (pair && rem > 0 && rem <= kTileRows) {
        lg = rem;
        n2 = r / kItemRows;
      }
      long_of[i] = lg;
      nl += lg > 0;
      it += n2;
    }
    rowoff[QC] = acc;
    itembase[QC] = it;
    s_total2 = it;
    s_nlong = nl;
    const int total = it + (nl + 1) / 2;
    counts[bh] = total < max_items ? total : max_items;
  }
  __syncthreads();
  for (int qb = threadIdx.x; qb < QC; qb += blockDim.x) {
    const int r = rowoff[qb + 1] - rowoff[qb];
    if (r == 0) continue;
    const size_t list = (static_cast<size_t>(bh) * QC + qb) * chunk_cap;
    const int n = nch_of[qb];
    const int nit = itembase[qb + 1] - itembase[qb];
    for (int t = 0; t < nit; ++t) {
      const int idx = itembase[qb] + t;
      if (idx < max_items)
        put_item(items + 2 * (static_cast<size_t>(bh) * max_items + idx), rowoff[qb] + t * kItemRows,
                 min(kItemRows, r - t * kItemRows), static_cast<int>(list), n);
    }
  }
  if (!pair) return;
  // tails: rank by (chunk count descending, q-block ascending); ranks 2i and 2i+1 are streams 0 and 1 of CTA i
  const int base = s_total2;
  int4* pairs = items + 2 * (static_cast<size_t>(bh) * max_items + base);
  const int cap = max_items - base;
  for (int qb = threadIdx.x; qb < QC; qb += blockDim.x) {
    const int rows = long_of[qb];
    if (rows == 0) continue;
    const int mine = nch_of[qb];
    int rank = 0;
    for (int o = 0; o < QC; ++o)
      if (long_of[o] > 0 && (nch_of[o] > mine || (nch_of[o] == mine && o < qb))) ++rank;
    const int r = rowoff[qb + 1] - rowoff[qb];
    const int4 it = make_int4(rowoff[qb] + (r / kItemRows) * kItemRows, rows,
                              static_cast<int>((static_cast<size_t>(bh) * QC + qb) * chunk_cap), mine);
    if ((rank >> 1) < cap) {
      pairs[rank] = it;
      if (rank == s_nlong - 1 && (rank & 1) == 0) pairs[rank + 1] = make_int4(0, 0, 0, 0);  // odd one out
    }
  }
}

// =============================================================================================
// Plan: element-exact band masks (SVG1).  One CTA per work item; thread = query row; for every
// 128-column chunk the block votes any/all over the item's rows.  Exact by construction.
// Items never straddle a row-region boundary of the mask (video | prompt | padding for HunyuanVideo,
// text | video for CogVideoX), so text rows -- which see every column -- do not drag 256-row items of
// video rows onto the per-element path; the heavy text items are issued first (LPT).
// =============================================================================================
struct BandSegs {
  int n;             // number of row segments
  int bound[6];      // bound[s] .. bound[s+1]
  int item_base[6];  // first item index of segment s (launch order)
  int item_cnt[6];
  int reversed[6];   // the segment's items run from its last rows back (heaviest first under a one-sided band)
};

// transposed = 1 builds the KEY-MAJOR plan of the backward pass: rows are keys, chunks are query ranges, and the vote
// evaluates mask_allowed(mode, query = column, key = row).
__global__ void plan_band_kernel(int mode, int m0, int m1, int m2, int S, int n_chunks_total, BandSegs segs,
                                 int transposed, int* __restrict__ counts, int4* __restrict__ items,
                                 int2* __restrict__ chunks) {
  const int item = blockIdx.x;
  int seg = 0;
  for (int s = 0; s < segs.n; ++s)
    if (item >= segs.item_base[s] && item < segs.item_base[s] + segs.item_cnt[s]) seg = s;
  const int k = item - segs.item_base[seg];
  const int q_row0 = segs.bound[seg] + (segs.reversed[seg] ? segs.item_cnt[seg] - 1 - k : k) * kItemRows;
  const int nrows = min(kItemRows, segs.bound[seg + 1] - q_row0);
  int q = q_row0 + threadIdx.x;
  const bool row_live = static_cast<int>(threadIdx.x) < nrows;
  if (mode == MASK_BLOCK_CAUSAL && !transposed) {  // the row's block end, once: then the local band, as the kernel does
    q = block_last(q, m1);
    mode = MASK_LOCAL;
    m1 = m2 - 1;
    m2 = 0;
  }
  int2* out = chunks + static_cast<size_t>(item) * n_chunks_total;
  int n = 0;
  for (int c = 0; c < n_chunks_total; ++c) {
    const int kv0 = c * kChunkCols;
    const int valid = min(kChunkCols, S - kv0);
    bool any = false, all = true;
    if (row_live) {
      for (int i = 0; i < valid; ++i) {
        const bool a = transposed ? mask_allowed(mode, kv0 + i, q, m0, m1, m2) : mask_allowed(mode, q, kv0 + i, m0, m1, m2);
        any |= a;
        all &= a;
      }
    }
    const int block_any = __syncthreads_or(any ? 1 : 0);
    const int block_all = __syncthreads_and((all || !row_live) ? 1 : 0);
    if (block_any) {
      if (threadIdx.x == 0) out[n] = make_int2(kv0, chunk_meta(valid, !block_all));
      ++n;
    }
  }
  if (threadIdx.x == 0) {
    put_item(items + 2 * item, q_row0, nrows, static_cast<int>(static_cast<size_t>(item) * n_chunks_total), n);
    if (item == 0) counts[0] = gridDim.x;
  }
}

// row-region boundaries of each mask family, and the launch order of the segments.  Key-major (transposed): the
// HunyuanVideo regions are the same; the Wan and local sink keys (kv < m0) and the CogVideoX first columns (kv < m0)
// are seen by every query and form the heavy first segment.  A one-sided local band (left != right) makes list length
// grow along the rows: query-major with left > right the last rows see the most keys, key-major with right > left the
// last keys are reached by the most queries, and that segment's items are then issued from its end (LPT).
// The block-causal mask segments as its local band (sink, W - 1, 0): its query-major items run from the last rows back
// when W > 1 (an unbounded window gives the last blocks the longest lists), key-major the sink keys come first.
static BandSegs band_segments(int mode, int m0, int m1, int m2, int S, bool transposed = false) {
  if (mode == MASK_BLOCK_CAUSAL) {
    mode = MASK_LOCAL;
    m1 = m2 - 1;
    m2 = 0;
  }
  int cuts[4], nc = 0;
  auto add = [&](int c) {
    if (c > 0 && c < S && (nc == 0 || cuts[nc - 1] < c)) cuts[nc++] = c;
  };
  if (mode == MASK_HY) {
    add(m0);  // end of video
    add(m1);  // end of real prompt
  } else if (mode == MASK_COG) {
    add(transposed ? m0 : m1);  // end of the first columns (key-major) / of the text prefix
  } else if ((mode == MASK_WAN || mode == MASK_LOCAL) && transposed) {
    add(m0);  // end of the sink keys
  }
  BandSegs sg{};
  sg.n = nc + 1;
  sg.bound[0] = 0;
  for (int i = 0; i < nc; ++i) sg.bound[i + 1] = cuts[i];
  sg.bound[sg.n] = S;
  for (int s = 0; s < sg.n; ++s) sg.item_cnt[s] = (sg.bound[s + 1] - sg.bound[s] + kItemRows - 1) / kItemRows;
  int base = 0;
  if (mode == MASK_HY) {  // text segments (heavy: they see every column) first
    for (int s = sg.n - 1; s >= 0; --s) {
      sg.item_base[s] = base;
      base += sg.item_cnt[s];
    }
  } else {
    for (int s = 0; s < sg.n; ++s) {
      sg.item_base[s] = base;
      base += sg.item_cnt[s];
    }
  }
  if (mode == MASK_LOCAL && (transposed ? m2 > m1 : m1 > m2)) sg.reversed[sg.n - 1] = 1;  // the band, after any sinks
  return sg;
}
static int band_total_items(const BandSegs& sg) {
  int t = 0;
  for (int s = 0; s < sg.n; ++s) t += sg.item_cnt[s];
  return t;
}

// =============================================================================================
// Plan: local mask inside packed variable-length segments (svgb_attn_plan_local_varlen[_t]).  Count, scan and fill:
//   seg_bounds_kernel  one CTA: the plan's copy of the bounds (clamped, monotone), per segment its items and chunk
//                      slots, their exclusive scans and the item count
//   seg_lists_kernel   one warp per item: its rows, and its chunk list, classified from the band's interval form
//                      (seg_chunk_kind) and compacted with a ballot, and its two stream descriptors
// Items launch in row order (segments in turn, first rows first).  Longest-list-first (LPT) was measured against it
// (tools/varlen_local_perf.py --order) and came within 1 % either way: the grid walks every head's items before the next
// head's, so many heads make many waves and only the last head's tail could gain.
// Item rows are cut in 256 from the start of their segment; key-major, the sink keys of a segment are items of their
// own.  An item's list has one slot per chunk of its segment, so the chunk storage is the sum over segments of
// items x chunks (svgb_attn_plan_local_varlen_bytes bounds it).
// =============================================================================================
constexpr int kSegThreads = 1024;

// in-place scan of a[0..n) by one CTA of kSegThreads threads, inclusive running maximum (kMax) or exclusive sum:
// contiguous slices per thread, a warp scan of the slice totals, a serial pass over the 32 warp totals
template <bool kMax>
__device__ void seg_block_scan(int* a, int n, int* wtot) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int per = (n + kSegThreads - 1) / kSegThreads;
  const int j0 = min(n, static_cast<int>(threadIdx.x) * per), j1 = min(n, j0 + per);
  auto op = [](int x, int y) { return kMax ? max(x, y) : x + y; };
  const int id = kMax ? INT_MIN : 0;
  int acc = id;
  for (int j = j0; j < j1; ++j) acc = op(acc, a[j]);
  int incl = acc;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int x = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl = op(incl, x);
  }
  if (lane == 31) wtot[warp] = incl;
  __syncthreads();
  int run = id;
  for (int w = 0; w < warp; ++w) run = op(run, wtot[w]);
  const int lane_prev = __shfl_up_sync(0xffffffffu, incl, 1);
  if (lane > 0) run = op(run, lane_prev);
  for (int j = j0; j < j1; ++j) {
    const int x = a[j];
    a[j] = kMax ? op(run, x) : run;
    run = op(run, x);
  }
  __syncthreads();
}

// seg: {nseg, cq[0..nseg], ck[0..nseg]}; base: {item base [nseg + 1], chunk base [nseg + 1]} (exclusive scans, last =
// total)
__global__ void __launch_bounds__(kSegThreads)
seg_bounds_kernel(const int* __restrict__ cu_q, const int* __restrict__ cu_k, int nseg, int Sq, int Skv, int sink,
                  int transposed, int* __restrict__ seg, int* __restrict__ base, int* __restrict__ counts) {
  __shared__ int wtot[32];
  if (threadIdx.x == 0) seg[0] = nseg;
  int* segs = seg + 1;
  for (int i = threadIdx.x; i <= nseg; i += kSegThreads) {
    segs[i] = i == 0 ? 0 : i == nseg ? Sq : min(max(cu_q[i], 0), Sq);
    segs[nseg + 1 + i] = i == 0 ? 0 : i == nseg ? Skv : min(max(cu_k[i], 0), Skv);
  }
  __syncthreads();
  seg_block_scan<true>(segs, nseg + 1, wtot);
  seg_block_scan<true>(segs + nseg + 1, nseg + 1, wtot);
  int* ib = base;
  int* cb = base + nseg + 1;
  const int* rb = segs + (transposed ? nseg + 1 : 0);  // rows of the items: queries, or keys (key-major)
  const int* colb = segs + (transposed ? 0 : nseg + 1);
  for (int i = threadIdx.x; i <= nseg; i += kSegThreads) {
    int items = 0, per = 0;
    if (i < nseg) {
      const int rows = rb[i + 1] - rb[i], cols = colb[i + 1] - colb[i];
      const int s = transposed ? min(sink, rows) : 0;
      items = (s + kItemRows - 1) / kItemRows + (rows - s + kItemRows - 1) / kItemRows;
      per = (cols + kChunkCols - 1) / kChunkCols;
    }
    ib[i] = items;
    cb[i] = items * per;
  }
  __syncthreads();
  seg_block_scan<false>(ib, nseg + 1, wtot);  // entry nseg is 0, so it receives the total
  seg_block_scan<false>(cb, nseg + 1, wtot);
  if (threadIdx.x == 0) counts[0] = ib[nseg];
}

// One warp per item it < counts[0]: its chunk list and its two stream descriptors, items[2 it], items[2 it + 1].
__global__ void __launch_bounds__(256)
seg_lists_kernel(const int* __restrict__ seg, const int* __restrict__ base, const int* __restrict__ counts, int nseg,
                 int sink, int left, int right, int block, int transposed, int2* __restrict__ chunks,
                 int4* __restrict__ items) {
  const int* segs = seg + 1;
  const int lane = threadIdx.x & 31;
  const int it = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (it >= counts[0]) return;
  const int* ib = base;
  const int* cb = base + nseg + 1;
  int si = 0, hi = nseg - 1;  // the last segment whose first item is at or before `it` (empty ones have no items)
  while (si < hi) {
    const int mid = (si + hi + 1) >> 1;
    if (ib[mid] <= it) si = mid;
    else hi = mid - 1;
  }
  const int k = it - ib[si];
  const int* rb = segs + (transposed ? nseg + 1 : 0);
  const int* colb = segs + (transposed ? 0 : nseg + 1);
  const int rs = rb[si], re = rb[si + 1], cs = colb[si], ce = colb[si + 1];
  const int s = transposed ? min(sink, re - rs) : 0;  // key-major: the sink keys end an item run of their own
  const int ns = (s + kItemRows - 1) / kItemRows;
  const int r0 = k < ns ? rs + k * kItemRows : rs + s + (k - ns) * kItemRows;
  const int nr = min(kItemRows, (k < ns ? rs + s : re) - r0);
  const int per = (ce - cs + kChunkCols - 1) / kChunkCols;
  const int list = cb[si] + k * per;
  const SegOrigin o = seg_origin(seg, r0, transposed != 0, sink);
  // block-causal (block = m1 != 0, left = W - 1, right = 0), query-major: the item's first and last rows rounded to their
  // block ends inside the segment, where the mask is the local band; rounding is monotone, so rows a0 .. a1 give the
  // chunk kinds of the item's rows exactly.  Key-major: the interval form of seg_block_chunk_kind_t
  int a0 = r0, a1 = r0 + nr - 1;
  if (block && !transposed) {
    a0 = seg_block_last(a0 - o.shift, o.key0, block) + o.shift;
    a1 = seg_block_last(a1 - o.shift, o.key0, block) + o.shift;
  }
  int n = 0;
  for (int j0 = 0; j0 < per; j0 += 32) {
    const int j = j0 + lane;
    const int c0 = cs + j * kChunkCols, valid = min(kChunkCols, ce - c0);
    int kind = 0;
    if (j < per)
      kind = block && transposed ? seg_block_chunk_kind_t(r0, r0 + nr - 1, c0, c0 + valid - 1, o, block, left + 1)
                                 : seg_chunk_kind(transposed != 0, a0, a1, c0, c0 + valid - 1, o, left, right);
    const unsigned m = __ballot_sync(0xffffffffu, kind != 0);
    if (kind != 0) chunks[list + n + __popc(m & ((1u << lane) - 1u))] = make_int2(c0, chunk_meta(valid, kind == 2));
    n += __popc(m);
  }
  if (lane == 0) put_item(items + 2 * it, r0, nr, list, n);
}

// =============================================================================================
// density_calculation (svg/kmeans_utils.py:13-31)
// =============================================================================================
__global__ void density_kernel(const uint8_t* __restrict__ map, const int* __restrict__ row_sz,
                               const int* __restrict__ col_sz, int QC, int KC,
                               float* __restrict__ density) {
  const int bh = blockIdx.x;
  __shared__ unsigned long long s_num[32], s_den[32];
  unsigned long long num = 0, den = 0;
  for (int idx = threadIdx.x; idx < QC * KC; idx += blockDim.x) {
    const int i = idx / KC, j = idx - i * KC;
    const unsigned long long a =
        static_cast<unsigned long long>(row_sz[static_cast<size_t>(bh) * QC + i]) *
        static_cast<unsigned long long>(col_sz[static_cast<size_t>(bh) * KC + j]);
    den += a;
    if (map[(static_cast<size_t>(bh) * QC + i) * KC + j]) num += a;
  }
  for (int o = 16; o > 0; o >>= 1) {
    num += __shfl_xor_sync(0xffffffffu, num, o);
    den += __shfl_xor_sync(0xffffffffu, den, o);
  }
  if ((threadIdx.x & 31) == 0) {
    s_num[threadIdx.x >> 5] = num;
    s_den[threadIdx.x >> 5] = den;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    num = den = 0;
    for (int w = 0; w < (blockDim.x + 31) / 32; ++w) {
      num += s_num[w];
      den += s_den[w];
    }
    density[bh] = static_cast<float>(static_cast<double>(num) / static_cast<double>(den));
  }
}

// =============================================================================================
// Merge of a split KV-cache forward (svgb_attn_fwd_kvcache_split): one warp per (query row, query head), D / 32 columns
// per lane.  Over the splits s = 0 .. n-1 in order: m = max lse_s, w_s = exp(lse_s - m) (0 for lse_s = -inf), o = sum w_s
// o_s / sum w_s and lse = m + log sum w_s; every split -inf gives o = 0, lse = -inf.  With one live split w = 1, so o and
// lse are that split's bits.  o_part [n, R, Hq, D] and lse_part [n, Hq, R] fp32; o 16-bit at its strides, lse [Hq, R].
// =============================================================================================
template <int D, bool BF16>
__global__ void __launch_bounds__(256)
kv_split_merge_kernel(const float* __restrict__ o_part, const float* __restrict__ lse_part, int nsplit, int R, int Hq,
                      uint16_t* __restrict__ o, long long o_row_stride, long long o_head_stride, float* __restrict__ lse) {
  constexpr int kPer = D / 32;
  const long long w = blockIdx.x * 8ll + (threadIdx.x >> 5);
  if (w >= static_cast<long long>(R) * Hq) return;
  const int lane = threadIdx.x & 31;
  const int r = static_cast<int>(w / Hq), h = static_cast<int>(w - static_cast<long long>(r) * Hq);
  const size_t split_o = static_cast<size_t>(R) * Hq * D, split_l = static_cast<size_t>(Hq) * R;
  const float* lp = lse_part + static_cast<size_t>(h) * R + r;
  const float* op = o_part + static_cast<size_t>(w) * D + lane * kPer;
  float m = -INFINITY;
  for (int s = 0; s < nsplit; ++s) m = fmaxf(m, __ldg(lp + s * split_l));
  float acc[kPer], den = 0.f;
#pragma unroll
  for (int i = 0; i < kPer; ++i) acc[i] = 0.f;
  for (int s = 0; s < nsplit; ++s) {
    const float l = __ldg(lp + s * split_l);
    if (l == -INFINITY) continue;  // weight 0: the split saw no key of this row
    const float ws = expf(l - m);
    float x[kPer];
    if constexpr (kPer == 4) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(op + s * split_o));
      x[0] = v.x, x[1] = v.y, x[2] = v.z, x[3] = v.w;
    } else {
      const float2 v = __ldg(reinterpret_cast<const float2*>(op + s * split_o));
      x[0] = v.x, x[1] = v.y;
    }
#pragma unroll
    for (int i = 0; i < kPer; ++i) acc[i] = fmaf(ws, x[i], acc[i]);
    den += ws;
  }
  const float inv = den > 0.f ? 1.f / den : 0.f;
  uint32_t packed[kPer / 2];
#pragma unroll
  for (int i = 0; i < kPer / 2; ++i) packed[i] = pack2<BF16>(acc[2 * i] * inv, acc[2 * i + 1] * inv);
  uint16_t* dst = o + r * o_row_stride + h * o_head_stride + lane * kPer;
  if constexpr (kPer == 4) *reinterpret_cast<uint2*>(dst) = make_uint2(packed[0], packed[1]);
  else *reinterpret_cast<uint32_t*>(dst) = packed[0];
  if (lse && lane == 0) lse[static_cast<size_t>(h) * R + r] = den > 0.f ? m + logf(den) : -INFINITY;
}

// =============================================================================================
// Tile self-test: the exact descriptor paths of the attention kernel on one 128x128xD tile.
// =============================================================================================
template <int D, bool BF16>
__global__ void __launch_bounds__(256, 1)
selftest_tile_kernel(const __grid_constant__ CUtensorMap qmap, const __grid_constant__ CUtensorMap kmap,
                     const __grid_constant__ CUtensorMap vmap, float* __restrict__ s_out,
                     float* __restrict__ o_out, float p_scale) {
  constexpr int DT = BF16 ? DT_BF16 : DT_F16;
  using Cfg = AttnCfg<D, DT>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_al = smem_raw + (smem_base - smem_u32(smem_raw));
  const uint32_t sQ = smem_base, sK = sQ + Cfg::kTileBytes, sV = sK + Cfg::kTileBytes;
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem_al + 3 * Cfg::kTileBytes);
  const int wg = threadIdx.x >> 7, lane = threadIdx.x & 31, wq = (threadIdx.x >> 5) & 3;
  if (threadIdx.x == 0) {
    mbar_init(smem_u32(bar), 1);
    mbar_fence_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_expect_tx(smem_u32(bar), 3 * Cfg::kTileBytes);
    for (int h = 0; h < Cfg::kHalves; ++h) {
      tma_load_3d(sQ + h * Cfg::kPanelBytes, &qmap, smem_u32(bar), h * 64, 0, 0);
      tma_load_3d(sK + h * Cfg::kPanelBytes, &kmap, smem_u32(bar), h * 64, 0, 0);
      tma_load_3d(sV + h * Cfg::kPanelBytes, &vmap, smem_u32(bar), h * 64, 0, 0);
    }
  }
  mbar_wait(smem_u32(bar), 0, 20);
  float s[64];
  attn_qk_issue<D, DT>(s, sQ + 64 * wg * 128, sK);
  attn_wait<0>(s);
  // S -> global, P = 16-bit(S * p_scale), O = P V
  const int row0 = 64 * wg + 16 * wq + (lane >> 2), col0 = 2 * (lane & 3);
#pragma unroll
  for (int jj = 0; jj < 16; ++jj)
#pragma unroll
    for (int v1 = 0; v1 < 2; ++v1)
#pragma unroll
      for (int v0 = 0; v0 < 2; ++v0) {
        float& x = s[4 * jj + 2 * v1 + v0];
        s_out[(row0 + 8 * v1) * 128 + 8 * jj + col0 + v0] = x;
        x *= p_scale;
      }
  float o[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) o[i] = 0.f;
  uint32_t pa[8][4];
  attn_pack_p<BF16>(pa, s);
  attn_pv_issue<D, BF16>(o, pa, sV);
  attn_wait<0>(o);
#pragma unroll
  for (int jj = 0; jj < D / 8; ++jj)
#pragma unroll
    for (int v1 = 0; v1 < 2; ++v1)
#pragma unroll
      for (int v0 = 0; v0 < 2; ++v0) o_out[(row0 + 8 * v1) * D + 8 * jj + col0 + v0] = o[4 * jj + 2 * v1 + v0];
}

// ksm, vsm: the row-scale maps of DT_E4M3_ROWS, which has no row-gather instantiation
template <int D, int DT>
static int launch_attn(const CUtensorMap& qm, const CUtensorMap& km, const CUtensorMap& vm,
                       const AttnArgs& args, bool gather, dim3 grid, cudaStream_t stream,
                       const CUtensorMap& ksm = CUtensorMap{}, const CUtensorMap& vsm = CUtensorMap{}) {
  using Cfg = AttnCfg<D, DT>;
  auto kern = attn_fwd_kernel<D, DT, false>;
  if constexpr (DT != DT_E4M3_ROWS) {
    if (gather) kern = attn_fwd_kernel<D, DT, true>;
  }
  SVGB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
  kern<<<grid, Cfg::kThreads, Cfg::kSmemBytes, stream>>>(qm, km, vm, args, ksm, vsm);
  SVGB_LAUNCH_OK();
  return 0;
}

template <int D, bool BF16>
static int launch_selftest(const CUtensorMap& qm, const CUtensorMap& km, const CUtensorMap& vm,
                           float* s_out, float* o_out, float p_scale, cudaStream_t stream) {
  using Cfg = AttnCfg<D, BF16 ? DT_BF16 : DT_F16>;
  auto kern = selftest_tile_kernel<D, BF16>;
  const int smem = 1024 + 3 * Cfg::kTileBytes + 256;
  SVGB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  kern<<<1, 256, smem, stream>>>(qm, km, vm, s_out, o_out, p_scale);
  SVGB_LAUNCH_OK();
  return 0;
}

int attn_fwd_impl(const void* q, Strides qs, int Sq, const void* k, Strides ks, const void* v, Strides vs, int Skv,
                  int dtype, int B, int BH, int D, const AttnArgs& a, bool gather, int grid_x, cudaStream_t st) {
  SVGB_REQUIRE(D == 64 || D == 128, "head_dim %d unsupported (64 or 128)", D);
  SVGB_REQUIRE(dtype == SVGB_BF16 || dtype == SVGB_F16 || dtype == SVGB_E4M3, "dtype %d unsupported", dtype);
  CUtensorMap qm, km, vm;
  const int Hq = BH / B, Hkv = Hq / a.kv_group;  // BH counts the query heads
  if (encode_tmap_bhsd(&qm, q, dtype, B, Hq, Sq, D, qs)) return -1;
  if (encode_tmap_bhsd(&km, k, dtype, B, Hkv, Skv, D, ks)) return -1;
  if (encode_tmap_bhsd(&vm, v, dtype, B, Hkv, Skv, D, vs)) return -1;
  AttnArgs args = a;
  args.Hq = Hq;
  dim3 grid(grid_x, BH);
  if (dtype == SVGB_E4M3) {
    SVGB_REQUIRE(D == 128, "the e4m3 path needs head_dim 128 (got %d): 64-byte e4m3 rows have no 128-byte swizzle", D);
    if (a.scale_block_rows > 0) {  // per-row scales: the cache is Skv / block_rows blocks (svgb_attn_fwd_kvcache_e4m3_rows)
      CUtensorMap ksm, vsm;
      const int nblk = Skv / a.scale_block_rows;
      if (encode_tmap_scale_rows(&ksm, a.k_scale, nblk, Hkv, a.scale_block_rows)) return -1;
      if (encode_tmap_scale_rows(&vsm, a.v_scale, nblk, Hkv, a.scale_block_rows)) return -1;
      return launch_attn<128, DT_E4M3_ROWS>(qm, km, vm, args, false, grid, st, ksm, vsm);
    }
    return launch_attn<128, DT_E4M3>(qm, km, vm, args, gather, grid, st);
  }
  if (D == 128) {
    return dtype == SVGB_BF16 ? launch_attn<128, DT_BF16>(qm, km, vm, args, gather, grid, st)
                              : launch_attn<128, DT_F16>(qm, km, vm, args, gather, grid, st);
  }
  return dtype == SVGB_BF16 ? launch_attn<64, DT_BF16>(qm, km, vm, args, gather, grid, st)
                            : launch_attn<64, DT_F16>(qm, km, vm, args, gather, grid, st);
}

// a chunk list covers the key side (Skv columns), the items the query side (Sq rows)
static int varblock_chunk_cap(int Skv, int KC) { return Skv / kChunkCols + (KC + 1) / 2 + 2; }
static int varblock_max_items(int Sq, int QC) { return Sq / kItemRows + QC + 1; }

static int plan_varblock_bytes(int BH, int Sq, int Skv, int QC, int KC, size_t* bytes) {
  SVGB_REQUIRE(BH > 0 && Sq > 0 && Skv > 0 && QC > 0 && KC > 0 && bytes, "bad arguments");
  const size_t counts = align_up(sizeof(int) * BH, 256);
  const size_t items = align_up(2 * sizeof(int4) * BH * varblock_max_items(Sq, QC), 256);
  const size_t chunks = align_up(sizeof(int2) * static_cast<size_t>(BH) * QC * varblock_chunk_cap(Skv, KC), 256);
  const size_t lens = align_up(sizeof(int) * static_cast<size_t>(BH) * QC, 256);  // per q-block list length
  *bytes = counts + items + chunks + lens;
  return 0;
}

// rect: the plan of svgb_attn_plan_varblock_kv, which records Skv in m0 (0 leaves Skv = S, svgb200.h)
static int plan_varblock_impl(const uint8_t* map, const int32_t* row_sz, const int32_t* col_sz, int BH, int Sq,
                              int Skv, int QC, int KC, void* plan_ws, size_t ws_bytes, svgb_plan* plan, void* stream,
                              bool gather, bool rect) {
  size_t need = 0;
  if (plan_varblock_bytes(BH, Sq, Skv, QC, KC, &need)) return -1;
  SVGB_REQUIRE(map && row_sz && col_sz && plan_ws && plan, "null pointer");
  SVGB_REQUIRE(ws_bytes >= need, "plan workspace too small: %zu < %zu", ws_bytes, need);
  SVGB_REQUIRE(static_cast<size_t>(BH) * QC * varblock_chunk_cap(Skv, KC) < (1ull << 31),
               "plan too large for 32-bit chunk offsets");
  const int max_items = varblock_max_items(Sq, QC);
  const int cap = varblock_chunk_cap(Skv, KC);
  const int64_t items_off = align_up(sizeof(int) * BH, 256);
  write_plan(plan, gather ? SVGB_PLAN_GATHER : SVGB_PLAN_VARBLOCK, BH, Sq, max_items, max_items, MASK_NONE,
             rect ? Skv : 0, 0, 0, 0, items_off, items_off + align_up(2 * sizeof(int4) * BH * max_items, 256), need);
  char* ws = static_cast<char*>(plan_ws);
  // per q-block list lengths: scratch of the two plan kernels, after the lists
  const size_t lens_off = plan->chunks_off + align_up(sizeof(int2) * static_cast<size_t>(BH) * QC * cap, 256);
  int* nch_of = reinterpret_cast<int*>(ws + lens_off);
  const size_t smem1 = sizeof(int) * (KC + 1);
  const size_t smem2 = sizeof(int) * (2 * (QC + 1) + 2 * QC);
  SVGB_REQUIRE(smem1 <= 48 * 1024 && smem2 <= 48 * 1024, "QC/KC too large for the plan kernels (%zu / %zu B smem)", smem1, smem2);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  plan_lists_kernel<<<dim3((QC + kPlanWarps - 1) / kPlanWarps, BH), kPlanWarps * 32, smem1, st>>>(map, row_sz, col_sz, QC, KC, cap, gather ? 1 : 0,
                                                                 reinterpret_cast<int2*>(ws + plan->chunks_off), nch_of);
  SVGB_LAUNCH_OK();
  plan_items_kernel<<<BH, 256, smem2, st>>>(row_sz, nch_of, QC, max_items, cap, gather ? 1 : 0,
                                            reinterpret_cast<int*>(ws + plan->counts_off),
                                            reinterpret_cast<int4*>(ws + plan->items_off));
  SVGB_LAUNCH_OK();
  return 0;
}

// Workspace of a segment plan (one layout for both directions), 16-byte aligned pieces:
//   counts (16 B) | bounds {nseg, 2 (nseg + 1)} | bases 2 (nseg + 1) | items 2 int4 [items] | chunks [C]
// items: every segment adds at most one partial item (key-major two: its sink keys end an item), so
//   I = min(R, (R + 510 nseg) / 256) for R = Sq (query-major) and Skv (key-major) covers both.
// chunks: sum over segments of items x ceil(cols / 128) <= sum (rows + 510)(cols + 127) / 32768 with sum rows x cols <=
//   Sq Skv, and never more than I x ceil(max(Sq, Skv) / 128).
struct SegLayout {
  int max_items;
  long long max_chunks;
  size_t segs_off, base_off, items_off, chunks_off, bytes;
};
static SegLayout seg_layout(int nseg, int Sq, int Skv) {
  SegLayout L;
  const long long n = nseg, q = Sq, k = Skv, mx = q > k ? q : k;
  const long long iq = std::min(q, (q + 510 * n) / 256), ik = std::min(k, (k + 510 * n) / 256);
  const long long items = std::max(iq, ik);
  const long long sum_bound = (q * k + 510 * (q + k) + 510 * 127 * n) / 32768;
  L.max_items = static_cast<int>(std::min<long long>(items, INT_MAX));
  L.max_chunks = std::min(items * ((mx + kChunkCols - 1) / kChunkCols), sum_bound);
  L.segs_off = SVGB_PLAN_SEG_BOUNDS_OFF;
  L.base_off = L.segs_off + align_up(sizeof(int) * (2 * n + 3), 16);
  L.items_off = L.base_off + align_up(sizeof(int) * 2 * (n + 1), 16);
  L.chunks_off = L.items_off + 2 * sizeof(int4) * items;
  L.bytes = L.chunks_off + sizeof(int2) * L.max_chunks;
  return L;
}

static int plan_local_varlen_bytes(int nseg, int Sq, int Skv, size_t* bytes) {
  SVGB_REQUIRE(nseg > 0 && Sq > 0 && Skv > 0 && bytes, "bad arguments (nseg=%d, Sq=%d, Skv=%d)", nseg, Sq, Skv);
  *bytes = seg_layout(nseg, Sq, Skv).bytes;
  return 0;
}

// block = 0: MASK_LOCAL(sink, left, right); block = m1 of MASK_BLOCK_CAUSAL (checked by the caller): the block rule with
// the window W = left + 1 and right = 0
static int plan_local_varlen_impl(const int32_t* cu_q, const int32_t* cu_k, int nseg, int Sq, int Skv, int sink,
                                  int left, int right, void* plan_ws, size_t ws_bytes, svgb_plan* plan, void* stream,
                                  bool transposed, int block = 0) {
  size_t need = 0;
  if (plan_local_varlen_bytes(nseg, Sq, Skv, &need)) return -1;
  SVGB_REQUIRE(cu_q && cu_k && plan_ws && plan, "null pointer");
  SVGB_REQUIRE(ws_bytes >= need, "plan workspace too small: %zu < %zu", ws_bytes, need);
  SVGB_REQUIRE(sink >= 0 && left >= 0 && right >= 0,
               "local varlen mask: sink (%d), left (%d) and right (%d) must be >= 0", sink, left, right);
  const SegLayout L = seg_layout(nseg, Sq, Skv);
  SVGB_REQUIRE(L.max_chunks < (1ll << 31) && nseg < (1 << 29), "plan too large for 32-bit chunk offsets");
  const int rows = transposed ? Skv : Sq, cols = transposed ? Sq : Skv;
  const int max_items = static_cast<int>(std::min<long long>(rows, (rows + 510ll * nseg) / 256));
  // a segment plan serves every head: BH holds its key/value length (svgb200.h)
  write_plan(plan, transposed ? SVGB_PLAN_SEG_T : SVGB_PLAN_SEG, cols, rows, max_items, 0,
             block ? MASK_BLOCK_CAUSAL : MASK_LOCAL, sink, block ? block : left, block ? left + 1 : right, 0,
             static_cast<int64_t>(L.items_off), static_cast<int64_t>(L.chunks_off), static_cast<int64_t>(need));
  char* ws = static_cast<char*>(plan_ws);
  int* counts = reinterpret_cast<int*>(ws);
  int* segs = reinterpret_cast<int*>(ws + L.segs_off);
  int* base = reinterpret_cast<int*>(ws + L.base_off);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  seg_bounds_kernel<<<1, kSegThreads, 0, st>>>(cu_q, cu_k, nseg, Sq, Skv, sink, transposed ? 1 : 0, segs, base, counts);
  SVGB_LAUNCH_OK();
  seg_lists_kernel<<<(max_items + 7) / 8, 256, 0, st>>>(segs, base, counts, nseg, sink, left, right, block,
                                                        transposed ? 1 : 0, reinterpret_cast<int2*>(ws + L.chunks_off),
                                                        reinterpret_cast<int4*>(ws + L.items_off));
  SVGB_LAUNCH_OK();
  return 0;
}

// One forward call, as every entry hands it over: q / o over Sq rows and Hq heads in B batch elements, k / v over Skv
// rows and Hkv heads, each tensor with its own strides.  A split plan's call has B streams of Sq rows each, run as
// B * Sq packed rows; a KV-cache entry's Skv is its num_blocks x block_rows cache rows.
struct AttnFwdCall {
  const void *q, *k, *v;
  const float *q_scale, *k_scale, *v_scale;
  void* o;
  float* lse;
  const int32_t *q_rows, *kv_rows, *o_rows;
  int dtype, row_scales;  // row_scales: e4m3 with per-row k / v scales beside the cache rows
  int B, Hq, Hkv, Sq, Skv, D;
  Strides qs, ks, vs, os;
  float sm_scale;
  const svgb_plan* plan;
  const void* plan_ws;
  int num_blocks, block_rows;  // KV-cache entries: the cache geometry (0: none)
  void* ws;                    // split plans: the fp32 partials
  size_t ws_bytes;
  void* stream;
};

// input formats
enum { FMT_16BIT = 1, FMT_E4M3 = 2, FMT_E4M3_ROWS = 4 };
// addressing: one stride pair for q, k, v and one for o; a q and a k / v pair; or per-tensor strides
enum { ADDR_FLAT, ADDR_FLAT_KV, ADDR_STRIDED };
// bit k: plan kind k; bit 0: kinds outside 1 .. 8, which svgb_attn_fwd runs as variable-block plans
constexpr unsigned kind_bit(int kind) { return kind >= 1 && kind <= 8 ? 1u << kind : 1u; }
constexpr unsigned K_VARBLOCK = 1u << SVGB_PLAN_VARBLOCK, K_BAND = 1u << SVGB_PLAN_BAND, K_GATHER = 1u << SVGB_PLAN_GATHER,
                   K_SEG = 1u << SVGB_PLAN_SEG, K_KVCACHE = 1u << SVGB_PLAN_KVCACHE,
                   K_SPLIT = 1u << SVGB_PLAN_KVCACHE_SPLIT;

// what one forward entry accepts
struct AttnFwdRule {
  const char* who;
  unsigned kinds;
  const char* kinds_text;  // the accepted kinds, for the refusal
  unsigned formats;
  int addr;
  bool row_vectors;  // q_rows / kv_rows / o_rows
  bool split;        // split KV-cache plans, with a partials workspace
};
enum { FWD, FWD_KV, FWD_GQA, FWD_STRIDED, FWD_STRIDED_E4M3, FWD_KVCACHE_E4M3_ROWS, FWD_KVCACHE_SPLIT };
static constexpr AttnFwdRule kFwdRules[] = {
    {"svgb_attn_fwd", K_VARBLOCK | K_BAND | K_GATHER | K_SEG | K_KVCACHE | 1u,
     "variable-block, band, gather, segment or KV-cache plans", FMT_16BIT | FMT_E4M3, ADDR_FLAT, true, false},
    {"svgb_attn_fwd_kv", K_VARBLOCK | K_SEG, "segment plans and variable-block plans", FMT_16BIT, ADDR_FLAT_KV, false,
     false},
    {"svgb_attn_fwd_gqa", K_VARBLOCK | K_BAND | K_SEG | K_KVCACHE, "variable-block, band, segment or KV-cache plans",
     FMT_16BIT, ADDR_FLAT_KV, false, false},
    {"svgb_attn_fwd_strided", K_VARBLOCK | K_BAND | K_SEG | K_KVCACHE, "variable-block, band, segment or KV-cache plans",
     FMT_16BIT, ADDR_STRIDED, false, false},
    {"svgb_attn_fwd_strided_e4m3", K_VARBLOCK | K_BAND | K_KVCACHE, "variable-block, band or KV-cache plans", FMT_E4M3,
     ADDR_STRIDED, false, false},
    {"svgb_attn_fwd_kvcache_e4m3_rows", K_KVCACHE, "KV-cache plans (svgb_attn_plan_kvcache)", FMT_E4M3_ROWS,
     ADDR_STRIDED, false, false},
    {"svgb_attn_fwd_kvcache_split", K_SPLIT, "split KV-cache plans (svgb_attn_plan_kvcache_split)",
     FMT_16BIT | FMT_E4M3 | FMT_E4M3_ROWS, ADDR_STRIDED, false, true},
};

static bool e4m3_strides(Strides s) { return s.b % 16 == 0 && s.h % 16 == 0 && s.r % 16 == 0; }

// items per split of a split plan: recorded by a varlen plan, whose item count depends on lengths only the device holds
static int split_items(const AttnFwdCall& c) {
  return c.plan->varlen_items > 0 ? c.plan->varlen_items : c.B * ((c.Sq + kItemRows - 1) / kItemRows);
}

// Every rule of the forward, in one order, before any device work.
static int attn_fwd_check(const AttnFwdCall& c, const AttnFwdRule& r) {
  const char* who = r.who;
  const svgb_plan* plan = c.plan;
  SVGB_REQUIRE(c.q && c.k && c.v && c.o && plan && c.plan_ws && (!r.split || c.ws), "null pointer");
  const int kind = plan->kind;
  // plan kinds
  const char* hint = kind == SVGB_PLAN_KVCACHE_SPLIT
                         ? "; a split KV-cache plan (svgb_attn_plan_kvcache_split) runs on svgb_attn_fwd_kvcache_split only"
                     : kind == SVGB_PLAN_BAND_T || kind == SVGB_PLAN_SEG_T
                         ? "; a key-major plan (svgb_attn_plan_band_t or svgb_attn_plan_local_varlen_t) is for the "
                           "backward: key-major plans have no GQA, strided or forward path"
                     : kind == SVGB_PLAN_GATHER
                         ? "; gather plans (svgb_attn_plan_varblock_gather) and row vectors run on svgb_attn_fwd only"
                     : kind == SVGB_PLAN_SEG ? "; segment plans (svgb_attn_plan_local_varlen) take bf16 or fp16 inputs"
                                             : "";
  SVGB_REQUIRE(r.kinds & kind_bit(kind), "%s takes %s only (kind %d)%s", who, r.kinds_text, kind, hint);
  // input format: 16-bit, or e4m3 with per-head or per-row scales
  const bool e4m3 = c.dtype == SVGB_E4M3;
  SVGB_REQUIRE(e4m3 || c.dtype == SVGB_BF16 || c.dtype == SVGB_F16, "%s: dtype %d unsupported", who, c.dtype);
  SVGB_REQUIRE(r.formats & (!e4m3 ? FMT_16BIT : c.row_scales ? FMT_E4M3_ROWS : FMT_E4M3),
               "%s takes bf16 or fp16 inputs (dtype %d; e4m3 attention has no path here)", who, c.dtype);
  SVGB_REQUIRE(!e4m3 || (kind != SVGB_PLAN_SEG && kind != SVGB_PLAN_SEG_T),
               "%s: segment plans (svgb_attn_plan_local_varlen) take bf16 or fp16 inputs, not e4m3", who);
  // the flat entry's scales are [BH] by query head: an e4m3 cache, whose scales are by key/value head, is strided
  SVGB_REQUIRE(!e4m3 || r.addr != ADDR_FLAT || kind != SVGB_PLAN_KVCACHE,
               "KV-cache plans (svgb_attn_plan_kvcache) take bf16 or fp16 inputs here; an e4m3 cache takes "
               "svgb_attn_fwd_strided_e4m3");
  if (e4m3) {
    SVGB_REQUIRE(c.D == 128, "%s: the e4m3 path needs head_dim 128 (got %d): 64-byte e4m3 rows have no 128-byte swizzle",
                 who, c.D);
    if (c.row_scales) {
      SVGB_REQUIRE(c.q_scale, "%s needs the three scale tensors: the query row scales q_scale (float [Hq, Sq]), then "
                   "k_scale and v_scale", who);
      if (kv_scale_rows_check(c.k_scale, c.v_scale, c.block_rows, who)) return -1;
    } else {
      SVGB_REQUIRE(c.q_scale && c.k_scale && c.v_scale,
                   "%s needs the three scale vectors q_scale [B*Hq], k_scale and v_scale [B*Hkv]; an e4m3 cache needs "
                   "the three scale tensors", who);
    }
    for (Strides s : {c.qs, c.ks, c.vs})
      SVGB_REQUIRE(e4m3_strides(s),
                   "%s: every e4m3 (batch, head, row) stride must be a multiple of 16 bytes (got %lld, %lld, %lld)", who,
                   s.b, s.h, s.r);
  } else {
    SVGB_REQUIRE(!c.q_scale && !c.k_scale && !c.v_scale && !c.row_scales,
                 "%s: 16-bit inputs (dtype %d) take no scales; scales are for e4m3 inputs", who, c.dtype);
  }
  // row vectors
  const bool kvc = kind == SVGB_PLAN_KVCACHE || kind == SVGB_PLAN_KVCACHE_SPLIT;
  SVGB_REQUIRE(!kvc || (!c.q_rows && !c.kv_rows && !c.o_rows),
               "KV-cache plans (svgb_attn_plan_kvcache) take no row vectors or gathers (q_rows / kv_rows / o_rows)");
  SVGB_REQUIRE(kind != SVGB_PLAN_SEG || (!c.q_rows && !c.kv_rows && !c.o_rows),
               "segment plans (svgb_attn_plan_local_varlen) take no row vectors (q_rows / kv_rows / o_rows)");
  SVGB_REQUIRE(kind == SVGB_PLAN_GATHER || (!c.q_rows && !c.kv_rows),
               "row gathers (q_rows / kv_rows) need a gather plan from svgb_attn_plan_varblock_gather");
  // heads, addressing and the cache
  SVGB_REQUIRE(c.B > 0 && c.Hq > 0 && c.Hkv > 0 && c.Hq % c.Hkv == 0,
               "%s: the query heads Hq=%d must be a multiple of the key/value heads Hkv=%d (B=%d)", who, c.Hq, c.Hkv, c.B);
  SVGB_REQUIRE(c.D == 64 || c.D == 128, "head_dim %d unsupported (64 or 128)", c.D);
  if (r.addr == ADDR_FLAT_KV) {
    for (const void* p : {c.q, c.k, c.v})
      SVGB_REQUIRE((reinterpret_cast<uintptr_t>(p) & 15) == 0, "q, k, v must be 16-byte aligned with strides multiple of 8 elements");
    for (Strides s : {c.qs, c.ks})
      SVGB_REQUIRE(s.r % 8 == 0 && s.h % 8 == 0, "q, k, v must be 16-byte aligned with strides multiple of 8 elements");
  }
  SVGB_REQUIRE((reinterpret_cast<uintptr_t>(c.o) & 15) == 0 && c.os.r % 8 == 0 && c.os.h % 8 == 0 && c.os.b % 8 == 0,
               "output must be 16-byte aligned with strides multiple of 8 elements");
  if (c.block_rows || c.num_blocks)
    SVGB_REQUIRE(c.num_blocks > 0 && c.block_rows > 0 && static_cast<long long>(c.num_blocks) * c.block_rows < (1ll << 31),
                 "%s: bad cache geometry (num_blocks=%d, block_rows=%d)", who, c.num_blocks, c.block_rows);
  // the plan's lengths and heads; a split plan serves B streams of Sq rows as B * Sq packed rows
  int Sq = c.Sq;
  if (r.split) {
    SVGB_REQUIRE(c.Sq > 0 && static_cast<long long>(c.B) * c.Sq == plan->S,
                 "%s: the plan was built for %d query rows, called with B=%d streams of Sq=%d", who, plan->S, c.B, c.Sq);
    Sq = plan->S;
  }
  const int BHkv = (r.split ? 1 : c.B) * c.Hkv;
  SVGB_REQUIRE(kind != SVGB_PLAN_BAND || Sq == c.Skv, "%s: band plans need Sq == Skv (got %d, %d)", who, Sq, c.Skv);
  SVGB_REQUIRE(plan->items_stride == 0 || plan->BH == BHkv,
               "%s: a per-head plan is built over the BHkv=%d key/value heads (plan BH=%d)", who, BHkv, plan->BH);
  SVGB_REQUIRE(plan->S == Sq && plan_kv_len(plan) == c.Skv,
               "plan was built for BH=%d Sq=%d Skv=%d, called with BH=%d Sq=%d Skv=%d", plan->BH, plan->S,
               plan_kv_len(plan), BHkv, Sq, c.Skv);
  if (r.split) {
    const int items = split_items(c);
    SVGB_REQUIRE(plan->max_items > 0 && plan->max_items % items == 0,
                 "%s: the plan's %d items are no whole number of splits of %d items (B=%d, Sq=%d)", who, plan->max_items,
                 items, c.B, c.Sq);
    size_t need = 0;
    if (svgb_attn_fwd_kvcache_split_bytes(plan->max_items / items, Sq, c.Hq, c.D, &need)) return -1;
    SVGB_REQUIRE(c.ws_bytes >= need, "%s: workspace too small: %zu < %zu", who, c.ws_bytes, need);
    SVGB_REQUIRE((reinterpret_cast<uintptr_t>(c.ws) & 15) == 0, "%s: the workspace must be 16-byte aligned", who);
  }
  return 0;
}

// A checked call: one launch, and for a split plan the LSE merge of its fp32 partials.
static int attn_fwd_run(const AttnFwdCall& c) {
  const svgb_plan* plan = c.plan;
  const int kind = plan->kind;
  const bool seg = kind == SVGB_PLAN_SEG, split = kind == SVGB_PLAN_KVCACHE_SPLIT;
  const bool kvc = kind == SVGB_PLAN_KVCACHE || split;
  const int B = split ? 1 : c.B, Sq = split ? plan->S : c.Sq, BH = B * c.Hq;
  const int items = split ? split_items(c) : 0, nsplit = split ? plan->max_items / items : 0;
  // split: o is the fp32 partials o [n, R, Hq, D] (the split as its batch dimension), then lse [n, Hq, R]
  float* o_part = static_cast<float*>(c.ws);
  float* lse_part = split ? o_part + static_cast<size_t>(nsplit) * Sq * c.Hq * c.D : nullptr;
  const Strides os = split ? Strides{static_cast<long long>(Sq) * c.Hq * c.D, c.D, static_cast<long long>(c.Hq) * c.D}
                           : c.os;
  const char* ws = static_cast<const char*>(c.plan_ws);
  AttnArgs a;
  a.items = reinterpret_cast<const int4*>(ws + plan->items_off);
  a.item_count = reinterpret_cast<const int*>(ws + plan->counts_off);
  a.chunks = reinterpret_cast<const int2*>(ws + plan->chunks_off);
  a.items_stride = plan->items_stride;
  a.kv_group = c.Hq / c.Hkv;
  a.o = split ? static_cast<void*>(o_part) : c.o;
  a.o_row_stride = os.r;
  a.o_head_stride = os.h;
  a.o_batch_stride = os.b;
  a.o_rows = c.o_rows;
  a.lse = split ? lse_part : c.lse;
  a.scale_log2 = c.sm_scale * 1.4426950408889634f;
  a.S = Sq;
  if (kind == SVGB_PLAN_BAND || seg || kvc) {  // a variable-block plan's m0 is its Skv, not a mask parameter
    a.mask_mode = plan->mask_mode;
    a.m0 = plan->m0;
    a.m1 = plan->m1;
    a.m2 = plan->m2;
  }
  if (seg || kvc) a.segs = reinterpret_cast<const int*>(ws + SVGB_PLAN_SEG_BOUNDS_OFF);
  a.kv_logical = kvc ? 1 : 0;
  a.q_scale = c.q_scale;
  a.k_scale = c.k_scale;
  a.v_scale = c.v_scale;
  a.q_rows = c.q_rows;
  a.kv_rows = c.kv_rows;
  a.q_ptr = c.q;
  a.k_ptr = c.k;
  a.v_ptr = c.v;
  a.in_row_stride = c.qs.r;  // gather plans: q, k and v share one stride pair (svgb_attn_fwd)
  a.in_head_stride = c.qs.h;
  a.scale_block_rows = c.dtype == SVGB_E4M3 && c.row_scales ? c.block_rows : 0;
  if (split) {
    a.out_f32 = 1;
    a.split_items = items;
    a.o_split_stride = os.b;
  }
  cudaStream_t st = static_cast<cudaStream_t>(c.stream);
  if (attn_fwd_impl(c.q, c.qs, Sq, c.k, c.ks, c.v, c.vs, c.Skv, c.dtype, B, BH, c.D, a, kind == SVGB_PLAN_GATHER,
                    plan->max_items, st))
    return -1;
  if (!split) return 0;
  const bool bf16 = c.dtype != SVGB_F16;  // e4m3 caches give bf16 o
  auto merge = c.D == 128 ? (bf16 ? kv_split_merge_kernel<128, true> : kv_split_merge_kernel<128, false>)
                          : (bf16 ? kv_split_merge_kernel<64, true> : kv_split_merge_kernel<64, false>);
  const long long warps = static_cast<long long>(Sq) * c.Hq;
  merge<<<static_cast<unsigned>((warps + 7) / 8), 256, 0, st>>>(o_part, lse_part, nsplit, Sq, c.Hq,
                                                                 static_cast<uint16_t*>(c.o), c.os.r, c.os.h, c.lse);
  SVGB_LAUNCH_OK();
  return 0;
}

static int attn_fwd(const AttnFwdCall& c, int row) {
  if (attn_fwd_check(c, kFwdRules[row])) return -1;
  return attn_fwd_run(c);
}

}  // namespace svgb

using namespace svgb;

extern "C" {

int svgb_attn_plan_varblock_bytes(int BH, int S, int QC, int KC, size_t* bytes) {
  return plan_varblock_bytes(BH, S, S, QC, KC, bytes);
}

int svgb_attn_plan_varblock(const uint8_t* map, const int32_t* row_sz, const int32_t* col_sz, int BH,
                            int S, int QC, int KC, void* plan_ws, size_t ws_bytes, svgb_plan* plan,
                            void* stream) {
  return plan_varblock_impl(map, row_sz, col_sz, BH, S, S, QC, KC, plan_ws, ws_bytes, plan, stream, false, false);
}

int svgb_attn_plan_varblock_kv_bytes(int BH, int Sq, int Skv, int QC, int KC, size_t* bytes) {
  return plan_varblock_bytes(BH, Sq, Skv, QC, KC, bytes);
}

int svgb_attn_plan_varblock_kv(const uint8_t* map, const int32_t* row_sz, const int32_t* col_sz, int BH, int Sq,
                               int Skv, int QC, int KC, void* plan_ws, size_t ws_bytes, svgb_plan* plan,
                               void* stream) {
  return plan_varblock_impl(map, row_sz, col_sz, BH, Sq, Skv, QC, KC, plan_ws, ws_bytes, plan, stream, false, true);
}

int svgb_attn_plan_varblock_gather(const uint8_t* map, const int32_t* row_sz, const int32_t* col_sz, int BH,
                                   int S, int QC, int KC, void* plan_ws, size_t ws_bytes, svgb_plan* plan,
                                   void* stream) {
  return plan_varblock_impl(map, row_sz, col_sz, BH, S, S, QC, KC, plan_ws, ws_bytes, plan, stream, true, false);
}

int svgb_attn_plan_band_bytes(int S, size_t* bytes) {
  SVGB_REQUIRE(S > 0 && bytes, "bad arguments");
  const size_t n_items = (S + kItemRows - 1) / kItemRows + 4;  // + one partial item per extra row segment
  const size_t n_chunks = (S + kChunkCols - 1) / kChunkCols;
  *bytes = 256 + align_up(2 * sizeof(int4) * n_items, 256) + align_up(sizeof(int2) * n_items * n_chunks, 256);
  return 0;
}

static int plan_band_impl(int mask_mode, int m0, int m1, int m2, int BH, int S, void* plan_ws, size_t ws_bytes,
                          svgb_plan* plan, void* stream, bool transposed) {
  size_t need = 0;
  if (svgb_attn_plan_band_bytes(S, &need)) return -1;
  SVGB_REQUIRE(plan_ws && plan, "null pointer");
  SVGB_REQUIRE(ws_bytes >= need, "plan workspace too small: %zu < %zu", ws_bytes, need);
  SVGB_REQUIRE((mask_mode >= MASK_NONE && mask_mode <= MASK_LOCAL) || mask_mode == MASK_BLOCK_CAUSAL,
               "unknown mask mode %d", mask_mode);
  SVGB_REQUIRE(mask_mode != MASK_LOCAL || (m0 >= 0 && m1 >= 0 && m2 >= 0),
               "local mask: sink (m0 = %d), left (m1 = %d) and right (m2 = %d) must be >= 0", m0, m1, m2);
  if (mask_mode == MASK_BLOCK_CAUSAL &&
      block_causal_check(m0, m1, m2, transposed ? "svgb_attn_plan_band_t" : "svgb_attn_plan_band"))
    return -1;
  const BandSegs sg = band_segments(mask_mode, m0, m1, m2, S, transposed);
  const int n_items = band_total_items(sg);
  const int n_items_cap = (S + kItemRows - 1) / kItemRows + 4;
  const int n_chunks = (S + kChunkCols - 1) / kChunkCols;
  SVGB_REQUIRE(n_items <= n_items_cap, "internal: item count");
  SVGB_REQUIRE(static_cast<size_t>(n_items_cap) * n_chunks < (1ull << 31), "plan too large");
  write_plan(plan, transposed ? SVGB_PLAN_BAND_T : SVGB_PLAN_BAND, BH, S, n_items, 0, mask_mode, m0, m1, m2, 0, 256,
             256 + align_up(2 * sizeof(int4) * n_items_cap, 256), need);
  char* ws = static_cast<char*>(plan_ws);
  plan_band_kernel<<<n_items, kItemRows, 0, static_cast<cudaStream_t>(stream)>>>(
      mask_mode, m0, m1, m2, S, n_chunks, sg, transposed ? 1 : 0, reinterpret_cast<int*>(ws + plan->counts_off),
      reinterpret_cast<int4*>(ws + plan->items_off), reinterpret_cast<int2*>(ws + plan->chunks_off));
  SVGB_LAUNCH_OK();
  return 0;
}

int svgb_attn_plan_band(int mask_mode, int m0, int m1, int m2, int BH, int S, void* plan_ws,
                        size_t ws_bytes, svgb_plan* plan, void* stream) {
  return plan_band_impl(mask_mode, m0, m1, m2, BH, S, plan_ws, ws_bytes, plan, stream, false);
}

int svgb_attn_plan_band_t_bytes(int S, size_t* bytes) { return svgb_attn_plan_band_bytes(S, bytes); }

int svgb_attn_plan_band_t(int mask_mode, int m0, int m1, int m2, int BH, int S, void* plan_ws, size_t ws_bytes,
                          svgb_plan* plan, void* stream) {
  return plan_band_impl(mask_mode, m0, m1, m2, BH, S, plan_ws, ws_bytes, plan, stream, true);
}

int svgb_attn_plan_local_varlen_bytes(int nseg, int Sq, int Skv, size_t* bytes) {
  return plan_local_varlen_bytes(nseg, Sq, Skv, bytes);
}

int svgb_attn_plan_local_varlen(const int32_t* cu_q, const int32_t* cu_k, int nseg, int Sq, int Skv, int sink, int left,
                                int right, void* plan_ws, size_t ws_bytes, svgb_plan* plan, void* stream) {
  return plan_local_varlen_impl(cu_q, cu_k, nseg, Sq, Skv, sink, left, right, plan_ws, ws_bytes, plan, stream, false);
}

int svgb_attn_plan_local_varlen_t(const int32_t* cu_q, const int32_t* cu_k, int nseg, int Sq, int Skv, int sink,
                                  int left, int right, void* plan_ws, size_t ws_bytes, svgb_plan* plan, void* stream) {
  return plan_local_varlen_impl(cu_q, cu_k, nseg, Sq, Skv, sink, left, right, plan_ws, ws_bytes, plan, stream, true);
}

static int plan_block_varlen(const int32_t* cu_q, const int32_t* cu_k, int nseg, int Sq, int Skv, int sink, int window,
                             int block, int first_block, void* plan_ws, size_t ws_bytes, svgb_plan* plan, void* stream,
                             bool transposed) {
  const char* who = transposed ? "svgb_attn_plan_block_varlen_t" : "svgb_attn_plan_block_varlen";
  int m1 = 0;
  if (block_causal_m1(block, first_block, &m1, who) || block_causal_check(sink, m1, window, who)) return -1;
  return plan_local_varlen_impl(cu_q, cu_k, nseg, Sq, Skv, sink, window - 1, 0, plan_ws, ws_bytes, plan, stream,
                                transposed, m1);
}

int svgb_attn_plan_block_varlen(const int32_t* cu_q, const int32_t* cu_k, int nseg, int Sq, int Skv, int sink,
                                int window, int block, int first_block, void* plan_ws, size_t ws_bytes, svgb_plan* plan,
                                void* stream) {
  return plan_block_varlen(cu_q, cu_k, nseg, Sq, Skv, sink, window, block, first_block, plan_ws, ws_bytes, plan, stream,
                           false);
}

int svgb_attn_plan_block_varlen_t(const int32_t* cu_q, const int32_t* cu_k, int nseg, int Sq, int Skv, int sink,
                                  int window, int block, int first_block, void* plan_ws, size_t ws_bytes,
                                  svgb_plan* plan, void* stream) {
  return plan_block_varlen(cu_q, cu_k, nseg, Sq, Skv, sink, window, block, first_block, plan_ws, ws_bytes, plan, stream,
                           true);
}

int svgb_attn_fwd(const void* q, const void* k, const void* v, const float* q_scale, const float* k_scale,
                  const float* v_scale, void* o, float* lse, const int32_t* q_rows, const int32_t* kv_rows,
                  const int32_t* o_rows, int dtype, int BH, int S, int D, long long row_stride,
                  long long head_stride, long long o_row_stride, long long o_head_stride, float sm_scale,
                  const svgb_plan* plan, const void* plan_ws, void* stream) {
  const Strides in = flat_strides(row_stride, head_stride, BH);
  return attn_fwd({q, k, v, q_scale, k_scale, v_scale, o, lse, q_rows, kv_rows, o_rows, dtype, 0, 1, BH, BH, S, S, D,
                   in, in, in, flat_strides(o_row_stride, o_head_stride, BH), sm_scale, plan, plan_ws, 0, 0, nullptr,
                   0, stream},
                  FWD);
}

int svgb_attn_fwd_kv(const void* q, const void* k, const void* v, void* o, float* lse, int dtype, int BH, int Sq,
                     int Skv, int D, long long q_row_stride, long long q_head_stride, long long kv_row_stride,
                     long long kv_head_stride, long long o_row_stride, long long o_head_stride, float sm_scale,
                     const svgb_plan* plan, const void* plan_ws, void* stream) {
  const Strides kv = flat_strides(kv_row_stride, kv_head_stride, BH);
  return attn_fwd({q, k, v, nullptr, nullptr, nullptr, o, lse, nullptr, nullptr, nullptr, dtype, 0, 1, BH, BH, Sq, Skv,
                   D, flat_strides(q_row_stride, q_head_stride, BH), kv, kv,
                   flat_strides(o_row_stride, o_head_stride, BH), sm_scale, plan, plan_ws, 0, 0, nullptr, 0, stream},
                  FWD_KV);
}

int svgb_attn_fwd_gqa(const void* q, const void* k, const void* v, void* o, float* lse, int dtype, int BHq, int BHkv,
                      int Sq, int Skv, int D, long long q_row_stride, long long q_head_stride, long long kv_row_stride,
                      long long kv_head_stride, long long o_row_stride, long long o_head_stride, float sm_scale,
                      const svgb_plan* plan, const void* plan_ws, void* stream) {
  const Strides kv = flat_strides(kv_row_stride, kv_head_stride, BHkv);
  return attn_fwd({q, k, v, nullptr, nullptr, nullptr, o, lse, nullptr, nullptr, nullptr, dtype, 0, 1, BHq, BHkv, Sq,
                   Skv, D, flat_strides(q_row_stride, q_head_stride, BHq), kv, kv,
                   flat_strides(o_row_stride, o_head_stride, BHq), sm_scale, plan, plan_ws, 0, 0, nullptr, 0, stream},
                  FWD_GQA);
}

int svgb_attn_fwd_strided(const void* q, const void* k, const void* v, void* o, float* lse, int dtype, int B, int Hq,
                          int Hkv, int Sq, int Skv, int D, const long long* q_strides, const long long* k_strides,
                          const long long* v_strides, const long long* o_strides, float sm_scale,
                          const svgb_plan* plan, const void* plan_ws, void* stream) {
  Strides st[4];
  if (attn_strided_check(B, Hq, Hkv, {q, k, v, o}, {q_strides, k_strides, v_strides, o_strides}, st,
                         kFwdRules[FWD_STRIDED].who))
    return -1;
  return attn_fwd({q, k, v, nullptr, nullptr, nullptr, o, lse, nullptr, nullptr, nullptr, dtype, 0, B, Hq, Hkv, Sq, Skv,
                   D, st[0], st[1], st[2], st[3], sm_scale, plan, plan_ws, 0, 0, nullptr, 0, stream},
                  FWD_STRIDED);
}

int svgb_attn_fwd_strided_e4m3(const void* q, const void* k, const void* v, const float* q_scale,
                               const float* k_scale, const float* v_scale, void* o, float* lse, int B, int Hq, int Hkv,
                               int Sq, int Skv, int D, const long long* q_strides, const long long* k_strides,
                               const long long* v_strides, const long long* o_strides, float sm_scale,
                               const svgb_plan* plan, const void* plan_ws, void* stream) {
  Strides st[4];
  if (attn_strided_check(B, Hq, Hkv, {q, k, v, o}, {q_strides, k_strides, v_strides, o_strides}, st,
                         kFwdRules[FWD_STRIDED_E4M3].who))
    return -1;
  return attn_fwd({q, k, v, q_scale, k_scale, v_scale, o, lse, nullptr, nullptr, nullptr, SVGB_E4M3, 0, B, Hq, Hkv, Sq,
                   Skv, D, st[0], st[1], st[2], st[3], sm_scale, plan, plan_ws, 0, 0, nullptr, 0, stream},
                  FWD_STRIDED_E4M3);
}

int svgb_attn_fwd_kvcache_e4m3_rows(const void* q, const void* k, const void* v, const float* q_scale,
                                    const float* k_scale, const float* v_scale, void* o, float* lse, int Hq, int Hkv,
                                    int Sq, int num_blocks, int block_rows, int D, const long long* q_strides,
                                    const long long* k_strides, const long long* v_strides, const long long* o_strides,
                                    float sm_scale, const svgb_plan* plan, const void* plan_ws, void* stream) {
  Strides st[4];
  if (attn_strided_check(1, Hq, Hkv, {q, k, v, o}, {q_strides, k_strides, v_strides, o_strides}, st,
                         kFwdRules[FWD_KVCACHE_E4M3_ROWS].who))
    return -1;
  return attn_fwd({q, k, v, q_scale, k_scale, v_scale, o, lse, nullptr, nullptr, nullptr, SVGB_E4M3, 1, 1, Hq, Hkv, Sq,
                   static_cast<int>(static_cast<long long>(num_blocks) * block_rows), D, st[0], st[1], st[2], st[3],
                   sm_scale, plan, plan_ws, num_blocks, block_rows, nullptr, 0, stream},
                  FWD_KVCACHE_E4M3_ROWS);
}

int svgb_attn_fwd_kvcache_split_bytes(int num_splits, int rows, int Hq, int D, size_t* bytes) {
  SVGB_REQUIRE(num_splits >= 1 && rows > 0 && Hq > 0 && (D == 64 || D == 128) && bytes,
               "bad arguments (num_splits=%d, rows=%d, Hq=%d, D=%d)", num_splits, rows, Hq, D);
  const size_t n = static_cast<size_t>(num_splits) * rows * Hq;
  *bytes = n * D * sizeof(float) + n * sizeof(float);
  return 0;
}

int svgb_attn_fwd_kvcache_split(const void* q, const void* k, const void* v, const float* q_scale, const float* k_scale,
                                const float* v_scale, void* o, float* lse, int dtype, int row_scales, int B, int Hq,
                                int Hkv, int Sq, int num_blocks, int block_rows, int D, const long long* q_strides,
                                const long long* k_strides, const long long* v_strides, const long long* o_strides,
                                float sm_scale, const svgb_plan* plan, const void* plan_ws, void* ws, size_t ws_bytes,
                                void* stream) {
  Strides st[4];
  if (attn_strided_check(1, Hq, Hkv, {q, k, v, o}, {q_strides, k_strides, v_strides, o_strides}, st,
                         kFwdRules[FWD_KVCACHE_SPLIT].who))
    return -1;
  return attn_fwd({q, k, v, q_scale, k_scale, v_scale, o, lse, nullptr, nullptr, nullptr, dtype, row_scales, B, Hq, Hkv,
                   Sq, static_cast<int>(static_cast<long long>(num_blocks) * block_rows), D, st[0], st[1], st[2], st[3],
                   sm_scale, plan, plan_ws, num_blocks, block_rows, ws, ws_bytes, stream},
                  FWD_KVCACHE_SPLIT);
}

int svgb_density(const uint8_t* map, const int32_t* row_sz, const int32_t* col_sz, int BH, int QC,
                 int KC, float* density, void* stream) {
  SVGB_REQUIRE(map && row_sz && col_sz && density && BH > 0 && QC > 0 && KC > 0, "bad arguments");
  density_kernel<<<BH, 256, 0, static_cast<cudaStream_t>(stream)>>>(map, row_sz, col_sz, QC, KC, density);
  SVGB_LAUNCH_OK();
  return 0;
}

int svgb_selftest_tile(const void* q, const void* k, const void* v, float* s_out, float* o_out,
                       int D, int dtype, float p_scale, void* stream) {
  SVGB_REQUIRE(q && k && v && s_out && o_out, "null pointer");
  SVGB_REQUIRE(D == 64 || D == 128, "head_dim %d unsupported", D);
  CUtensorMap qm, km, vm;
  if (encode_tmap_hsd(&qm, q, dtype, 1, 128, D, D, 128LL * D)) return -1;
  if (encode_tmap_hsd(&km, k, dtype, 1, 128, D, D, 128LL * D)) return -1;
  if (encode_tmap_hsd(&vm, v, dtype, 1, 128, D, D, 128LL * D)) return -1;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (D == 128)
    return dtype == SVGB_BF16 ? launch_selftest<128, true>(qm, km, vm, s_out, o_out, p_scale, st)
                              : launch_selftest<128, false>(qm, km, vm, s_out, o_out, p_scale, st);
  return dtype == SVGB_BF16 ? launch_selftest<64, true>(qm, km, vm, s_out, o_out, p_scale, st)
                            : launch_selftest<64, false>(qm, km, vm, s_out, o_out, p_scale, st);
}

}  // extern "C"
