// KV cache: the in-place append of new key / value rows (svgb_kvcache_append, and svgb_kvcache_append_e4m3 and
// svgb_kvcache_append_e4m3_rows into an e4m3 cache with per-head or per-row scales) and the plan of the attention of a
// batch of streams into a contiguous or paged cache (svgb_attn_plan_kvcache), run by the attention forward
// (attn_kernel.cuh).
// Both read the per-stream lengths on the device only.
#include <cuda_fp16.h>

#include <algorithm>
#include <type_traits>

#include "../../include/svgb200.h"
#include "attn_common.cuh"
#include "fp8_rows.cuh"
#include "host_common.h"

namespace svgb {

// Logical keys of stream b after the append, clamped to its capacity: lengths past the capacity or negative give an
// unspecified result that stays inside the cache
__device__ __forceinline__ int kv_len(int cache_seqlen, int new_len, int cap) {
  const long long x = static_cast<long long>(max(cache_seqlen, 0)) + new_len;
  return static_cast<int>(x < cap ? x : cap);
}

// The cache is num_blocks blocks of block_rows rows: a contiguous cache [B_cache, S_cache, Hkv, D] (stream b in block
// cache_batch_idx[b], or b) or a paged one [num_pages, page_size, Hkv, D] (logical key t of stream b in row t % page_size
// of page block_table[b, t / page_size]).  Out-of-range blocks are clamped to the cache.
__device__ __forceinline__ int kv_block(const int* __restrict__ batch_idx, const int* __restrict__ table, int b, int t,
                                        int nblocks, int block_rows, int max_pages) {
  const int blk = table ? __ldg(&table[static_cast<size_t>(b) * max_pages + t / block_rows])
                        : (batch_idx ? __ldg(&batch_idx[b]) : b);
  return min(max(blk, 0), nblocks - 1);
}

// what the append writes from 16-bit new rows: the rows themselves, e4m3 quantised from bf16 or fp16 rows with the
// caller's per-head scales, or e4m3 quantised with a power-of-two scale per row, written beside the row (fp8_rows.cuh)
enum KvStore { KV_COPY, KV_E4M3_BF16, KV_E4M3_F16, KV_E4M3_ROWS_BF16, KV_E4M3_ROWS_F16 };

// 8 16-bit elements -> 8 e4m3 bytes, RN-satfinite(x * inv), as quantize_kernel (quant_fp8.cu)
template <bool BF16>
__device__ __forceinline__ uint2 kv_to_e4m3(uint4 x, float inv) {
  const uint32_t w[4] = {x.x, x.y, x.z, x.w};
  uint32_t out[2];
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    uint16_t p[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const uint16_t lo16 = static_cast<uint16_t>(w[2 * j + i] & 0xffff), hi16 = static_cast<uint16_t>(w[2 * j + i] >> 16);
      const float a = (BF16 ? __uint_as_float(static_cast<uint32_t>(lo16) << 16) : __half2float(__ushort_as_half(lo16))) * inv;
      const float b = (BF16 ? __uint_as_float(static_cast<uint32_t>(hi16) << 16) : __half2float(__ushort_as_half(hi16))) * inv;
      asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(p[i]) : "f"(b), "f"(a));
    }
    out[j] = static_cast<uint32_t>(p[0]) | (static_cast<uint32_t>(p[1]) << 16);
  }
  return make_uint2(out[0], out[1]);
}

// =============================================================================================
// Append: new rows k, v [B, Snew, Hkv, D] at logical keys cache_seqlens[b] .. + Snew - 1 of each stream, one 16-byte
// vector of K and one of V per thread (e4m3 caches: 8 elements of each, written as 8 bytes).  Rows whose logical key
// lies outside [0, capacity) or whose block lies outside the cache are not written.
// =============================================================================================
// Variable-length append (cu_new != NULL): the new rows are k, v [Snew = total_new, Hkv, D] and stream b's are rows
// [cu_new[b], cu_new[b+1]) (the last stream that starts at or before a row holds it), written at keys cache_seqlens[b] ..
// under the same skip rules; a row outside every stream is not written.
__device__ __forceinline__ int kv_row_stream(const int* __restrict__ cu, int B, int row) {
  int lo = 0, hi = B - 1;  // largest b < B with cu[b] <= row
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(&cu[mid]) <= row) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

template <int kStore, typename Cache = typename std::conditional<kStore == KV_COPY, uint16_t, uint8_t>::type>
__global__ void __launch_bounds__(256)
kv_append_kernel(Cache* __restrict__ kc, Cache* __restrict__ vc, const uint16_t* __restrict__ k,
                 const uint16_t* __restrict__ v, const int* __restrict__ seqlens, const int* __restrict__ batch_idx,
                 const int* __restrict__ table, int B, int Snew, int Hkv, int nvec, int nblocks, int block_rows,
                 int max_pages, int cap, Strides kcs, Strides vcs, Strides ks, Strides vs,
                 const float* __restrict__ k_scale, const float* __restrict__ v_scale, float* __restrict__ k_rows,
                 float* __restrict__ v_rows, const int* __restrict__ cu_new = nullptr) {
  const long long total = static_cast<long long>(cu_new ? 1 : B) * Snew * Hkv * nvec;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(idx % nvec);
    long long r = idx / nvec;
    const int h = static_cast<int>(r % Hkv);
    r /= Hkv;
    int i = static_cast<int>(r % Snew), b = static_cast<int>(r / Snew);
    const long long ko = b * ks.b + i * ks.r, vo = b * vs.b + i * vs.r;  // varlen: b = 0 and i = r, the packed row
    if (cu_new) {  // the packed row's stream, and its index inside that stream
      b = kv_row_stream(cu_new, B, i);
      i -= __ldg(&cu_new[b]);
      if (i < 0 || r >= __ldg(&cu_new[b + 1])) continue;
    }
    const long long t = static_cast<long long>(__ldg(&seqlens[b])) + i;
    if (t < 0 || t >= cap) continue;
    const int tt = static_cast<int>(t);
    int blk, row;
    if (table) {
      blk = __ldg(&table[static_cast<size_t>(b) * max_pages + tt / block_rows]);
      row = tt % block_rows;
    } else {
      blk = batch_idx ? __ldg(&batch_idx[b]) : b;
      row = tt;
    }
    if (blk < 0 || blk >= nblocks) continue;
    const long long e = 8ll * c;
    const uint4 kx = *reinterpret_cast<const uint4*>(k + ko + h * ks.h + e);
    const uint4 vx = *reinterpret_cast<const uint4*>(v + vo + h * vs.h + e);
    if constexpr (kStore == KV_COPY) {
      *reinterpret_cast<uint4*>(kc + blk * kcs.b + row * kcs.r + h * kcs.h + e) = kx;
      *reinterpret_cast<uint4*>(vc + blk * vcs.b + row * vcs.r + h * vcs.h + e) = vx;
    } else if constexpr (kStore == KV_E4M3_BF16 || kStore == KV_E4M3_F16) {
      constexpr bool BF16 = kStore == KV_E4M3_BF16;
      *reinterpret_cast<uint2*>(kc + blk * kcs.b + row * kcs.r + h * kcs.h + e) =
          kv_to_e4m3<BF16>(kx, 1.f / __ldg(&k_scale[h]));
      *reinterpret_cast<uint2*>(vc + blk * vcs.b + row * vcs.r + h * vcs.h + e) =
          kv_to_e4m3<BF16>(vx, 1.f / __ldg(&v_scale[h]));
    } else {
      // per row (D = 128, nvec = 16): the 16 threads of a (row, head) are an aligned half-warp, since the block size
      // and the grid stride are multiples of 16, and every skip above is uniform over them
      constexpr bool BF16 = kStore == KV_E4M3_ROWS_BF16;
      const unsigned half = 0xffffu << (threadIdx.x & 16);
      int ek, ev;
      *reinterpret_cast<uint2*>(kc + blk * kcs.b + row * kcs.r + h * kcs.h + e) = e4m3_row_quantise<BF16>(kx, half, &ek);
      *reinterpret_cast<uint2*>(vc + blk * vcs.b + row * vcs.r + h * vcs.h + e) = e4m3_row_quantise<BF16>(vx, half, &ev);
      if (c == 0) {
        const long long si = (static_cast<long long>(blk) * Hkv + h) * block_rows + row;  // [num_blocks, Hkv, block_rows]
        k_rows[si] = e4m3_row_scale(ek);
        v_rows[si] = e4m3_row_scale(ev);
      }
    }
  }
}

// =============================================================================================
// Plan: one warp per item.  Stream b's Sq query rows (packed rows b Sq ..) are cut into items of 256 rows from its first
// row, and every item has `slots` chunk slots.  The warp visits the chunks that can hold an allowed key -- those of the
// sinks and those of the item's window, so the pages behind a window are never read -- classifies each from the band's
// interval form on logical positions (seg_chunk_kind) and writes the kept ones, compacted with a ballot, with the
// physical row its TMA box loads from and its logical index in the meta's high bits.
// Split plans (nsplit > 1) repeat the B I items once per split, split-major: item s B I + i is split s of item i, and
// visits the s-th piece of ceil(nvis / nsplit) of the item's nvis visited chunks (sinks first, then the window), so the
// item's split lists, concatenated in split order, are its single-pass list.
// Block-causal plans (block = m1 of SVGB_MASK_BLOCK_CAUSAL, left = W - 1, right = 0) round the item's first and last
// positions to their block ends first: the visited window is [e(p0) - W, e(p1) - 1], and block = 0 is the token rule.
// =============================================================================================
// The list of one item (one warp): rows r0 .. r0 + nr - 1 of stream b, whose L keys sit at logical positions 0 .. L - 1
// and whose query row q sits at position q - shift; split sp of nsplit.  Writes the kept chunks at `list` and returns
// their count (at most slots).
__device__ __forceinline__ int kv_item_list(const int* __restrict__ batch_idx, const int* __restrict__ table, int b,
                                            int L, int shift, int r0, int nr, int sp, int nsplit, int nblocks,
                                            int block_rows, int max_pages, int slots, int sink, int left, int right,
                                            int block, int2* __restrict__ list) {
  const int lane = threadIdx.x & 31;
  SegOrigin o;
  o.shift = shift;
  o.sink_end = sink;
  // chunks that can hold an allowed key: [0, ns) with sinks, [jlo, jhi] inside the window of positions p0 .. p1
  const int nch = (L + kChunkCols - 1) / kChunkCols;
  const int ns = (min(sink, L) + kChunkCols - 1) / kChunkCols;
  // block-causal (block != 0): the rows' positions rounded to their block ends, where the mask is the local band
  // (sink, W - 1, 0); rounding is monotone, so rows e0 .. e1 give the chunk kinds of the item's rows exactly
  const int p0 = r0 - o.shift, p1 = p0 + nr - 1;
  const int e0 = block ? block_last(p0, block) : p0, e1 = block ? block_last(p1, block) : p1;
  const long long lo = std::max(static_cast<long long>(e0) - left, 0ll),
                  hi = std::min(static_cast<long long>(e1) + right, static_cast<long long>(L) - 1);
  const int jlo = max(ns, static_cast<int>(lo / kChunkCols));
  const int jhi = hi < lo ? -1 : min(nch - 1, static_cast<int>(hi / kChunkCols));
  const int nvis = ns + max(0, jhi - jlo + 1);
  const int piece = (nvis + nsplit - 1) / nsplit;  // this split's visited chunks: [v_lo, v_hi)
  const int v_lo = min(nvis, sp * piece), v_hi = min(nvis, v_lo + piece);
  int n = 0;
  for (int v0 = v_lo; v0 < v_hi; v0 += 32) {
    const int vi = v0 + lane;
    const int j = vi < ns ? vi : jlo + (vi - ns);
    const int c0 = j * kChunkCols, valid = min(kChunkCols, L - c0);
    const int kind = vi < v_hi ? seg_chunk_kind(false, e0 + o.shift, e1 + o.shift, c0, c0 + valid - 1, o, left, right) : 0;
    const unsigned m = __ballot_sync(0xffffffffu, kind != 0);
    const int at = n + __popc(m & ((1u << lane) - 1u));
    if (kind != 0 && at < slots) {
      const int blk = kv_block(batch_idx, table, b, c0, nblocks, block_rows, max_pages);
      const int row = blk * block_rows + (table ? c0 % block_rows : c0);
      list[at] = make_int2(row, chunk_meta(valid, kind == 2) | (j << kChunkLogicalShift));
    }
    n += __popc(m);
  }
  return min(n, slots);
}

__global__ void __launch_bounds__(256)
kv_lists_kernel(const int* __restrict__ seqlens, const int* __restrict__ batch_idx, const int* __restrict__ table, int B,
                int Sq, int Snew, int nblocks, int block_rows, int max_pages, int cap, int slots, int nsplit, int sink,
                int left, int right, int block, int* __restrict__ counts, int* __restrict__ kv,
                int2* __restrict__ chunks, int4* __restrict__ items) {
  const int lane = threadIdx.x & 31;
  const int per = (Sq + kItemRows - 1) / kItemRows;  // items per stream
  const int it = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (it == 0 && lane == 0) {
    counts[0] = nsplit * B * per;
    kv[0] = B;
    kv[1] = Sq;
  }
  if (it >= nsplit * B * per) return;
  const int sp = it / (B * per), bi = it - sp * (B * per);
  const int b = bi / per, k = bi - b * per;
  const int L = kv_len(__ldg(&seqlens[b]), Snew, cap);
  if (sp == 0 && k == 0 && lane == 0) kv[2 + b] = L;
  const int r0 = b * Sq + k * kItemRows, nr = min(kItemRows, Sq - k * kItemRows);
  const int list = it * slots;
  const int n = kv_item_list(batch_idx, table, b, L, (b + 1) * Sq - L, r0, nr, sp, nsplit, nblocks, block_rows,
                             max_pages, slots, sink, left, right, block, chunks + list);
  if (lane == 0) put_item(items + 2 * it, r0, nr, list, n);
}

// Variable-length plans: stream b's queries are packed rows [cq_b, cq_b+1) with cq_b = cu_q[b] clamped to [0, total_q],
// and its L_b = min(cache_seqlens[b] + cu_new[b+1] - cu_new[b], cap) keys (no cu_new: no rows appended).  Its rows are
// cut into ceil(Lq_b / 256) items from its first row, numbered in stream order; item s I + i is split s of item i, and
// items i past the streams' items get zero rows and an empty list, so they write nothing.  Block 0 writes the header
// {B, kKvVarlen, L_b, cq_b}; each warp finds its item's stream from the scanned item counts, 32 streams at a time.
__device__ __forceinline__ int kv_row_bound(const int* __restrict__ cu, int b, int total) {
  return min(max(__ldg(&cu[b]), 0), total);
}
__device__ __forceinline__ int kv_new_rows(const int* __restrict__ cu_new, int b) {
  return cu_new ? max(__ldg(&cu_new[b + 1]) - __ldg(&cu_new[b]), 0) : 0;
}

__global__ void __launch_bounds__(256)
kv_varlen_lists_kernel(const int* __restrict__ cu_q, const int* __restrict__ seqlens, const int* __restrict__ cu_new,
                       const int* __restrict__ batch_idx, const int* __restrict__ table, int B, int total_q, int I,
                       int nblocks, int block_rows, int max_pages, int cap, int slots, int nsplit, int sink, int left,
                       int right, int block, int* __restrict__ counts, int* __restrict__ kv, int2* __restrict__ chunks,
                       int4* __restrict__ items) {
  const int lane = threadIdx.x & 31;
  const int it = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (blockIdx.x == 0) {
    for (int b = threadIdx.x; b <= B; b += blockDim.x) {
      kv[2 + B + b] = kv_row_bound(cu_q, b, total_q);
      if (b < B) kv[2 + b] = kv_len(__ldg(&seqlens[b]), kv_new_rows(cu_new, b), cap);
    }
    if (threadIdx.x == 0) {
      counts[0] = nsplit * I;
      kv[0] = B;
      kv[1] = kKvVarlen;
    }
  }
  if (it >= nsplit * I) return;
  const int sp = it / I, i = it - sp * I;
  int b = -1, k = 0;  // item i is item k of stream b
  for (int b0 = 0, before = 0; b0 < B && b < 0; b0 += 32) {
    const int bb = b0 + lane;
    int lo = 0, nq = 0;
    if (bb < B) {
      lo = kv_row_bound(cu_q, bb, total_q);
      nq = max(kv_row_bound(cu_q, bb + 1, total_q) - lo, 0);
    }
    const int n = (nq + kItemRows - 1) / kItemRows;
    int incl = n;  // inclusive scan of the item counts over the lanes
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int x = __shfl_up_sync(0xffffffffu, incl, d);
      if (lane >= d) incl += x;
    }
    const int first = before + incl - n;
    const unsigned hit = __ballot_sync(0xffffffffu, i >= first && i < first + n);
    if (hit) {
      const int src = __ffs(hit) - 1;
      b = b0 + src;
      k = i - __shfl_sync(0xffffffffu, first, src);
    }
    before += __shfl_sync(0xffffffffu, incl, 31);
  }
  const int list = it * slots;
  if (b < 0) {
    if (lane == 0) put_item(items + 2 * it, 0, 0, list, 0);
    return;
  }
  const int lo = kv_row_bound(cu_q, b, total_q), hi = max(kv_row_bound(cu_q, b + 1, total_q), lo);
  const int L = kv_len(__ldg(&seqlens[b]), kv_new_rows(cu_new, b), cap);
  const int r0 = lo + k * kItemRows, nr = min(kItemRows, hi - r0);
  const int n = kv_item_list(batch_idx, table, b, L, hi - L, r0, nr, sp, nsplit, nblocks, block_rows, max_pages, slots,
                             sink, left, right, block, chunks + list);
  if (lane == 0) put_item(items + 2 * it, r0, nr, list, n);
}

// Workspace of a KV-cache plan, 16-byte aligned pieces:
//   counts (16 B) | {B, Sq, L_0 .. L_B-1} | items 2 int4 [nsplit B I] | chunks [nsplit B I slots]
// with I = ceil(Sq / 256) items per stream and slots = min(ceil(cap / 128), ceil(sink / 128) + (255 + left + right) / 128
// + 2), the chunks an item can visit: its sinks and the window of its 256 rows; a split plan's items have
// ceil(slots / nsplit) slots each, the most a split's piece can hold.  A block-causal plan passes right = C - 1 here: its
// rows' block ends lie up to C - 1 past them, so an item's window [e(p0) - W, e(p1) - 1] spans at most 255 + (W - 1) +
// (C - 1) + 1 keys.
// A variable-length plan (varlen_items = I > 0, its items per split) has nsplit I items, and its header
// {B, kKvVarlen, L_0 .. L_B-1, cq_0 .. cq_B} holds B + 1 more ints.
struct KvLayout {
  long long items, slots;
  size_t items_off, chunks_off, bytes;
};
static KvLayout kv_layout(int B, int Sq, int cap, int sink, int left, int right, int nsplit = 1,
                          long long varlen_items = 0) {
  KvLayout L;
  L.items = static_cast<long long>(nsplit) *
            (varlen_items > 0 ? varlen_items : static_cast<long long>(B) * ((Sq + kItemRows - 1) / kItemRows));
  const long long win = (static_cast<long long>(sink) + kChunkCols - 1) / kChunkCols +
                        (kItemRows - 1 + static_cast<long long>(left) + right) / kChunkCols + 2;
  const long long slots = std::min<long long>((static_cast<long long>(cap) + kChunkCols - 1) / kChunkCols, win);
  L.slots = (slots + nsplit - 1) / nsplit;
  L.items_off = SVGB_PLAN_SEG_BOUNDS_OFF +
                align_up(sizeof(int) * (2 + static_cast<size_t>(B) + (varlen_items > 0 ? B + 1 : 0)), 16);
  L.chunks_off = L.items_off + 2 * sizeof(int4) * L.items;
  L.bytes = L.chunks_off + sizeof(int2) * L.items * L.slots;
  return L;
}

// the cache geometry both entries take: num_blocks blocks of block_rows rows, paged when block_table is given; returns
// the capacity of a stream in *cap
static int kv_geometry(const int32_t* cache_batch_idx, const int32_t* block_table, int num_blocks, int block_rows,
                       int max_pages, int* cap, const char* who) {
  SVGB_REQUIRE(num_blocks > 0 && block_rows > 0, "%s: bad cache geometry (num_blocks=%d, block_rows=%d)", who,
               num_blocks, block_rows);
  SVGB_REQUIRE(static_cast<long long>(num_blocks) * block_rows < (1ll << 31), "%s: cache of %d x %d rows too large",
               who, num_blocks, block_rows);
  long long c = block_rows;
  if (block_table) {
    SVGB_REQUIRE(block_rows % kChunkCols == 0,
                 "%s: page_size %d must be a multiple of 128 (no 128-key chunk may straddle two pages)", who, block_rows);
    SVGB_REQUIRE(max_pages > 0, "%s: block_table needs max_pages > 0 (got %d)", who, max_pages);
    SVGB_REQUIRE(!cache_batch_idx, "%s: cache_batch_idx is for contiguous caches; a paged cache takes block_table only",
                 who);
    c = static_cast<long long>(max_pages) * block_rows;
  }
  // the logical chunk index lives in 22 bits of the chunk meta
  SVGB_REQUIRE(c <= (1ll << 29), "%s: a stream's capacity (%lld keys) exceeds 2^29", who, c);
  *cap = static_cast<int>(c);
  return 0;
}

}  // namespace svgb

using namespace svgb;

// the per-row scale tensors of an e4m3 cache, float [num_blocks, Hkv, block_rows] contiguous: one 128-key chunk of one
// head is 512 contiguous bytes that the attention loads with one TMA box, whose rows need 16-byte alignment
int svgb::kv_scale_rows_check(const float* k_scale, const float* v_scale, int block_rows, const char* who) {
  SVGB_REQUIRE(k_scale && v_scale, "%s needs both per-row scale tensors k_scale and v_scale (float [num_blocks, Hkv, "
               "block_rows])", who);
  SVGB_REQUIRE((reinterpret_cast<uintptr_t>(k_scale) & 15) == 0 && (reinterpret_cast<uintptr_t>(v_scale) & 15) == 0,
               "%s: the per-row scale tensors must be 16-byte aligned", who);
  SVGB_REQUIRE(block_rows % 4 == 0,
               "%s: per-row scales need block_rows (%d) a multiple of 4, so that every scale row is 16-byte aligned", who,
               block_rows);
  return 0;
}

// every append: 16-bit new rows (dtype) into a 16-bit cache of that dtype (no scales), into an e4m3 cache with the
// per-head scales k_scale, v_scale, or (row_scales) into an e4m3 cache with per-row scales k_scale, v_scale that the
// append writes; `formats` are those the entry takes (FMT_*)
enum { FMT_16BIT = 1, FMT_E4M3 = 2, FMT_E4M3_ROWS = 4 };
static int kv_append_run(void* k_cache, void* v_cache, const void* k, const void* v, const int32_t* cache_seqlens,
                         const int32_t* cache_batch_idx, const int32_t* block_table, int dtype, int B, int Snew,
                         int Hkv, int D, int num_blocks, int block_rows, int max_pages, const long long* kc_strides,
                         const long long* vc_strides, const long long* k_strides, const long long* v_strides,
                         float* k_scale, float* v_scale, bool row_scales, unsigned formats, void* stream,
                         const char* who, const int32_t* cu_new = nullptr) {
  const int fmt = row_scales ? FMT_E4M3_ROWS : k_scale || v_scale ? FMT_E4M3 : FMT_16BIT;
  const bool e4m3 = fmt != FMT_16BIT;
  SVGB_REQUIRE(formats & fmt, "%s needs both scale vectors k_scale and v_scale (float [Hkv])", who);
  if (fmt == FMT_E4M3_ROWS && kv_scale_rows_check(k_scale, v_scale, block_rows, who)) return -1;
  SVGB_REQUIRE(fmt != FMT_E4M3 || (k_scale && v_scale), "%s: an e4m3 cache needs both scale vectors k_scale and "
               "v_scale (float [Hkv]); a 16-bit cache takes neither", who);
  SVGB_REQUIRE(cache_seqlens, "null pointer");
  SVGB_REQUIRE(dtype == SVGB_BF16 || dtype == SVGB_F16, "%s takes bf16 or fp16 %s (dtype %d)", who,
               e4m3 ? "new rows" : "caches", dtype);
  SVGB_REQUIRE(D == 64 || D == 128, "%s: head_dim %d unsupported (64 or 128)", who, D);
  SVGB_REQUIRE(fmt != FMT_E4M3_ROWS || D == 128, "%s: per-row scales need head_dim 128 (got %d)", who, D);
  SVGB_REQUIRE(Snew > 0, "%s: no new rows (Snew=%d)", who, Snew);
  Strides st[4];
  if (attn_strided_check(B, Hkv, Hkv, {k_cache, v_cache, k, v}, {kc_strides, vc_strides, k_strides, v_strides}, st, who))
    return -1;
  if (e4m3)
    for (int i = 0; i < 2; ++i)
      SVGB_REQUIRE(st[i].b % 16 == 0 && st[i].h % 16 == 0 && st[i].r % 16 == 0,
                   "%s: every e4m3 cache (block, head, row) stride must be a multiple of 16 bytes (got %lld, %lld, %lld)",
                   who, st[i].b, st[i].h, st[i].r);
  int cap = 0;
  if (kv_geometry(cache_batch_idx, block_table, num_blocks, block_rows, max_pages, &cap, who)) return -1;
  const int nvec = D / 8;
  const long long total = static_cast<long long>(cu_new ? 1 : B) * Snew * Hkv * nvec;
  const unsigned blocks = static_cast<unsigned>(std::min<long long>((total + 255) / 256, 1 << 20));
  cudaStream_t cs = static_cast<cudaStream_t>(stream);
  const uint16_t *kn = static_cast<const uint16_t*>(k), *vn = static_cast<const uint16_t*>(v);
  if (!e4m3) {
    kv_append_kernel<KV_COPY><<<blocks, 256, 0, cs>>>(
        static_cast<uint16_t*>(k_cache), static_cast<uint16_t*>(v_cache), kn, vn, cache_seqlens, cache_batch_idx,
        block_table, B, Snew, Hkv, nvec, num_blocks, block_rows, max_pages, cap, st[0], st[1], st[2], st[3], nullptr,
        nullptr, nullptr, nullptr, cu_new);
  } else if (row_scales) {
    auto kern = dtype == SVGB_BF16 ? kv_append_kernel<KV_E4M3_ROWS_BF16> : kv_append_kernel<KV_E4M3_ROWS_F16>;
    kern<<<blocks, 256, 0, cs>>>(static_cast<uint8_t*>(k_cache), static_cast<uint8_t*>(v_cache), kn, vn, cache_seqlens,
                                 cache_batch_idx, block_table, B, Snew, Hkv, nvec, num_blocks, block_rows, max_pages,
                                 cap, st[0], st[1], st[2], st[3], nullptr, nullptr, k_scale, v_scale, cu_new);
  } else {
    auto kern = dtype == SVGB_BF16 ? kv_append_kernel<KV_E4M3_BF16> : kv_append_kernel<KV_E4M3_F16>;
    kern<<<blocks, 256, 0, cs>>>(static_cast<uint8_t*>(k_cache), static_cast<uint8_t*>(v_cache), kn, vn, cache_seqlens,
                                 cache_batch_idx, block_table, B, Snew, Hkv, nvec, num_blocks, block_rows, max_pages,
                                 cap, st[0], st[1], st[2], st[3], k_scale, v_scale, nullptr, nullptr, cu_new);
  }
  SVGB_LAUNCH_OK();
  return 0;
}

// Variable-length plans (svgb_attn_plan_kvcache_varlen): the item bound I per split, at most ceil(max_q / 256) items
// per stream and at most (total_q + 255 B) / 256 in all, since sum ceil(Lq_b / 256) <= (sum Lq_b + 255 B) / 256
static long long kv_varlen_items(int B, int total_q, int max_q) {
  return std::min<long long>(static_cast<long long>(B) * ((max_q + kItemRows - 1) / kItemRows),
                             (static_cast<long long>(total_q) + (kItemRows - 1) * static_cast<long long>(B)) / kItemRows);
}

// What one KV-cache plan is: B streams of Sq query rows each (uniform), or total_q = Sq packed rows of which a stream
// holds at most max_q (varlen); the local band (sink, left, right) or the block-causal mask (sink, window, block,
// first_block); n splits, and whether it is a split plan (SVGB_PLAN_KVCACHE_SPLIT).
struct KvPlanSpec {
  int B, Sq, max_q;
  bool varlen;
  int sink, left, right;
  bool block_causal;
  int window, block, first_block;
  int nsplit;
  bool split;
};
// the checked plan: its mask (m1 = 0, or m1 of SVGB_MASK_BLOCK_CAUSAL), the planner's left and right, I and the layout
struct KvPlanArgs {
  int m1, left, right;
  long long I;
  KvLayout L;
};

// Every argument rule of the KV-cache planners and their _bytes twins, against the capacity cap of a stream.
static int kv_plan_check(const KvPlanSpec& s, int cap, KvPlanArgs* a, const char* who) {
  SVGB_REQUIRE(s.B > 0 && s.Sq > 0 && cap > 0, "%s: bad arguments (B=%d, rows=%d, capacity=%d)", who, s.B, s.Sq, cap);
  const long long rows = s.varlen ? s.Sq : static_cast<long long>(s.B) * s.Sq;
  SVGB_REQUIRE(rows < (1ll << 30), "%s: %lld query rows too many", who, rows);
  SVGB_REQUIRE(!s.varlen || (s.max_q >= 1 && s.max_q <= s.Sq), "%s: max_q (%d) must lie in [1, total_q = %d]", who,
               s.max_q, s.Sq);
  SVGB_REQUIRE(s.nsplit >= 1, "%s: num_splits (%d) must be >= 1", who, s.nsplit);
  a->m1 = 0;
  int widen = 0;  // the layout's right beyond the planner's: C - 1 for a block-causal plan
  if (s.block_causal) {
    SVGB_REQUIRE(s.left == 0 && s.right == 0,
                 "%s: a block-causal plan (block = %d) takes (window, block, first_block); left and right must be 0 "
                 "(got %d, %d)", who, s.block, s.left, s.right);
    if (block_causal_m1(s.block, s.first_block, &a->m1, who) || block_causal_check(s.sink, a->m1, s.window, who))
      return -1;
    a->left = s.window - 1;
    a->right = 0;
    widen = s.block - 1;
  } else {
    SVGB_REQUIRE(s.window == 0 && s.first_block == 0,
                 "%s: a local plan (block = 0) takes (left, right); window and first_block must be 0 (got %d, %d)", who,
                 s.window, s.first_block);
    SVGB_REQUIRE(s.sink >= 0 && s.left >= 0 && s.right >= 0, "%s: sink (%d), left (%d) and right (%d) must be >= 0",
                 who, s.sink, s.left, s.right);
    a->left = s.left;
    a->right = s.right;
  }
  a->I = s.varlen ? kv_varlen_items(s.B, s.Sq, s.max_q) : 0;
  a->L = kv_layout(s.B, s.Sq, cap, s.sink, a->left, a->right + widen, s.nsplit, a->I);
  SVGB_REQUIRE(a->L.items * a->L.slots < (1ll << 31) && a->L.items < (1ll << 31),
               "%s: plan too large for 32-bit chunk offsets", who);
  return 0;
}

static int kv_plan_bytes(const KvPlanSpec& s, int cap, size_t* bytes, const char* who) {
  SVGB_REQUIRE(bytes, "null pointer");
  KvPlanArgs a;
  if (kv_plan_check(s, cap, &a, who)) return -1;
  *bytes = a.L.bytes;
  return 0;
}

// Every KV-cache planner: the checks, the descriptor and one launch of the uniform or the variable-length list kernel.
// Uniform plans take Snew new rows per stream, variable-length plans cu_q and the optional cu_new.
static int kv_plan(const KvPlanSpec& s, const int32_t* cu_q, const int32_t* cache_seqlens, const int32_t* cu_new,
                   int Snew, const int32_t* cache_batch_idx, const int32_t* block_table, int num_blocks, int block_rows,
                   int max_pages, void* plan_ws, size_t ws_bytes, svgb_plan* plan, void* stream, const char* who) {
  SVGB_REQUIRE((cu_q || !s.varlen) && cache_seqlens && plan_ws && plan, "null pointer");
  SVGB_REQUIRE(Snew >= 0, "%s: Snew=%d < 0", who, Snew);
  int cap = 0;
  if (kv_geometry(cache_batch_idx, block_table, num_blocks, block_rows, max_pages, &cap, who)) return -1;
  KvPlanArgs a;
  if (kv_plan_check(s, cap, &a, who)) return -1;
  const KvLayout& L = a.L;
  SVGB_REQUIRE(ws_bytes >= L.bytes, "plan workspace too small: %zu < %zu", ws_bytes, L.bytes);
  // a KV-cache plan serves every head: BH holds the cache rows (svgb200.h)
  write_plan(plan, s.split ? SVGB_PLAN_KVCACHE_SPLIT : SVGB_PLAN_KVCACHE, num_blocks * block_rows,
             s.varlen ? s.Sq : s.B * s.Sq, static_cast<int>(L.items), 0, s.block_causal ? MASK_BLOCK_CAUSAL : MASK_LOCAL,
             s.sink, s.block_causal ? a.m1 : a.left, s.block_causal ? s.window : a.right, static_cast<int>(a.I),
             static_cast<int64_t>(L.items_off), static_cast<int64_t>(L.chunks_off), static_cast<int64_t>(L.bytes));
  char* ws = static_cast<char*>(plan_ws);
  int* counts = reinterpret_cast<int*>(ws);
  int* kv = reinterpret_cast<int*>(ws + SVGB_PLAN_SEG_BOUNDS_OFF);
  int2* chunks = reinterpret_cast<int2*>(ws + L.chunks_off);
  int4* items = reinterpret_cast<int4*>(ws + L.items_off);
  const unsigned grid = static_cast<unsigned>((L.items + 7) / 8);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (s.varlen)
    kv_varlen_lists_kernel<<<grid, 256, 0, st>>>(cu_q, cache_seqlens, cu_new, cache_batch_idx, block_table, s.B, s.Sq,
                                                 static_cast<int>(a.I), num_blocks, block_rows, max_pages, cap,
                                                 static_cast<int>(L.slots), s.nsplit, s.sink, a.left, a.right, a.m1,
                                                 counts, kv, chunks, items);
  else
    kv_lists_kernel<<<grid, 256, 0, st>>>(cache_seqlens, cache_batch_idx, block_table, s.B, s.Sq, Snew, num_blocks,
                                          block_rows, max_pages, cap, static_cast<int>(L.slots), s.nsplit, s.sink,
                                          a.left, a.right, a.m1, counts, kv, chunks, items);
  SVGB_LAUNCH_OK();
  return 0;
}

extern "C" {

int svgb_kvcache_append(void* k_cache, void* v_cache, const void* k, const void* v, const int32_t* cache_seqlens,
                        const int32_t* cache_batch_idx, const int32_t* block_table, int dtype, int B, int Snew, int Hkv,
                        int D, int num_blocks, int block_rows, int max_pages, const long long* kc_strides,
                        const long long* vc_strides, const long long* k_strides, const long long* v_strides,
                        void* stream) {
  return kv_append_run(k_cache, v_cache, k, v, cache_seqlens, cache_batch_idx, block_table, dtype, B, Snew, Hkv, D,
                       num_blocks, block_rows, max_pages, kc_strides, vc_strides, k_strides, v_strides, nullptr,
                       nullptr, false, FMT_16BIT, stream, "svgb_kvcache_append");
}

int svgb_kvcache_append_e4m3(void* k_cache, void* v_cache, const void* k, const void* v, const int32_t* cache_seqlens,
                             const int32_t* cache_batch_idx, const int32_t* block_table, int dtype, int B, int Snew,
                             int Hkv, int D, int num_blocks, int block_rows, int max_pages, const long long* kc_strides,
                             const long long* vc_strides, const long long* k_strides, const long long* v_strides,
                             const float* k_scale, const float* v_scale, void* stream) {
  // the per-head scales are only read
  return kv_append_run(k_cache, v_cache, k, v, cache_seqlens, cache_batch_idx, block_table, dtype, B, Snew, Hkv, D,
                       num_blocks, block_rows, max_pages, kc_strides, vc_strides, k_strides, v_strides,
                       const_cast<float*>(k_scale), const_cast<float*>(v_scale), false, FMT_E4M3, stream,
                       "svgb_kvcache_append_e4m3");
}

int svgb_kvcache_append_e4m3_rows(void* k_cache, void* v_cache, const void* k, const void* v,
                                  const int32_t* cache_seqlens, const int32_t* cache_batch_idx,
                                  const int32_t* block_table, int dtype, int B, int Snew, int Hkv, int D,
                                  int num_blocks, int block_rows, int max_pages, const long long* kc_strides,
                                  const long long* vc_strides, const long long* k_strides, const long long* v_strides,
                                  float* k_scale, float* v_scale, void* stream) {
  return kv_append_run(k_cache, v_cache, k, v, cache_seqlens, cache_batch_idx, block_table, dtype, B, Snew, Hkv, D,
                       num_blocks, block_rows, max_pages, kc_strides, vc_strides, k_strides, v_strides, k_scale,
                       v_scale, true, FMT_E4M3_ROWS, stream, "svgb_kvcache_append_e4m3_rows");
}

int svgb_kvcache_append_varlen(void* k_cache, void* v_cache, const void* k, const void* v, const int32_t* cu_new,
                               const int32_t* cache_seqlens, const int32_t* cache_batch_idx,
                               const int32_t* block_table, int dtype, int B, int total_new, int Hkv, int D,
                               int num_blocks, int block_rows, int max_pages, const long long* kc_strides,
                               const long long* vc_strides, const long long* k_strides, const long long* v_strides,
                               float* k_scale, float* v_scale, int row_scales, void* stream) {
  const char* who = "svgb_kvcache_append_varlen";
  SVGB_REQUIRE(cu_new, "%s needs cu_new (device int32 [B + 1], the new rows of each stream)", who);
  SVGB_REQUIRE(B > 0, "%s: bad stream count B=%d", who, B);
  return kv_append_run(k_cache, v_cache, k, v, cache_seqlens, cache_batch_idx, block_table, dtype, B, total_new, Hkv, D,
                       num_blocks, block_rows, max_pages, kc_strides, vc_strides, k_strides, v_strides, k_scale, v_scale,
                       row_scales != 0, FMT_16BIT | FMT_E4M3 | FMT_E4M3_ROWS, stream, who, cu_new);
}

// the spec of each planner: B, Sq, max_q, varlen, sink, left, right, block_causal, window, block, first_block, nsplit,
// split
int svgb_attn_plan_kvcache_bytes(int B, int Sq, int cap, int sink, int left, int right, size_t* bytes) {
  return kv_plan_bytes({B, Sq, 0, false, sink, left, right, false, 0, 0, 0, 1, false}, cap, bytes,
                       "svgb_attn_plan_kvcache_bytes");
}

int svgb_attn_plan_kvcache(const int32_t* cache_seqlens, const int32_t* cache_batch_idx, const int32_t* block_table,
                           int B, int Sq, int Snew, int num_blocks, int block_rows, int max_pages, int sink, int left,
                           int right, void* plan_ws, size_t ws_bytes, svgb_plan* plan, void* stream) {
  return kv_plan({B, Sq, 0, false, sink, left, right, false, 0, 0, 0, 1, false}, nullptr, cache_seqlens, nullptr, Snew,
                 cache_batch_idx, block_table, num_blocks, block_rows, max_pages, plan_ws, ws_bytes, plan, stream,
                 "svgb_attn_plan_kvcache");
}

int svgb_attn_plan_kvcache_split_bytes(int B, int Sq, int cap, int sink, int left, int right, int num_splits,
                                       size_t* bytes) {
  return kv_plan_bytes({B, Sq, 0, false, sink, left, right, false, 0, 0, 0, num_splits, true}, cap, bytes,
                       "svgb_attn_plan_kvcache_split_bytes");
}

int svgb_attn_plan_kvcache_split(const int32_t* cache_seqlens, const int32_t* cache_batch_idx,
                                 const int32_t* block_table, int B, int Sq, int Snew, int num_blocks, int block_rows,
                                 int max_pages, int sink, int left, int right, int num_splits, void* plan_ws,
                                 size_t ws_bytes, svgb_plan* plan, void* stream) {
  return kv_plan({B, Sq, 0, false, sink, left, right, false, 0, 0, 0, num_splits, true}, nullptr, cache_seqlens, nullptr,
                 Snew, cache_batch_idx, block_table, num_blocks, block_rows, max_pages, plan_ws, ws_bytes, plan, stream,
                 "svgb_attn_plan_kvcache_split");
}

int svgb_attn_plan_kvcache_block_bytes(int B, int Sq, int cap, int sink, int window, int block, int first_block,
                                       int num_splits, size_t* bytes) {
  return kv_plan_bytes({B, Sq, 0, false, sink, 0, 0, true, window, block, first_block, num_splits, num_splits > 1}, cap,
                       bytes, "svgb_attn_plan_kvcache_block_bytes");
}

int svgb_attn_plan_kvcache_block(const int32_t* cache_seqlens, const int32_t* cache_batch_idx,
                                 const int32_t* block_table, int B, int Sq, int Snew, int num_blocks, int block_rows,
                                 int max_pages, int sink, int window, int block, int first_block, int num_splits,
                                 void* plan_ws, size_t ws_bytes, svgb_plan* plan, void* stream) {
  return kv_plan({B, Sq, 0, false, sink, 0, 0, true, window, block, first_block, num_splits, num_splits > 1}, nullptr,
                 cache_seqlens, nullptr, Snew, cache_batch_idx, block_table, num_blocks, block_rows, max_pages, plan_ws,
                 ws_bytes, plan, stream, "svgb_attn_plan_kvcache_block");
}

int svgb_attn_plan_kvcache_varlen_bytes(int B, int total_q, int max_q, int cap, int sink, int left, int right,
                                        int window, int block, int first_block, int num_splits, size_t* bytes) {
  return kv_plan_bytes({B, total_q, max_q, true, sink, left, right, block != 0, window, block, first_block, num_splits,
                        num_splits > 1},
                       cap, bytes, "svgb_attn_plan_kvcache_varlen_bytes");
}

int svgb_attn_plan_kvcache_varlen(const int32_t* cu_q, const int32_t* cache_seqlens, const int32_t* cu_new,
                                  const int32_t* cache_batch_idx, const int32_t* block_table, int B, int total_q,
                                  int max_q, int num_blocks, int block_rows, int max_pages, int sink, int left,
                                  int right, int window, int block, int first_block, int num_splits, void* plan_ws,
                                  size_t ws_bytes, svgb_plan* plan, void* stream) {
  return kv_plan({B, total_q, max_q, true, sink, left, right, block != 0, window, block, first_block, num_splits,
                  num_splits > 1},
                 cu_q, cache_seqlens, cu_new, 0, cache_batch_idx, block_table, num_blocks, block_rows, max_pages,
                 plan_ws, ws_bytes, plan, stream, "svgb_attn_plan_kvcache_varlen");
}

}  // extern "C"
