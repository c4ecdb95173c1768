/* svgb200 — C ABI of the Hopper-native (H100, sm_90a) sparse video-DiT attention engine.
 *
 * The reference (svg-project/Sparse-VideoGen) has no FFI on this path: its boundary is the set of
 * Python operator signatures imported by svg/models/<m>/attention.py (hyvideo/attention.py:12-28)
 * and the svg/kernels/ops API.  This header is the boundary our own Python shim binds with ctypes;
 * each entry point names the reference operator it stands behind.  INTEGRATION.md shows the binding.
 *
 * Conventions
 *   - extern "C", plain pointers and sizes, no torch types.
 *   - every function returns 0 on success, <0 on error; svgb_last_error() returns a thread-local
 *     message for the last failure on the calling thread.
 *   - all data pointers are DEVICE pointers unless a parameter is documented "host".
 *   - no function allocates device memory or synchronises the device: the caller provides the
 *     workspace (sizes from the *_bytes queries) and the cudaStream_t (passed as void*).
 *   - integer outputs (labels, permutations, plans, maps) are bit-exact, deterministic.
 *   - dtype: SVGB_BF16 or SVGB_F16 for q/k/v/o (svgb_attn_fwd also takes SVGB_E4M3 inputs).
 */
#ifndef SVGB200_H_
#define SVGB200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SVGB_BF16 0
#define SVGB_F16 1
#define SVGB_E4M3 2 /* fp8 e4m3 q/k/v of svgb_attn_fwd (with per-head scales) */
#define SVGB_F32 3  /* fp32 storage (transformer-block glue ops only) */

/* element-mask families for the SVG1 band plan (reference generate_temporal_head_mask_mod) */
#define SVGB_MASK_NONE 0
#define SVGB_MASK_HY 1  /* hyvideo/utils.py:20-44  m0=F*P, m1=F*P+prompt_len, m2=W              */
#define SVGB_MASK_WAN 2 /* wan/utils.py:25-41      m0=P (first-frame sink), m2=W  (|q-kv| <= W) */
#define SVGB_MASK_COG 3 /* cog/utils.py:30-46      m0=first-col limit, m1=prompt_len, m2=W      */
/* SVG1 online-profiling masks (get_attention_mask), 128-token block band |bq - bk| < thres; m0=F, m1=P.
 * HY / WAN: m2=thres.  COG: m2=thres | ctx << 12 (thres < 4096).  See attn_common.cuh MaskMode. */
#define SVGB_MASK_PROF_HY_S 4   /* hyvideo/utils.py:47-93 spatial, text last (text rows / columns attend)   */
#define SVGB_MASK_PROF_HY_T 5   /* ... temporal (token-major order)                                      */
#define SVGB_MASK_PROF_WAN_S 6  /* wan/utils.py:63-110 spatial, first-frame sink                          */
#define SVGB_MASK_PROF_WAN_T 7  /* ... temporal                                                           */
#define SVGB_MASK_PROF_COG_S 8  /* cog/utils.py:61-88 spatial, text first (text rows / columns attend)    */
#define SVGB_MASK_PROF_COG_T 9  /* ... temporal, video x video only (text rows / columns see nothing)     */
/* Local band with attention sinks: m0 = sink, m1 = left, m2 = right, all >= 0 (so every row keeps its diagonal key).
 *   allowed(q, kv) = (kv < sink) | ((q - kv <= left) & (kv - q <= right))
 * Causal attention is (0, S, 0); FlashAttention's window_size = (l, r) is (0, l, r) with -1 taken as S; a streaming
 * sink-plus-window is (sink, l, 0).  SVGB_MASK_WAN(P, W) is SVGB_MASK_LOCAL(P, W, W).  Forward and backward. */
#define SVGB_MASK_LOCAL 10
/* Block-causal mask of autoregressive video (chunk-wise causal attention, CausVid / Self-Forcing).  Positions form blocks
 * of C >= 1 whose ends lie at F, F + C, F + 2C, ... with 1 <= F <= C (a shorter first block: F < C); e(p) is the first
 * block end greater than p.  With a window W >= C (W >= S: unbounded) and a sink >= 0:
 *   allowed(q, kv) = (kv < sink) | (e(q) - W <= kv < e(q))
 * m0 = sink, m1 = SVGB_BLOCK_M1(C, F) (C < 2^16), m2 = W.  Every row sees its whole block and all earlier ones (within
 * the window); C = 1 is SVGB_MASK_LOCAL(sink, W - 1, 0).  The band planners refuse C < 1, F outside [1, C], W < C and a
 * negative sink by name.  Forward and backward.  Mode 11 is unassigned. */
#define SVGB_MASK_BLOCK_CAUSAL 12
#define SVGB_BLOCK_M1(C, F) ((C) | ((C) - (F)) << 16)

/* ---- library ---------------------------------------------------------------------------- */
int svgb_version(void);
const char* svgb_last_error(void);
/* 0 iff the current CUDA device is sm_90 (H100); fills optional outputs */
int svgb_device_check(int* sm_major, int* sm_minor, int* num_sms);

/* ---- attention plans -------------------------------------------------------------------- */
/* Host-side descriptor of a device-resident plan (filled by the plan functions, read by
 * svgb_attn_fwd).  Plain data; copyable. */
#define SVGB_PLAN_VARBLOCK 1 /* variable-block map, TMA chunks (svgb_attn_plan_varblock) */
#define SVGB_PLAN_BAND 2     /* element-exact band mask (svgb_attn_plan_band) */
#define SVGB_PLAN_GATHER 3   /* variable-block map, row gather (svgb_attn_plan_varblock_gather) */
#define SVGB_PLAN_BAND_T 4   /* key-major band plan of the backward pass (svgb_attn_plan_band_t) */
#define SVGB_PLAN_SEG 5      /* local mask inside packed variable-length segments (svgb_attn_plan_local_varlen) */
#define SVGB_PLAN_SEG_T 6    /* its key-major companion for the backward (svgb_attn_plan_local_varlen_t) */
#define SVGB_PLAN_KVCACHE 7  /* local mask into a contiguous or paged KV cache, forward only (svgb_attn_plan_kvcache) */
#define SVGB_PLAN_KVCACHE_SPLIT 8 /* the same, split across the keys (svgb_attn_plan_kvcache_split) */
typedef struct svgb_plan {
  int32_t kind;          /* SVGB_PLAN_* */
  int32_t BH, S;
  int32_t max_items;     /* grid.x of the attention launch */
  int32_t items_stride;  /* 0 when one plan serves every head */
  int32_t mask_mode, m0, m1, m2;
  int32_t varlen_items;  /* KV-cache plans of svgb_attn_plan_kvcache_varlen: items per split (> 0); 0 otherwise */
  int64_t counts_off, items_off, chunks_off; /* byte offsets inside the plan workspace */
  int64_t bytes;
} svgb_plan;
/* A plan built with BH == 1 may serve every head of a launch (one map for all heads, e.g. BSR masks):
 * set items_stride = 0 in the host struct. */
/* S is the query length.  A variable-block plan has no element mask (mask_mode = SVGB_MASK_NONE), and its m0 holds the
 * key/value length Skv when svgb_attn_plan_varblock_kv built it; m0 = 0 (every other planner) means Skv = S.  The
 * attention entries reject a plan whose lengths differ from the call's.  A segment plan (SVGB_PLAN_SEG / _SEG_T) serves
 * every head (items_stride = 0), so its BH holds its key/value length instead (key-major: the query length); its
 * segment count and its copy of the bounds are in its workspace, int32 {nseg, cu_q[0..nseg], cu_k[0..nseg]} at byte
 * SVGB_PLAN_SEG_BOUNDS_OFF. */
#define SVGB_PLAN_SEG_BOUNDS_OFF 16

/* SVG2 / BSR / dense: q-block i of head h attends k-block j iff map[h,i,j] != 0.
 * Stands behind dynamic_block_sparse_fwd_flashinfer's wrapper.plan (svg/kmeans_utils.py:1355-1385).
 *   map    uint8 [BH, QC, KC]     row_sz int32 [BH, QC]     col_sz int32 [BH, KC]
 * Each head's row sizes and col sizes must sum to S (not checked on device). */
int svgb_attn_plan_varblock_bytes(int BH, int S, int QC, int KC, size_t* bytes);
int svgb_attn_plan_varblock(const uint8_t* map, const int32_t* row_sz, const int32_t* col_sz, int BH,
                            int S, int QC, int KC, void* plan_ws, size_t ws_bytes, svgb_plan* plan,
                            void* stream);

/* Rectangular form, for queries attending a key/value sequence of another length (cross-attention, a chunk of frames
 * against context frames): row sizes sum to Sq, column sizes to Skv; the items cover Sq query rows and the chunk lists
 * Skv keys.  plan->kind = SVGB_PLAN_VARBLOCK, plan->S = Sq, plan->m0 = Skv; runs with svgb_attn_fwd_kv / svgb_attn_bwd_kv.
 * Its key-major companion for the backward is the same planner on the transpose: (map^T, col_sz, row_sz, Skv, Sq). */
int svgb_attn_plan_varblock_kv_bytes(int BH, int Sq, int Skv, int QC, int KC, size_t* bytes);
int svgb_attn_plan_varblock_kv(const uint8_t* map, const int32_t* row_sz, const int32_t* col_sz, int BH, int Sq,
                               int Skv, int QC, int KC, void* plan_ws, size_t ws_bytes, svgb_plan* plan,
                               void* stream);

/* Same map, lowered for the row-gather kernel path: the selected key ranges are kept as runs and the
 * kernel gathers exactly-full 128-key chunks across run boundaries with cp.async (no padded tail chunk per
 * run), optionally through row-index vectors (q_rows / kv_rows of svgb_attn_fwd) so the cluster permutation of Q, K, V
 * (permute_tensor_by_labels_triton x3, svg/models/hyvideo/attention.py:651-653) never materialises. */
int svgb_attn_plan_varblock_gather(const uint8_t* map, const int32_t* row_sz, const int32_t* col_sz, int BH,
                                   int S, int QC, int KC, void* plan_ws, size_t ws_bytes, svgb_plan* plan,
                                   void* stream);

/* SVG1: one element-exact band mask shared by every head.  Stands behind prepare_flexattention /
 * create_block_mask (svg/models/hyvideo/attention.py:527-551), and, with SVGB_MASK_LOCAL, behind causal and
 * sliding-window attention (a negative sink, left or right is an error).  Items are issued heaviest first: under
 * SVGB_MASK_LOCAL with left > right the query-major plan lists its items from the last rows back, and with right > left
 * the key-major plan does; SVGB_MASK_BLOCK_CAUSAL is issued as its local band (sink, W - 1, 0). */
int svgb_attn_plan_band_bytes(int S, size_t* bytes);
int svgb_attn_plan_band(int mask_mode, int m0, int m1, int m2, int BH, int S, void* plan_ws,
                        size_t ws_bytes, svgb_plan* plan, void* stream);

/* Key-major form of the same band mask, for svgb_attn_bwd: its items are key ranges and its chunk lists the query ranges
 * that reach them, voted with mask_allowed(mode, query, key) exactly as the query-major plan votes.  Same parameters and
 * workspace size as svgb_attn_plan_band; plan->kind = SVGB_PLAN_BAND_T. */
int svgb_attn_plan_band_t_bytes(int S, size_t* bytes);
int svgb_attn_plan_band_t(int mask_mode, int m0, int m1, int m2, int BH, int S, void* plan_ws,
                          size_t ws_bytes, svgb_plan* plan, void* stream);

/* Local mask inside packed variable-length segments (FlashAttention's flash_attn_varlen_func with causal= /
 * window_size=), one plan shared by every head.  cu_q, cu_k: device int32 [nseg + 1], query segment i = rows
 * [cu_q[i], cu_q[i+1]) of length Lq_i, key segment i = keys [cu_k[i], cu_k[i+1]) of length Lk_i.  With qi, kj the
 * positions inside segment i and off_i = Lk_i - Lq_i (bottom-right alignment):
 *   allowed(q, kv) = same segment & (kj < sink | ((qi + off_i) - kj <= left & kj - (qi + off_i) <= right))
 * sink, left, right >= 0 (a negative one is an error); causal is right = 0.  With nseg = 1 and Sq == Skv this is
 * SVGB_MASK_LOCAL(sink, left, right) and the results are svgb_attn_plan_band's, bit for bit.  A row without an allowed
 * key gets o = 0, lse = -inf, dq = 0; a key no row reaches dk = dv = 0.  Empty segments are legal.
 * The planner copies the bounds into the workspace (the plan owns them) and reads nothing on the host: the item count
 * stays on the device, plan->max_items is a host bound.  The first bound is taken as 0 and the last as Sq (Skv), the
 * others are clamped to [0, Sq] ([0, Skv]) and made monotone (running maximum), so bounds out of range or out of order
 * give an unspecified result that stays inside the tensors.  No stream straddles a query segment and no chunk a key
 * segment (chunks start at cu_k[i] + 128 j); each chunk is FULL, ELEM or omitted, classified from the band's interval
 * form.  Items are issued in row order (segments in turn).
 * plan->kind = SVGB_PLAN_SEG, mask_mode = SVGB_MASK_LOCAL, m0..m2 = sink, left, right, S = Sq, BH = Skv.  Runs
 * with svgb_attn_fwd (Sq == Skv), _kv, _gqa and _strided, 16-bit inputs only (no e4m3, gather plans or row vectors).
 * Workspace (one size for the plan and its key-major companion; integer division, n = nseg):
 *   I = max over R in {Sq, Skv} of min(R, (R + 510 n) / 256)            items (at most one partial item per segment,
 *                                                                       key-major two)
 *   C = min(I * ceil(max(Sq, Skv) / 128), (Sq Skv + 510 (Sq + Skv) + 64770 n) / 32768)    chunk slots
 *   bytes = 16 + align16(4 (2 n + 3)) + align16(8 (n + 1)) + 32 I + 8 C
 * which depends on nseg, Sq and Skv only; at n = 1 and Sq == Skv == S it never exceeds svgb_attn_plan_band_bytes(S).
 * Sq, Skv > 0. */
int svgb_attn_plan_local_varlen_bytes(int nseg, int Sq, int Skv, size_t* bytes);
int svgb_attn_plan_local_varlen(const int32_t* cu_q, const int32_t* cu_k, int nseg, int Sq, int Skv, int sink, int left,
                                int right, void* plan_ws, size_t ws_bytes, svgb_plan* plan, void* stream);
/* Key-major companion for svgb_attn_bwd*: items are key ranges of one key segment (the sink keys of a segment form
 * items of their own), chunks the query ranges of that segment that reach them.  Same arguments and workspace size;
 * plan->kind = SVGB_PLAN_SEG_T, S = Skv, BH = Sq.  The backward checks that plan and plan_t have swapped lengths, the
 * same parameters and the same workspace layout (which is a function of nseg, Sq and Skv). */
int svgb_attn_plan_local_varlen_t(const int32_t* cu_q, const int32_t* cu_k, int nseg, int Sq, int Skv, int sink,
                                  int left, int right, void* plan_ws, size_t ws_bytes, svgb_plan* plan, void* stream);
/* Block-causal mask inside packed variable-length segments (chunk-wise causal video training on a batch of clips of
 * different lengths): the segments, bounds, alignment and plans of svgb_attn_plan_local_varlen, with SVGB_MASK_BLOCK_CAUSAL
 * inside every segment and its block grid anchored at the segment's key 0.  With kj the key's and p = qi + Lk_i - Lq_i
 * the query's position in segment i, and e(p) the first block end (F, F + C, F + 2C, ...) past p (p < F, negative p
 * too: F):
 *   allowed(q, kv) = same segment & (kj < sink | e(p) - W <= kj < e(p))
 * window = W >= C (W >= the longest segment + C: unbounded), block = C in [1, 2^16), first_block = F in [1, C],
 * sink >= 0, each refused by name before any launch.  A pair of entries of their own, so the _local_varlen signatures
 * stay as they are.  plan->kind = SVGB_PLAN_SEG (SVGB_PLAN_SEG_T for the key-major companion), mask_mode =
 * SVGB_MASK_BLOCK_CAUSAL, m0..m2 = sink, SVGB_BLOCK_M1(C, F), W; they run wherever the _local_varlen plans run, forward
 * and backward.  Query-major items round their first and last positions to their block ends inside the segment and
 * classify chunks as the local band (sink, W - 1, 0); key-major items classify them from the interval of positions that
 * reach each key.  Workspace: svgb_attn_plan_local_varlen_bytes (an item has one slot per chunk of its segment whatever
 * the mask). */
int svgb_attn_plan_block_varlen(const int32_t* cu_q, const int32_t* cu_k, int nseg, int Sq, int Skv, int sink,
                                int window, int block, int first_block, void* plan_ws, size_t ws_bytes, svgb_plan* plan,
                                void* stream);
int svgb_attn_plan_block_varlen_t(const int32_t* cu_q, const int32_t* cu_k, int nseg, int Sq, int Skv, int sink,
                                  int window, int block, int first_block, void* plan_ws, size_t ws_bytes,
                                  svgb_plan* plan, void* stream);

/* ---- KV cache (FlashAttention's flash_attn_with_kvcache) ----------------------------------
 * A batch of B streams attends into a cache of num_blocks blocks of block_rows rows, Hkv heads, D in {64, 128}:
 *   contiguous : k_cache, v_cache [B_cache, S_cache, Hkv, D] (num_blocks = B_cache, block_rows = S_cache, block_table
 *                NULL); stream b lives in block cache_batch_idx[b] (NULL: block b).  Capacity S_cache.
 *   paged      : k_cache, v_cache [num_pages, page_size, Hkv, D] (num_blocks = num_pages, block_rows = page_size, a
 *                multiple of 128, so no 128-key chunk straddles two pages) and block_table int32 [B, max_pages]: logical
 *                key t of stream b is row t % page_size of page block_table[b, t / page_size].  Capacity
 *                max_pages * page_size; cache_batch_idx must be NULL.
 * cache_seqlens: device int32 [B], the keys each stream holds before the append.  Nothing is read on the host.
 * Bad input never makes a kernel touch memory outside the tensors, and gives an unspecified result: a length is clamped
 * to [0, capacity], a block or page index to [0, num_blocks), and the append skips rows whose key or block falls
 * outside the cache.  A stream's capacity is at most 2^29 keys and num_blocks * block_rows < 2^31.
 *
 * Append: k, v [B, Snew, Hkv, D] (Snew > 0) are written at logical keys cache_seqlens[b] .. cache_seqlens[b] + Snew - 1
 * of each stream; nothing else is written.  One launch for K and V, 16-byte vectors.  Strides {batch or block, head,
 * row} in elements per tensor, nonzero multiples of 8; bases 16-byte aligned; 16-bit dtypes. */
int svgb_kvcache_append(void* k_cache, void* v_cache, const void* k, const void* v, const int32_t* cache_seqlens,
                        const int32_t* cache_batch_idx, const int32_t* block_table, int dtype, int B, int Snew, int Hkv,
                        int D, int num_blocks, int block_rows, int max_pages, const long long* kc_strides,
                        const long long* vc_strides, const long long* k_strides, const long long* v_strides,
                        void* stream);
/* Append into an e4m3 cache (FP8 KV cache): svgb_kvcache_append's arguments, with dtype the 16-bit (SVGB_BF16 / SVGB_F16)
 * type of the new rows k, v and the caches e4m3 bytes, plus k_scale, v_scale: device float [Hkv], one dequantisation
 * scale per key/value head for the cache's lifetime (cache element ~= e4m3 * scale[h]).  Each new element is written as
 * RN-satfinite(x * (1 / scale[h])), the conversion of svgb_quantize_e4m3, so a value past 448 * scale saturates to
 * +-448; the scales are not checked on the device.  One launch for K and V; nothing else is written.  The cache strides
 * (in elements, i.e. bytes) must be multiples of 16, as the attention's TMA maps need; the new rows' strides follow
 * svgb_kvcache_append.  Rows past a stream's length must be finite here too, and 0x7F / 0xFF are e4m3 NaN: allocate
 * the cache with zeros. */
int svgb_kvcache_append_e4m3(void* k_cache, void* v_cache, const void* k, const void* v, const int32_t* cache_seqlens,
                             const int32_t* cache_batch_idx, const int32_t* block_table, int dtype, int B, int Snew,
                             int Hkv, int D, int num_blocks, int block_rows, int max_pages, const long long* kc_strides,
                             const long long* vc_strides, const long long* k_strides, const long long* v_strides,
                             const float* k_scale, const float* v_scale, void* stream);
/* Append into an e4m3 cache with per-row scales (the per-row FP8 KV cache): svgb_kvcache_append_e4m3's arguments with
 * D = 128, where k_scale, v_scale are device float [num_blocks, Hkv, block_rows], contiguous and 16-byte aligned
 * (block_rows a multiple of 4): scale [blk, h, row] belongs to cache row `row` of block `blk`, head h, and the append
 * writes it.  A new row x (one position of one head, 128 values) with a = max|x| gets s = 2^e, e the smallest integer
 * with a <= 448 * 2^e, clamped to [-126, 127] (a = 0: e = 0), and its elements are stored as RN(x * 2^-e) in e4m3, so
 * nothing saturates and an overwrite computes a fresh scale.  Only the new rows and their scales are written, under
 * svgb_kvcache_append's skip rules; a row with a non-finite value is unspecified.  Allocate the scale tensors with
 * finite values (e.g. ones): rows past a stream's length in its last chunk are loaded and masked, like the cache bytes. */
int svgb_kvcache_append_e4m3_rows(void* k_cache, void* v_cache, const void* k, const void* v,
                                  const int32_t* cache_seqlens, const int32_t* cache_batch_idx,
                                  const int32_t* block_table, int dtype, int B, int Snew, int Hkv, int D,
                                  int num_blocks, int block_rows, int max_pages, const long long* kc_strides,
                                  const long long* vc_strides, const long long* k_strides, const long long* v_strides,
                                  float* k_scale, float* v_scale, void* stream);
/* Plan: stream b has L_b = min(cache_seqlens[b] + Snew, capacity) keys at logical positions 0 .. L_b - 1 (Snew: rows
 * appended before this attention), and Sq queries, query i at logical position L_b - Sq + i (FlashAttention's
 * bottom-right alignment).  Query p sees key kv when kv < sink, or when p - kv <= left and kv - p <= right (causal:
 * right = 0); all three >= 0.  A row without an allowed key gets o = 0 and lse = -inf.
 * The queries are the packed rows [B * Sq, Hq, D] (query i of stream b is row b Sq + i); k and v are the cache viewed as
 * num_blocks * block_rows rows.  Runs with svgb_attn_fwd_gqa and svgb_attn_fwd_strided (B = 1 at the ABI, Sq = B * Sq
 * rows, Skv = num_blocks * block_rows rows), 16-bit inputs, and with svgb_attn_fwd_strided_e4m3 on an e4m3 cache; no
 * backward, row vectors or gather.
 * One launch, one warp per item: a stream's queries are cut into items of 256 rows from its first row, and each item
 * visits only the chunks of its sinks and of its window (the pages behind a window are not read, so pages evicted from
 * behind a window may be recycled as long as the sink pages are kept).  Chunks are 128 logical keys from position 0,
 * FULL, ELEM or omitted; a kept chunk records the physical row its TMA box loads from and its logical index (mask
 * positions).  The 128 - valid rows after a stream's last key in its last chunk are loaded and masked, so they must hold
 * finite values (any cache allocated with zeros, or rows written earlier, qualifies).
 * plan->kind = SVGB_PLAN_KVCACHE, mask_mode = SVGB_MASK_LOCAL, m0..m2 = sink, left, right, S = B * Sq,
 * BH = num_blocks * block_rows (one plan for every head); the workspace keeps int32 {B, Sq, L_0 .. L_B-1} at byte
 * SVGB_PLAN_SEG_BOUNDS_OFF.
 * Workspace (integer division; cap = the capacity, I = B ceil(Sq / 256) items):
 *   slots = min(ceil(cap / 128), ceil(sink / 128) + (255 + left + right) / 128 + 2)   chunk slots per item
 *   bytes = 16 + align16(4 (B + 2)) + 32 I + 8 I slots
 * which depends on host-known sizes only. */
int svgb_attn_plan_kvcache_bytes(int B, int Sq, int cap, int sink, int left, int right, size_t* bytes);
int svgb_attn_plan_kvcache(const int32_t* cache_seqlens, const int32_t* cache_batch_idx, const int32_t* block_table,
                           int B, int Sq, int Snew, int num_blocks, int block_rows, int max_pages, int sink, int left,
                           int right, void* plan_ws, size_t ws_bytes, svgb_plan* plan, void* stream);
/* Split across the keys (split-KV, for decode and short chunks, where B ceil(Sq / 256) Hq CTAs leave SMs idle):
 * svgb_attn_plan_kvcache's arguments plus num_splits = n >= 1.  The plan has n B ceil(Sq / 256) items, split-major: item
 * s B I + i is split s of the single plan's item i, and visits the s-th piece of ceil(nvis / n) of that item's nvis
 * visited chunks (sinks first, then the window), classified and compacted as the single plan's, so the split lists of
 * an item concatenated in split order are its single-pass list chunk for chunk; splits past the last piece are empty.
 * plan->kind = SVGB_PLAN_KVCACHE_SPLIT, max_items = n B ceil(Sq / 256), every other field and the {B, Sq, L_b} header as
 * svgb_attn_plan_kvcache.  Workspace: svgb_attn_plan_kvcache_bytes's with I' = n I items of ceil(slots / n) slots:
 *   bytes = 16 + align16(4 (B + 2)) + 32 I' + 8 I' ceil(slots / n).
 * Runs on svgb_attn_fwd_kvcache_split only; every other attention entry and the backward refuse it by name. */
int svgb_attn_plan_kvcache_split_bytes(int B, int Sq, int cap, int sink, int left, int right, int num_splits,
                                       size_t* bytes);
int svgb_attn_plan_kvcache_split(const int32_t* cache_seqlens, const int32_t* cache_batch_idx,
                                 const int32_t* block_table, int B, int Sq, int Snew, int num_blocks, int block_rows,
                                 int max_pages, int sink, int left, int right, int num_splits, void* plan_ws,
                                 size_t ws_bytes, svgb_plan* plan, void* stream);
/* Block-causal KV-cache plan (SVGB_MASK_BLOCK_CAUSAL on logical positions, query i of stream b at L_b - Sq + i): the
 * arguments of svgb_attn_plan_kvcache_split with (window, block, first_block) = (W, C, F) in place of (left, right).
 * When the Sq queries of a call form one block (F chosen so that a block ends at L_b), they all attend
 * [L_b - W, L_b) plus the sinks.  Refuses C outside [1, 2^16), F outside [1, C], W < C, a negative sink and
 * num_splits < 1 by name.  num_splits = 1 is a single plan (plan->kind = SVGB_PLAN_KVCACHE, run as
 * svgb_attn_plan_kvcache's), n > 1 a split plan (SVGB_PLAN_KVCACHE_SPLIT, run as svgb_attn_plan_kvcache_split's);
 * mask_mode = SVGB_MASK_BLOCK_CAUSAL, m0..m2 = sink, SVGB_BLOCK_M1(C, F), W.  Each item visits the chunks of its sinks
 * and of [e(p0) - W, e(p1) - 1] for its first and last positions p0, p1.  Workspace: the _bytes of
 * svgb_attn_plan_kvcache_split (of svgb_attn_plan_kvcache at n = 1) with left = W - 1 and right = C - 1. */
int svgb_attn_plan_kvcache_block_bytes(int B, int Sq, int cap, int sink, int window, int block, int first_block,
                                       int num_splits, size_t* bytes);
int svgb_attn_plan_kvcache_block(const int32_t* cache_seqlens, const int32_t* cache_batch_idx,
                                 const int32_t* block_table, int B, int Sq, int Snew, int num_blocks, int block_rows,
                                 int max_pages, int sink, int window, int block, int first_block, int num_splits,
                                 void* plan_ws, size_t ws_bytes, svgb_plan* plan, void* stream);
/* Variable-length queries and appends (FlashAttention 3's cu_seqlens_q / cu_seqlens_k_new): B streams, each with its own
 * query count, in one plan.  cu_q: device int32 [B + 1], stream b's Lq_b = cu_q[b+1] - cu_q[b] queries are the packed
 * rows [cu_q[b], cu_q[b+1]) of q [total_q, Hq, D] (Lq_b = 0 is legal).  cu_new: optional device int32 [B + 1], stream b
 * appended Lnew_b = cu_new[b+1] - cu_new[b] rows before this attention (svgb_kvcache_append_varlen); NULL: none.  Stream
 * b has L_b = min(cache_seqlens[b] + Lnew_b, capacity) keys and its query i sits at L_b - Lq_b + i (Lq_b > L_b puts
 * queries at negative positions).  Mask: block = 0 is svgb_attn_plan_kvcache's local band (sink, left, right; window
 * and first_block must be 0), block = C > 0 svgb_attn_plan_kvcache_block's (sink, window = W, block = C, first_block =
 * F; left and right must be 0), one (C, F) for the batch.  With every Lq_b = Sq and Lnew_b = Snew the results are the
 * uniform plan's, bit for bit.  A row without an allowed key gets o = 0 and lse = -inf.  Nothing is read on the host:
 * the bounds are clamped to [0, total_q] on the device, and bounds out of order give an unspecified result that stays
 * inside the tensors.  total_q >= 1 and max_q in [1, total_q] are host values: max_q bounds every Lq_b (pass total_q
 * when unknown; a longer stream gives an unspecified result).
 * One launch, one warp per item.  Items are 256 rows cut from each stream's first row, numbered stream after stream;
 * their count is known on the device only, and the host bound per split is
 *   I = min(B ceil(max_q / 256), (total_q + 255 B) / 256)
 * (sum ceil(Lq_b / 256) <= (total_q + 255 B) / 256).  num_splits = n: n = 1 is a single plan (SVGB_PLAN_KVCACHE), n > 1
 * a split plan (SVGB_PLAN_KVCACHE_SPLIT), split-major, item s I + i being split s of item i as in
 * svgb_attn_plan_kvcache_split.  Items i past the streams' items have zero rows and an empty list: their CTAs write
 * nothing.  plan->S = total_q, max_items = n I, varlen_items = I, every other field as the uniform plans'.  The
 * workspace keeps the header int32 {B, -1, L_0 .. L_B-1, cq_0 .. cq_B} at SVGB_PLAN_SEG_BOUNDS_OFF (cq_b the clamped
 * bounds; -1 in the Sq slot marks it), from which the forward finds a row's stream by binary search.
 * Runs wherever the uniform plans run, on q [total_q, Hq, D] as B = 1 and Sq = total_q at the ABI:
 * svgb_attn_fwd_strided (16-bit, GQA), svgb_attn_fwd_strided_e4m3 (per-head e4m3), svgb_attn_fwd_kvcache_e4m3_rows
 * (per-row e4m3) and, split, svgb_attn_fwd_kvcache_split in every format, which takes I from plan->varlen_items.
 * Workspace (integer division; slots as svgb_attn_plan_kvcache_bytes, with left = W - 1 and right = C - 1 for a
 * block-causal plan):
 *   bytes = 16 + align16(4 (2 B + 3)) + 32 n I + 8 n I ceil(slots / n)
 * Refused by name: B < 1, total_q < 1, max_q outside [1, total_q], num_splits < 1, the mask arguments of the other form,
 * and bad sink, left, right, W, C or F. */
int svgb_attn_plan_kvcache_varlen_bytes(int B, int total_q, int max_q, int cap, int sink, int left, int right,
                                        int window, int block, int first_block, int num_splits, size_t* bytes);
int svgb_attn_plan_kvcache_varlen(const int32_t* cu_q, const int32_t* cache_seqlens, const int32_t* cu_new,
                                  const int32_t* cache_batch_idx, const int32_t* block_table, int B, int total_q,
                                  int max_q, int num_blocks, int block_rows, int max_pages, int sink, int left,
                                  int right, int window, int block, int first_block, int num_splits, void* plan_ws,
                                  size_t ws_bytes, svgb_plan* plan, void* stream);
/* Variable-length append, every cache format in one entry: new rows k, v [total_new, Hkv, D] (strides {batch, head, row},
 * the batch stride not stepped) where stream b's rows are [cu_new[b], cu_new[b+1]) (device int32 [B + 1]), written at
 * its logical keys cache_seqlens[b] .. + Lnew_b - 1 under svgb_kvcache_append's skip rules; a row outside every stream
 * is not written.  k_scale = v_scale = NULL: a 16-bit cache (svgb_kvcache_append); row_scales = 0 with k_scale, v_scale
 * float [Hkv]: an e4m3 cache with per-head scales (svgb_kvcache_append_e4m3); row_scales = 1 with k_scale, v_scale float
 * [num_blocks, Hkv, block_rows]: per-row scales the append writes (svgb_kvcache_append_e4m3_rows).  One launch;
 * total_new > 0.  With every Lnew_b = Snew it writes what the uniform append writes. */
int svgb_kvcache_append_varlen(void* k_cache, void* v_cache, const void* k, const void* v, const int32_t* cu_new,
                               const int32_t* cache_seqlens, const int32_t* cache_batch_idx,
                               const int32_t* block_table, int dtype, int B, int total_new, int Hkv, int D,
                               int num_blocks, int block_rows, int max_pages, const long long* kc_strides,
                               const long long* vc_strides, const long long* k_strides, const long long* v_strides,
                               float* k_scale, float* v_scale, int row_scales, void* stream);

/* ---- attention -------------------------------------------------------------------------- */
/* o = softmax(q k^T * sm_scale  [masked by plan]) v, per head.  Stands behind
 * dynamic_block_sparse_fwd_flashinfer (svg/kmeans_utils.py:1319-1392), flex_attention under the
 * SVG1 BlockMask (hyvideo/attention.py:401-403), the BSR ops (svg/kernels/ops/attention_ops.py:
 * 140-197) and the dense fall-backs.
 *   q,k,v : [BH, S, D] with explicit strides (elements): element (h,s,d) at h*head_stride +
 *           s*row_stride + d.  [B,H,S,D] contiguous: row_stride=D, head_stride=S*D.
 *           [S,H,D]: row_stride=H*D, head_stride=D.   D in {64,128}; base pointers 16-B aligned,
 *           strides multiples of 8 elements.
 *   o     : same addressing with its own strides; 16-byte aligned, strides multiples of 8 elements.
 *   o_rows: optional int32 [BH,S]; when non-NULL output row for query row s is o_rows[h,s]
 *           (fuses apply_inverse_permutation_triton, svg/kernels/triton/permute.py:131-170).
 *   lse   : optional float [BH,S], natural-log log-sum-exp of the scaled scores.
 *   plan  : host pointer, any SVGB_PLAN_* kind.
 * Row gathers (SVGB_PLAN_GATHER only; NULL = identity): row r of the plan's (cluster-sorted) query order is read
 *   from q[h, q_rows[h,r]], key/value row r from k/v[h, kv_rows[h,r]], and written to o[h, o_rows[h,r]] — pass
 *   the argsort of the q-labels as q_rows AND o_rows and the argsort of the k-labels as kv_rows to run SVG2
 *   attention directly on the un-permuted tensors.  q_rows / kv_rows with another plan kind are an error.
 * FP8 (dtype SVGB_E4M3; BASELINE config 5, the reference has no FP8 sparse attention, README.md:117): q,k,v are
 *   e4m3 bytes (D = 128) with per-head dequantisation scales q_scale, k_scale, v_scale float [BH] (x ~= x8 *
 *   scale[h]), all three required; QK^T runs as e4m3 wgmma, each V tile is widened to fp16 in shared memory and
 *   PV runs in fp16 (P in fp16); o is bf16.  Per-head absmax scales do not change under a row permutation, so
 *   the scales of the un-permuted tensors serve row gathers too.  16-bit dtypes take no scales (pass NULL; o has
 *   the input dtype).  svgb_quantize_e4m3 produces the inputs: per-head absmax scaling (scale = absmax / 448),
 *   round-to-nearest, saturating. */
int svgb_attn_fwd(const void* q, const void* k, const void* v, const float* q_scale, const float* k_scale,
                  const float* v_scale, void* o, float* lse, const int32_t* q_rows, const int32_t* kv_rows,
                  const int32_t* o_rows, int dtype, int BH, int S, int D, long long row_stride,
                  long long head_stride, long long o_row_stride, long long o_head_stride, float sm_scale,
                  const svgb_plan* plan, const void* plan_ws, void* stream);
/* svgb_attn_fwd with queries of length Sq against keys / values of length Skv:
 *   q     : [BH, Sq, D] at q_row_stride / q_head_stride;  k, v : [BH, Skv, D] at kv_row_stride / kv_head_stride;
 *   o     : [BH, Sq, D] at its own strides;  lse : optional float [BH, Sq].
 *   plan  : SVGB_PLAN_VARBLOCK built for (Sq, Skv) -- svgb_attn_plan_varblock_kv, or svgb_attn_plan_varblock when
 *           Sq == Skv -- or SVGB_PLAN_SEG (svgb_attn_plan_local_varlen).  16-bit inputs only (SVGB_BF16 / SVGB_F16),
 *           D in {64,128}; alignment as svgb_attn_fwd.
 * Same kernel as svgb_attn_fwd: a key chunk past Skv is cut by its valid count and TMA fills rows past Skv with zeros.
 * Band, gather and profiling plans, row-index vectors and e4m3 inputs need Sq == Skv and svgb_attn_fwd.  With
 * Sq == Skv and equal strides the result is svgb_attn_fwd's, bit for bit. */
int svgb_attn_fwd_kv(const void* q, const void* k, const void* v, void* o, float* lse, int dtype, int BH, int Sq,
                     int Skv, int D, long long q_row_stride, long long q_head_stride, long long kv_row_stride,
                     long long kv_head_stride, long long o_row_stride, long long o_head_stride, float sm_scale,
                     const svgb_plan* plan, const void* plan_ws, void* stream);
/* Grouped-query attention (GQA; multi-query when BHkv = 1): svgb_attn_fwd_kv with fewer key/value heads than query
 * heads, FlashInfer's head mapping.
 *   q, o  : [BHq, Sq, D] at the q / o strides;  k, v : [BHkv, Skv, D] at the k/v strides;  lse : optional [BHq, Sq].
 *   BHq = G * BHkv: flattened query head h attends with key/value head h / G (for a batch of B, query head hq of batch
 *           element b is h = b * Hq + hq and reads head b * Hkv + hq / G).
 *   plan  : SVGB_PLAN_VARBLOCK built over the BHkv key/value heads (map [BHkv, QC, KC]; plan->BH = BHkv), shared by the
 *           G query heads of a group, rectangular (Sq != Skv) or not; or SVGB_PLAN_BAND (one work list for every head,
 *           Sq == Skv); or SVGB_PLAN_SEG (one work list for every head).
 * 16-bit inputs, D in {64,128}, alignment as svgb_attn_fwd; no gather plans, row vectors or e4m3 inputs.  The kernel
 * is svgb_attn_fwd's, so each output row is bit for bit the one of svgb_attn_fwd / _kv on K / V repeated G times per
 * head under the map repeated per query head. */
int svgb_attn_fwd_gqa(const void* q, const void* k, const void* v, void* o, float* lse, int dtype, int BHq, int BHkv,
                      int Sq, int Skv, int D, long long q_row_stride, long long q_head_stride, long long kv_row_stride,
                      long long kv_head_stride, long long o_row_stride, long long o_head_stride, float sm_scale,
                      const svgb_plan* plan, const void* plan_ws, void* stream);
/* Attention on strided [B, H, S, D] views: svgb_attn_fwd_gqa with a batch dimension and strides per tensor, so that
 * a transposed [B, S, H, D] projection, one third of a packed [B, S, 3, H, D] QKV, every other head or a batch slice is
 * read and written in place.
 *   q, o  : [B, Hq, Sq, D];  k, v : [B, Hkv, Skv, D];  lse : optional float [B * Hq, Sq], contiguous.
 *   x_strides : {batch, head, row} element strides of tensor x (the last dimension is contiguous), each a nonzero
 *           multiple of 8; bases 16-byte aligned.  Element (b, h, s, d) of x is at x + b*st[0] + h*st[1] + s*st[2] + d.
 *   Hq = G * Hkv: query head hq of batch element b attends with key/value head hq / G of b.
 *   plan  : SVGB_PLAN_VARBLOCK built over the B * Hkv key/value heads (flat head b * Hkv + hkv; rectangular or not),
 *           SVGB_PLAN_BAND (Sq == Skv) or SVGB_PLAN_SEG (every batch element segmented alike).
 * 16-bit inputs, D in {64,128}; no gather plans, row vectors or e4m3 inputs.  The TMA maps are 4-D (d, row, head,
 * batch) and o is stored at its own strides (only the view's elements are written); each output row is bit for bit
 * the one svgb_attn_fwd_gqa (svgb_attn_fwd / _kv when Hq == Hkv) gives on contiguous copies.  svgb_attn_fwd, _kv and
 * _gqa run the same host path with B = 1 and batch stride = heads * head stride. */
int svgb_attn_fwd_strided(const void* q, const void* k, const void* v, void* o, float* lse, int dtype, int B, int Hq,
                          int Hkv, int Sq, int Skv, int D, const long long* q_strides, const long long* k_strides,
                          const long long* v_strides, const long long* o_strides, float sm_scale,
                          const svgb_plan* plan, const void* plan_ws, void* stream);
/* svgb_attn_fwd_strided on e4m3 inputs (the FP8 KV cache, and FP8 with grouped-query heads):
 *   q, k, v : e4m3 bytes, D = 128, strides (in elements, i.e. bytes) multiples of 16; bases 16-byte aligned.
 *   q_scale : float [B * Hq], by flat query head b * Hq + hq;  k_scale, v_scale : float [B * Hkv], by flat key/value
 *           head b * Hkv + hkv (x ~= x8 * scale), all three required.  Query head hq reads the scales of the key/value
 *           head hq / G it attends with.
 *   o     : bf16 at its own strides (nonzero multiples of 8 elements);  lse : optional float [B * Hq, Sq].
 *   plan  : SVGB_PLAN_KVCACHE (the cache as num_blocks * block_rows rows, B = 1 at the ABI), SVGB_PLAN_VARBLOCK (over
 *           the B * Hkv key/value heads) or SVGB_PLAN_BAND (Sq == Skv).
 * Refused by name: segment plans, gather plans (row vectors run on svgb_attn_fwd only) and D = 64.  The kernel is
 * svgb_attn_fwd's e4m3 instantiation: with G = 1 and B = 1 each output row is bit for bit svgb_attn_fwd's, and with
 * G > 1 the one of G = 1 on K, V and their scales repeated per group. */
int svgb_attn_fwd_strided_e4m3(const void* q, const void* k, const void* v, const float* q_scale,
                               const float* k_scale, const float* v_scale, void* o, float* lse, int B, int Hq, int Hkv,
                               int Sq, int Skv, int D, const long long* q_strides, const long long* k_strides,
                               const long long* v_strides, const long long* o_strides, float sm_scale,
                               const svgb_plan* plan, const void* plan_ws, void* stream);
int svgb_quantize_e4m3(const void* x, int dtype, void* x8, float* scale, int BH, int S, int D, void* stream);
/* Attention into an e4m3 cache with per-row scales (svgb_kvcache_append_e4m3_rows):
 *   q     : e4m3 [Sq, Hq, 128] (the packed queries of a KV-cache plan) with q_scale float [Hq, Sq], one scale per query
 *           row and head (svgb_quantize_e4m3_rows);  k, v : the e4m3 cache as num_blocks * block_rows rows of Hkv heads,
 *           with k_scale, v_scale float [num_blocks, Hkv, block_rows] (16-byte aligned, block_rows a multiple of 4).
 *   x_strides : {batch, head, row} strides in elements (bytes for e4m3, multiples of 16; the batch stride is not
 *           stepped);  o : bf16 [Sq, Hq, 128] at its strides (multiples of 8 elements);  lse : optional float [Hq, Sq].
 *   s_ij = (q8_i . k8_j) * sq_i * sk_j * sm_scale and o_i = sum_j p_ij (v8_j * sv_j) / l_i, with P and the widened V
 *   in bf16.  Query head hq attends with key/value head hq / (Hq / Hkv).
 * SVGB_PLAN_KVCACHE plans only (every other kind is refused by name), D = 128.  Rows past a block's end in a chunk read
 * zero scales; rows past a stream's length in its last chunk read the tensors and are masked. */
int svgb_attn_fwd_kvcache_e4m3_rows(const void* q, const void* k, const void* v, const float* q_scale,
                                    const float* k_scale, const float* v_scale, void* o, float* lse, int Hq, int Hkv,
                                    int Sq, int num_blocks, int block_rows, int D, const long long* q_strides,
                                    const long long* k_strides, const long long* v_strides, const long long* o_strides,
                                    float sm_scale, const svgb_plan* plan, const void* plan_ws, void* stream);
/* Attention under a split KV-cache plan (svgb_attn_plan_kvcache_split), for every cache format, in two launches: the
 * attention writes each split's fp32 partial o and natural-log lse into ws, then a merge combines the n splits of each
 * (row, query head) in order s = 0 .. n-1: m = max lse_s, w_s = exp(lse_s - m) (0 when lse_s = -inf),
 * o = sum w_s o_s / sum w_s, lse = m + log sum w_s; a row no split saw gets o = 0, lse = -inf.  With one live split the
 * result is the single pass's bit for bit.
 *   q     : the packed queries [B * Sq, Hq, D] at q_strides;  k, v : the cache as num_blocks * block_rows rows of Hkv
 *           heads;  o : [B * Sq, Hq, D] at o_strides;  lse : optional float [Hq, B * Sq].  Strides {batch, head, row}
 *           in elements (the batch stride is not stepped), as svgb_attn_fwd_strided.  Hq = G * Hkv.
 *   dtype : SVGB_BF16 / SVGB_F16 -- 16-bit q, k, v and o, no scales (NULL, row_scales = 0); or SVGB_E4M3 -- an e4m3
 *           cache, D = 128, strides multiples of 16 bytes, bf16 o, and all three scales: row_scales = 0 per head as
 *           svgb_attn_fwd_strided_e4m3 with B = 1 (q_scale [Hq], k_scale, v_scale [Hkv]), row_scales = 1 per row as
 *           svgb_attn_fwd_kvcache_e4m3_rows (q_scale [Hq, B * Sq], k_scale, v_scale [num_blocks, Hkv, block_rows]).
 *   ws    : device, 16-byte aligned, svgb_attn_fwd_kvcache_split_bytes(n, B * Sq, Hq, D) bytes:
 *           n (B Sq) Hq D 4 (partial o [n, B Sq, Hq, D]) + n Hq (B Sq) 4 (partial lse [n, Hq, B Sq]).
 * The split count n comes from the plan (max_items / (B ceil(Sq / 256))).  Deterministic, no atomics. */
int svgb_attn_fwd_kvcache_split_bytes(int num_splits, int rows, int Hq, int D, size_t* bytes);
int svgb_attn_fwd_kvcache_split(const void* q, const void* k, const void* v, const float* q_scale, const float* k_scale,
                                const float* v_scale, void* o, float* lse, int dtype, int row_scales, int B, int Hq,
                                int Hkv, int Sq, int num_blocks, int block_rows, int D, const long long* q_strides,
                                const long long* k_strides, const long long* v_strides, const long long* o_strides,
                                float sm_scale, const svgb_plan* plan, const void* plan_ws, void* ws, size_t ws_bytes,
                                void* stream);
/* Per-row quantisation of 16-bit x [rows, H, 128], read at row_stride / head_stride (elements, multiples of 8; base
 * 16-byte aligned), into e4m3 x8 [rows, H, 128] contiguous and scale float [H, rows], by the rule of
 * svgb_kvcache_append_e4m3_rows; one launch.  A row's bytes and scale depend on that row alone. */
int svgb_quantize_e4m3_rows(const void* x, int dtype, void* x8, float* scale, int rows, int H, int D,
                            long long row_stride, long long head_stride, void* stream);

/* Backward of svgb_attn_fwd: dq, dk, dv from q, k, v, the forward's o and natural-log lse, and the output gradient dO.
 *   q,k,v,o,dO,dq,dk,dv : [BH, S, D] 16-bit (SVGB_BF16 / SVGB_F16), D in {64,128}, all addressed with the one
 *           row_stride / head_stride pair (elements; 16-byte aligned bases, strides multiples of 8 elements).
 *   lse   : float [BH,S] written by svgb_attn_fwd under the same plan and sm_scale.
 *   plan  : the forward (query-major) plan, SVGB_PLAN_VARBLOCK or SVGB_PLAN_BAND with mask SVGB_MASK_NONE / HY / WAN /
 *           COG / LOCAL (not the profiling masks 4-9), or SVGB_PLAN_SEG.  plan_t: its key-major companion --
 *           svgb_attn_plan_band_t with the same mask for a band plan, svgb_attn_plan_varblock(map^T, col_sz, row_sz)
 *           for a variable-block plan, svgb_attn_plan_local_varlen_t with the same bounds and parameters for a segment
 *           plan.
 *   ws    : device scratch of svgb_attn_bwd_bytes (per-row delta = rowsum(dO * O)).
 * Every row of dq, dk, dv is written (rows without an allowed key: dq = 0; keys no row reaches: dk = dv = 0); the
 * result is deterministic (no atomics).  Gather plans, row gathers and e4m3 inputs have no backward. */
int svgb_attn_bwd_bytes(int BH, int S, size_t* bytes);
int svgb_attn_bwd(const void* q, const void* k, const void* v, const void* o, const void* dout, const float* lse,
                  void* dq, void* dk, void* dv, int dtype, int BH, int S, int D, long long row_stride,
                  long long head_stride, float sm_scale, const svgb_plan* plan, const void* plan_ws,
                  const svgb_plan* plan_t, const void* plan_t_ws, void* ws, size_t ws_bytes, void* stream);

/* Backward of svgb_attn_fwd_kv: q, o, dO, dq [BH, Sq, D] at the q strides; k, v, dk, dv [BH, Skv, D] at the k/v
 * strides; lse float [BH, Sq].  plan: the forward's SVGB_PLAN_VARBLOCK plan for (Sq, Skv); plan_t: its key-major
 * companion svgb_attn_plan_varblock_kv(map^T, col_sz, row_sz, Skv, Sq) (svgb_attn_plan_varblock(map^T, ...) when
 * Sq == Skv), or a segment plan and its svgb_attn_plan_local_varlen_t.  ws: device scratch of svgb_attn_bwd_kv_bytes
 * (the delta over Sq rows).  The dQ launch walks plan with
 * K / V over Skv rows; the dK / dV launch walks plan_t with K / V as its rows and Q / dO (Sq rows) as its chunks.
 * Guarantees as svgb_attn_bwd: every gradient row written, no atomics, deterministic; with Sq == Skv and equal
 * strides the gradients are svgb_attn_bwd's, bit for bit.  Variable-block plans and 16-bit inputs only. */
int svgb_attn_bwd_kv_bytes(int BH, int Sq, int Skv, size_t* bytes);
int svgb_attn_bwd_kv(const void* q, const void* k, const void* v, const void* o, const void* dout, const float* lse,
                     void* dq, void* dk, void* dv, int dtype, int BH, int Sq, int Skv, int D, long long q_row_stride,
                     long long q_head_stride, long long kv_row_stride, long long kv_head_stride, float sm_scale,
                     const svgb_plan* plan, const void* plan_ws, const svgb_plan* plan_t, const void* plan_t_ws,
                     void* ws, size_t ws_bytes, void* stream);

/* Backward of svgb_attn_fwd_gqa: q, o, dO, dq [BHq, Sq, D] at the q strides; k, v, dk, dv [BHkv, Skv, D] at the k/v
 * strides; lse float [BHq, Sq].  plan and plan_t are svgb_attn_bwd_kv's (band: svgb_attn_bwd's) built over the BHkv
 * key/value heads.  ws: device scratch of svgb_attn_bwd_gqa_bytes (the delta over BHq * Sq rows).  The dQ launch runs
 * one CTA row per query head on its group's plan; the dK / dV launch one CTA row per key/value head, whose key items
 * walk their chunk list once per query head of the group (g = 0 .. G-1 in order), so dk and dv are the sums over the
 * group's G query heads, kept in registers and stored once.  Guarantees as svgb_attn_bwd (every row written, no
 * atomics, deterministic); dq is bit for bit svgb_attn_bwd / _kv's on K / V repeated per head.  Variable-block and band
 * plans with the backward's masks, 16-bit inputs. */
int svgb_attn_bwd_gqa_bytes(int BHq, int BHkv, int Sq, int Skv, size_t* bytes);
int svgb_attn_bwd_gqa(const void* q, const void* k, const void* v, const void* o, const void* dout, const float* lse,
                      void* dq, void* dk, void* dv, int dtype, int BHq, int BHkv, int Sq, int Skv, int D,
                      long long q_row_stride, long long q_head_stride, long long kv_row_stride,
                      long long kv_head_stride, float sm_scale, const svgb_plan* plan, const void* plan_ws,
                      const svgb_plan* plan_t, const void* plan_t_ws, void* ws, size_t ws_bytes, void* stream);

/* Backward of svgb_attn_fwd_strided: q, o, dO, dq [B, Hq, Sq, D]; k, v, dk, dv [B, Hkv, Skv, D]; each of the eight
 * tensors with its own {batch, head, row} strides under the rules of svgb_attn_fwd_strided, so dO may be a transposed
 * view and the gradients may be written into views (every element of each view is written, nothing outside it).
 * lse float [B * Hq, Sq] contiguous.  plan and plan_t as svgb_attn_bwd_gqa's, built over the B * Hkv key/value heads.
 * ws: device scratch of svgb_attn_bwd_strided_bytes (the delta over B * Hq * Sq rows, read from o and dO at their own
 * strides).  Guarantees as svgb_attn_bwd_gqa, and the gradients are bit for bit its gradients on contiguous copies.
 * svgb_attn_bwd, _kv and _gqa run the same host path with B = 1. */
int svgb_attn_bwd_strided_bytes(int B, int Hq, int Hkv, int Sq, int Skv, size_t* bytes);
int svgb_attn_bwd_strided(const void* q, const void* k, const void* v, const void* o, const void* dout,
                          const float* lse, void* dq, void* dk, void* dv, int dtype, int B, int Hq, int Hkv, int Sq,
                          int Skv, int D, const long long* q_strides, const long long* k_strides,
                          const long long* v_strides, const long long* o_strides, const long long* do_strides,
                          const long long* dq_strides, const long long* dk_strides, const long long* dv_strides,
                          float sm_scale, const svgb_plan* plan, const void* plan_ws, const svgb_plan* plan_t,
                          const void* plan_t_ws, void* ws, size_t ws_bytes, void* stream);

/* density of a variable-block map (density_calculation, svg/kmeans_utils.py:13-31) -> float [BH] */
int svgb_density(const uint8_t* map, const int32_t* row_sz, const int32_t* col_sz, int BH, int QC,
                 int KC, float* density, void* stream);

/* ---- layout transforms ------------------------------------------------------------------ */
/* stable ascending argsort of labels in [0,K): perm int32 [BH,S] (sorted_indices of
 * permute_tensor_by_labels_triton, permute.py:113) and counts int32 [BH,K] (cluster sizes). */
int svgb_argsort_labels_bytes(int BH, int S, int K, size_t* bytes);
int svgb_argsort_labels(const int32_t* labels, int BH, int S, int K, int32_t* perm, int32_t* counts,
                        void* ws, size_t ws_bytes, void* stream);
/* out[h,s,:] = in[h,perm[h,s],:]   (_permute_kernel, permute.py:12-43);  16-bit elements */
int svgb_permute_gather(const void* in, const int32_t* perm, void* out, int BH, int S, int D,
                        void* stream);
/* out[h,perm[h,s],:] = in[h,s,:]   (_inverse_permute_kernel, permute.py:46-75) */
int svgb_permute_scatter(const void* in, const int32_t* perm, void* out, int BH, int S, int D,
                         void* stream);
/* SVG1 head placement (hunyuan_sparse_head_placement, hyvideo/placement.py:34-153): for heads with
 * best_mask_idx==1 the video part goes frame-major -> token-major (dst = patch*F + frame), text
 * untouched; other heads are copied.  text_first=1 selects the CogVideoX variant
 * (cog/placement.py).  inverse=1 is hunyuan_hidden_states_placement (placement.py:285-387).
 * n_tensors in {1,2,3}: in/out arrays of that many [BH,S,D] 16-bit tensors. */
int svgb_head_placement(const void* const* in, void* const* out, int n_tensors,
                        const int32_t* best_mask_idx, int BH, int S, int D, int ctx, int F, int P,
                        int text_first, int inverse, void* stream);

/* ---- flash k-means (svg/kmeans_utils.py:464-733) ------------------------------------------ */
/* one workspace serves assign / update / run for a given (BH, N, K, D); K <= 4096 */
int svgb_kmeans_bytes(int BH, int N, int K, int D, size_t* bytes);
/* x_sq[h,n] = sum_d round16(x^2): round_result=1 rounds the sum to the 16-bit dtype as
 * (x**2).sum(-1) does (batch_kmeans_Euclid :704); 0 keeps the fp32 sum (assign kernel :531) */
int svgb_row_sqnorm(const void* x, float* x_sq, int BH, int N, int D, int dtype, int round_result,
                    void* stream);
/* nearest centroid per point: argmin_k max(0, |x|^2 + |c_k|^2 - 2 x.c_k), lowest k wins ties;
 * x [BH,N,D], c [BH,K,D] 16-bit; x_sq float [BH,N]; labels int32 [BH,N].
 * (_euclid_assign_kernel :464-554).  X.C^T runs on wgmma. */
int svgb_kmeans_assign(const void* x, const void* c, const float* x_sq, int32_t* labels, int BH,
                       int N, int K, int D, int dtype, void* ws, size_t ws_bytes, void* stream);
/* centroid update (triton_centroid_update_sorted_euclid :375-421): fp32 mean of members in token
 * order (deterministic; the reference's atomics are not), empty cluster keeps the old centroid,
 * result rounded to the 16-bit dtype.  counts int32 [BH,K]; shift_max (optional) float[1] =
 * max_k |c_new - c_old|_2 evaluated with the reference's 16-bit tensor roundings (:642). */
int svgb_kmeans_update(const void* x, const int32_t* labels, const void* c_old, void* c_new,
                       int32_t* counts, float* shift_max, int BH, int N, int K, int D, int dtype,
                       void* ws, size_t ws_bytes, void* stream);
/* batch_kmeans_Euclid (:684-733) as one stream-ordered sequence without host syncs: up to
 * max_iters x (assign, update), device-side `break` when shift < tol.  Outputs follow the
 * reference exactly: labels / counts from the last executed assignment; centroids = the updated
 * ones unless the loop broke, then the ones that assignment was made against.  n_iter_out:
 * device int32[1] (optional). */
int svgb_kmeans_run(const void* x, const void* init_centroids, int BH, int N, int K, int D, int dtype,
                    int max_iters, float tol, int32_t* labels, void* centroids_out, int32_t* counts,
                    int32_t* n_iter_out, void* ws, size_t ws_bytes, void* stream);
/* Same loop for the caller the reference has (hyvideo/attention.py:584-626 -> :704-716): x may be a strided view
 * (x_head_stride elements between heads, 0 = N*D; rows stay D apart) so the video part of [H, S, D] is clustered in
 * place (the reference's `[:, :, :-context_length]` slice + `.contiguous()`), and perm_out (optional, int32 [BH,N])
 * receives the stable argsort of the returned labels -- what the reference recomputes with torch.argsort in
 * permute_tensor_by_labels_triton (svg/kernels/triton/permute.py:113; hyvideo/attention.py:651-652) -- for free: the
 * last centroid update already built it. */
int svgb_kmeans_run_sorted(const void* x, long long x_head_stride, const void* init_centroids, int BH, int N, int K,
                           int D, int dtype, int max_iters, float tol, int32_t* labels, void* centroids_out,
                           int32_t* counts, int32_t* n_iter_out, int32_t* perm_out, void* ws, size_t ws_bytes,
                           void* stream);

/* ---- mask selection --------------------------------------------------------------------- */
/* identify_dynamic_map (svg/kmeans_utils.py:864-896): qc [BH,QC,D], kc [BH,KC,D] 16-bit,
 * k_sizes int32 [BH,KC] -> map uint8 [BH,QC,KC].  Ties in the descending sort resolve to the
 * lower column index (stable).  The running sum is torch's CUDA block scan of BH*QC rows, bit for bit;
 * for a single row (BH*QC == 1) torch.cumsum runs cub::DeviceScan instead, and the map may differ from
 * torch's there. */
int svgb_dynamic_map(const void* qc, const void* kc, const int32_t* k_sizes, int BH, int QC, int KC,
                     int D, int dtype, float top_p, int preserve, uint8_t* map, void* stream);
/* sample_mse (hyvideo/attention.py:375-399): MSE between full attention and attention under the two
 * profiling masks (0 spatial, 1 temporal) on `n_rows` sampled query rows -> float [2, BH].
 * layout: 0 = HY (text last, band 1.5*P; hyvideo/utils.py:47-93), 1 = WAN (first-frame sink, band 2*P;
 * wan/utils.py:63-110), 2 = COG (text first, band 1.5*P; cog/utils.py:61-88 -- its temporal mask leaves text rows
 * empty: a sampled text row contributes 0 output here where the reference's softmax yields NaN; the Python mirror
 * CogSVG1Core.sample_mse restores the NaN so argmin picks the same head type).
 * q, k, v: 16-bit only (SVGB_BF16 or SVGB_F16), [BH, S, D] contiguous, D in {64, 128}; 1 <= n_rows <= 128;
 * S == ctx + F * P with F, P > 0, ctx == 0 for WAN and ctx < 2^19 for COG; the band threshold (1.5 * P or 2 * P) / 128
 * below 4096.  Each of these errors returns before the device is queried; only the workspace size depends on the
 * device (its SM count sets the split count).  Precondition, not checked (rows is device data):
 * every rows[i] lies in [0, S). */
int svgb_sample_mse_bytes(int BH, int S, int D, int n_rows, size_t* bytes);
int svgb_sample_mse(const void* q, const void* k, const void* v, const int32_t* rows, int n_rows,
                    int BH, int S, int D, int dtype, int layout, int ctx, int F, int P, float* mse,
                    void* ws, size_t ws_bytes, void* stream);

/* ---- pre-attention elementwise chain (SURVEY 8f-1; the reference's native `_kernels` module) ------- */
/* rms_norm_forward (svg/kernels/csrc/ops.h:52-75): in place on x [m, n] 16-bit, gamma [n]; n in
 * {32,64,128,256}; y = x * rsqrt(mean(x^2) + eps) * gamma, fp32 inside, one rounding. */
int svgb_rms_norm(void* x, const void* gamma, long long m, int n, float eps, int dtype, void* stream);
/* layer_norm_forward (ops.h:20-44): in place, eps fixed at 1e-5 like the reference kernel. */
int svgb_layer_norm(void* x, const void* gamma, const void* beta, long long m, int n, int dtype, void* stream);
/* apply_qk_rope_inplace_cossin{,_txtlast,_complex} (ops.h:77-260): q [B,Hq,S,D], k [B,Hk,S,D] 16-bit,
 * rotated in place on S - len_text rows of every head; interleaved pairs (2i, 2i+1).
 *   SVGB_ROPE_TXT_FIRST          skip the FIRST len_text rows; cos/sin float [S-len_text, D]
 *   SVGB_ROPE_TXT_LAST           skip the LAST  len_text rows; cos/sin float [S-len_text, D]
 *   SVGB_ROPE_COMPLEX_TXT_FIRST  cos/sin float [S-len_text, D/2] (real / imaginary parts), fp64 arithmetic */
#define SVGB_ROPE_TXT_FIRST 0
#define SVGB_ROPE_TXT_LAST 1
#define SVGB_ROPE_COMPLEX_TXT_FIRST 2
int svgb_qk_rope(void* q, void* k, const float* cos_t, const float* sin_t, int B, int Hq, int Hk, int S, int D,
                 int len_text, int mode, int dtype, void* stream);
/* The whole reference chain in one pass (hyvideo/attention.py:253-295, wan/attention.py:100-135):
 *   q_in,k_in,v_in [B, S_in, H*D] (projection outputs; element strides given, so a packed QKV works)
 *   -> unflatten + transpose + contiguous -> QK norm -> RoPE -> rows [out_row0, out_row0+S_in) of
 *   q_out,k_out,v_out [B, H, S_out, D] (so the video and prompt streams of a double block land in one
 *   tensor without torch.cat).  V is only transposed.
 * norm: SVGB_NORM_NONE | SVGB_NORM_RMS_HEAD (gamma [D]) | SVGB_NORM_LAYER (gamma,beta [D], eps 1e-5) |
 *       SVGB_NORM_RMS_HIDDEN (gamma [H*D]: RMS over the full hidden row before the head split, Wan).
 * rope: 0 none | 1 cos/sin float [rope_n, D] | 2 complex float [rope_n, D/2]; tokens
 *       [rope_lo, rope_lo+rope_n) of this input are rotated with table row (token - rope_lo).
 * The norm result is rounded to the 16-bit dtype before RoPE, exactly like the in-place sequence. */
#define SVGB_NORM_NONE 0
#define SVGB_NORM_RMS_HEAD 1
#define SVGB_NORM_LAYER 2
#define SVGB_NORM_RMS_HIDDEN 3
int svgb_qkv_prep(const void* q_in, const void* k_in, const void* v_in, long long in_token_stride,
                  long long in_batch_stride, void* q_out, void* k_out, void* v_out, long long out_head_stride,
                  long long out_batch_stride, int B, int S_in, int H, int D, int out_row0, int norm,
                  const void* gamma_q, const void* gamma_k, const void* beta_q, const void* beta_k, float eps,
                  int rope, const float* cos_t, const float* sin_t, int rope_lo, int rope_n, int dtype,
                  void* stream);

/* Backwards of the chain (DESIGN.md §5).  Deterministic: no atomics; dgamma / dbeta are fp32 sums of per-CTA partials
 * taken in a fixed order (ws holds the partials; two launches), so two calls give the same bits.
 * svgb_rms_norm_bwd / svgb_layer_norm_bwd: x [m, n] the norm's 16-bit input, dy the gradient at its output ->
 *   dx [m, n] (rounded once), dgamma (dbeta) float [n].  eps and n as the forward. */
int svgb_row_norm_bwd_bytes(long long m, int n, size_t* bytes);
int svgb_rms_norm_bwd(const void* x, const void* dy, const void* gamma, void* dx, float* dgamma, long long m, int n,
                      float eps, int dtype, void* ws, size_t ws_bytes, void* stream);
int svgb_layer_norm_bwd(const void* x, const void* dy, const void* gamma, void* dx, float* dgamma, float* dbeta,
                        long long m, int n, int dtype, void* ws, size_t ws_bytes, void* stream);
/* svgb_qk_rope's transpose, out of place: dq [B,Hq,S,D], dk [B,Hk,S,D] -> dq_out, dk_out (same shapes, contiguous);
 * the rotated rows get the transpose of the rotation, the text rows are copied.  Same modes and tables. */
int svgb_qk_rope_bwd(const void* dq, const void* dk, void* dq_out, void* dk_out, const float* cos_t,
                     const float* sin_t, int B, int Hq, int Hk, int S, int D, int len_text, int mode, int dtype,
                     void* stream);
/* svgb_qkv_prep's backward: reads rows [out_row0, out_row0+S_in) of dq, dk, dv [B, H, S_out, D] (no other rows) and
 * the forward's q_in, k_in through their strides (needed when norm != NONE) -> dq_in, dk_in, dv_in contiguous
 * [B, S_in, H*D], and float dgamma_q / dgamma_k ([D], or [H*D] for SVGB_NORM_RMS_HIDDEN), dbeta_q / dbeta_k for
 * SVGB_NORM_LAYER.  Arguments as the forward; the RoPE transpose is rounded to the 16-bit dtype before the norm
 * backward (the forward's rounding point), so it equals svgb_qk_rope_bwd followed by svgb_*_norm_bwd bit for bit. */
int svgb_qkv_prep_bwd_bytes(int B, int S_in, int H, int D, int norm, size_t* bytes);
int svgb_qkv_prep_bwd(const void* dq, const void* dk, const void* dv, long long out_head_stride,
                      long long out_batch_stride, const void* q_in, const void* k_in, long long in_token_stride,
                      long long in_batch_stride, void* dq_in, void* dk_in, void* dv_in, int B, int S_in, int H, int D,
                      int out_row0, int norm, const void* gamma_q, const void* gamma_k, float eps, int rope,
                      const float* cos_t, const float* sin_t, int rope_lo, int rope_n, float* dgamma_q,
                      float* dgamma_k, float* dbeta_q, float* dbeta_k, int dtype, void* ws, size_t ws_bytes,
                      void* stream);

/* ---- Wan transformer-block glue (SURVEY 8f-3; svg/kernels/triton/{layernorm,modulate,rmsnorm}.py) ---- */
/* rows of N elements (N % 8 == 0, N <= 8192), contiguous; x/y/w dtypes: SVGB_BF16 | SVGB_F16 | SVGB_F32;
 * scale/shift/gate are float [nb, N], row r uses vector r / rows_per_batch (rows_per_batch = 0: one vector). */
/* y = LayerNorm(x) [* w + b] [* (1 + scale) + shift]: triton_layernorm_forward followed by
 * triton_modulate_shift_forward (custom_models.py:37-56) in one pass; w/b and scale/shift optional. */
int svgb_layernorm_modulate(const void* x, int x_dtype, const void* w, const void* b, int w_dtype, float eps,
                            const float* scale, const float* shift, long long rows_per_batch, void* y, int y_dtype,
                            long long rows, int N, void* stream);
/* y = x * rsqrt(mean(x^2) + eps) * w over the full row (triton_rmsnorm_forward) */
int svgb_rmsnorm_hidden(const void* x, int x_dtype, const void* w, int w_dtype, float eps, void* y, int y_dtype,
                        long long rows, int N, void* stream);
/* y = x * (1 + scale) + shift (triton_modulate_shift_forward) */
int svgb_modulate_shift(const void* x, int x_dtype, const float* scale, const float* shift,
                        long long rows_per_batch, void* y, int y_dtype, long long rows, int N, void* stream);
/* y = residual + x * gate (triton_modulate_gate_residual_forward) */
int svgb_gate_residual(const void* residual, int res_dtype, const void* x, int x_dtype, const float* gate,
                       long long rows_per_batch, void* y, int y_dtype, long long rows, int N, void* stream);

/* ---- self tests (debug; exercised by tests/ on the GPU) ----------------------------------- */
/* One 128x128xD tile through the exact descriptor paths the attention kernel uses:
 * s_out[128,128] = q k^T (fp32), o_out[128,D] = bf16(s*p_scale) v (fp32). */
int svgb_selftest_tile(const void* q, const void* k, const void* v, float* s_out, float* o_out,
                       int D, int dtype, float p_scale, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SVGB200_H_ */
