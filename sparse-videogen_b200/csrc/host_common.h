// Host-side helpers shared by every translation unit of libsvgb200.so.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>

#include <initializer_list>

#include "../../include/svgb200.h"

namespace svgb {

// thread-local last-error message (api.cu)
void set_error(const char* fmt, ...);
const char* get_error();

#define SVGB_REQUIRE(cond, ...)   \
  do {                            \
    if (!(cond)) {                \
      svgb::set_error(__VA_ARGS__); \
      return -1;                  \
    }                             \
  } while (0)

#define SVGB_CUDA(expr)                                                                    \
  do {                                                                                     \
    cudaError_t _e = (expr);                                                               \
    if (_e != cudaSuccess) {                                                               \
      svgb::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__,    \
                      __LINE__);                                                           \
      return -2;                                                                           \
    }                                                                                      \
  } while (0)

// check the launch that just happened (no sync)
#define SVGB_LAUNCH_OK()                                                                   \
  do {                                                                                     \
    cudaError_t _e = cudaGetLastError();                                                   \
    if (_e != cudaSuccess) {                                                               \
      svgb::set_error("kernel launch failed: %s (%s:%d)", cudaGetErrorString(_e), __FILE__, \
                      __LINE__);                                                           \
      return -3;                                                                           \
    }                                                                                      \
  } while (0)

inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// 3-D TMA descriptor over a [BH, S, D] 16-bit tensor addressed as (d, s, h) with byte strides.
// box = 64 x 128 x 1, 128-byte swizzle.  Returns 0 on success.
int encode_tmap_hsd(CUtensorMap* map, const void* base, int dtype, int BH, int S, int D,
                    long long row_stride_elems, long long head_stride_elems, int box_rows = 128);

// element strides of one [B, H, S, D] attention operand; the last dimension is contiguous
struct Strides {
  long long b, h, r;
};
// the (row, head) stride pair of a flat [BH, S, D] operand: one batch element of BH heads
inline Strides flat_strides(long long rs, long long hs, int BH) { return {BH * hs, hs, rs}; }

// 4-D TMA descriptor over a [B, H, S, D] operand addressed as (d, s, h, b) with the byte strides of st.
// box = one 128-byte panel x 128 rows x 1 x 1, 128-byte swizzle.  Returns 0 on success.
int encode_tmap_bhsd(CUtensorMap* map, const void* base, int dtype, int B, int H, int S, int D, Strides st);

// 3-D TMA descriptor over per-row scales, float [num_blocks, H, block_rows] contiguous, addressed as (row, head, block),
// box = 128 x 1 x 1, no swizzle; rows past block_rows are filled with zeros.  Returns 0 on success.
int encode_tmap_scale_rows(CUtensorMap* map, const float* base, int num_blocks, int H, int block_rows);

// the per-row scale tensors of an e4m3 cache (kvcache.cu): both given, 16-byte aligned, block_rows a multiple of 4
int kv_scale_rows_check(const float* k_scale, const float* v_scale, int block_rows, const char* who);

// the parameters of SVGB_MASK_BLOCK_CAUSAL: sink >= 0, m1 = C | (C - F) << 16 with 1 <= C < 2^16 and 1 <= F <= C, and
// a window W >= C
inline int block_causal_check(int sink, int m1, int W, const char* who) {
  const int C = m1 & 0xffff, F = C - ((m1 >> 16) & 0xffff);
  SVGB_REQUIRE(m1 >= 0, "%s: block-causal m1 = %d is not C | (C - F) << 16 with C, C - F < 2^16", who, m1);
  SVGB_REQUIRE(C >= 1, "%s: block-causal block C = %d must be >= 1", who, C);
  SVGB_REQUIRE(F >= 1, "%s: block-causal first_block F = %d must lie in [1, C = %d]", who, F, C);
  SVGB_REQUIRE(W >= C, "%s: block-causal window W = %d must be >= the block C = %d (every row keeps its own block)", who,
               W, C);
  SVGB_REQUIRE(sink >= 0, "%s: block-causal sink = %d must be >= 0", who, sink);
  return 0;
}

// m1 of SVGB_MASK_BLOCK_CAUSAL from block C and first_block F, each checked by name
inline int block_causal_m1(int block, int first_block, int* m1, const char* who) {
  SVGB_REQUIRE(block >= 1 && block < (1 << 16), "%s: block C = %d must lie in [1, 2^16) (it is packed in 16 bits)", who,
               block);
  SVGB_REQUIRE(first_block >= 1 && first_block <= block, "%s: first_block F = %d must lie in [1, C = %d]", who,
               first_block, block);
  *m1 = block | (block - first_block) << 16;
  return 0;
}

// every field of a plan descriptor, so that no planner leaves one indeterminate; varlen_items is 0 outside the
// variable-length KV-cache planner
inline void write_plan(svgb_plan* p, int kind, int BH, int S, int max_items, int items_stride, int mask_mode, int m0,
                       int m1, int m2, int varlen_items, int64_t items_off, int64_t chunks_off, int64_t bytes) {
  *p = svgb_plan{kind, BH, S, max_items, items_stride, mask_mode, m0, m1, m2, varlen_items, 0, items_off, chunks_off,
                 bytes};
}

// key/value rows of a plan: a variable-block plan of svgb_attn_plan_varblock_kv records them in m0, a segment plan in
// BH (svgb200.h); every other plan has Skv = S
inline int plan_kv_len(const svgb_plan* p) {
  if (p->kind == SVGB_PLAN_SEG || p->kind == SVGB_PLAN_SEG_T || p->kind == SVGB_PLAN_KVCACHE ||
      p->kind == SVGB_PLAN_KVCACHE_SPLIT)
    return p->BH;
  return p->kind == SVGB_PLAN_VARBLOCK && p->m0 > 0 ? p->m0 : p->S;
}

// the operands of a strided entry (svgb_attn_fwd_strided, svgb_attn_bwd_strided), before any device work: B batch
// elements of Hq query heads over Hkv key/value heads, 16-byte aligned bases, and (batch, head, row) strides that are
// nonzero multiples of 8 elements, copied to st[i]
inline int attn_strided_check(int B, int Hq, int Hkv, std::initializer_list<const void*> ptrs,
                              std::initializer_list<const long long*> strides, Strides* st, const char* who) {
  SVGB_REQUIRE(B > 0 && Hq > 0 && Hkv > 0, "%s: bad head counts B=%d Hq=%d Hkv=%d", who, B, Hq, Hkv);
  for (const void* p : ptrs) {
    SVGB_REQUIRE(p, "null pointer");
    SVGB_REQUIRE((reinterpret_cast<uintptr_t>(p) & 15) == 0, "%s: every tensor must be 16-byte aligned", who);
  }
  for (const long long* s : strides) {
    SVGB_REQUIRE(s, "null pointer");
    for (int i = 0; i < 3; ++i)
      SVGB_REQUIRE(s[i] != 0 && s[i] % 8 == 0,
                   "%s: every (batch, head, row) stride must be a nonzero multiple of 8 elements (got %lld, %lld, %lld)",
                   who, s[0], s[1], s[2]);
    *st++ = {s[0], s[1], s[2]};
  }
  return 0;
}

struct AttnArgs;
// attention launch with independent query / key-value geometry (attn_fwd.cu); used by svgb_attn_fwd
// and by sample_mse's split-KV passes.  q over B batch elements of BH / B heads and Sq rows, k and v over
// BH / a.kv_group heads and Skv rows, each with its own strides.  Checks D and dtype; gather selects the row-gather
// kernel (run lists, B = 1).
int attn_fwd_impl(const void* q, Strides qs, int Sq, const void* k, Strides ks, const void* v, Strides vs, int Skv,
                  int dtype, int B, int BH, int D, const AttnArgs& a, bool gather, int grid_x, cudaStream_t st);

// stable counting-sort argsort (layout_ops.cu); `offs` (optional) receives the exclusive prefix of
// counts per head; `skip_flag` (optional, device) turns the three kernels into no-ops when non-zero.
int argsort_labels_impl(const int* labels, int BH, int S, int K, int* perm, int* counts, int* offs,
                        void* ws, const int* skip_flag, cudaStream_t stream);

}  // namespace svgb
