// Host-side helpers shared by every translation unit of libsvgb200.so.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>

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

// key/value rows of a plan: a variable-block plan of svgb_attn_plan_varblock_kv records them in m0 (svgb200.h);
// every other plan has Skv = S
inline int plan_kv_len(const svgb_plan* p) { return p->kind == SVGB_PLAN_VARBLOCK && p->m0 > 0 ? p->m0 : p->S; }

// the checks svgb_attn_fwd_gqa and svgb_attn_bwd_gqa share, before any device work: BHq query heads in groups over
// BHkv key/value heads, 16-bit inputs, and a variable-block plan over the key/value heads or a band plan (one work
// list for every head, Sq == Skv)
inline int attn_gqa_check(int dtype, int BHq, int BHkv, int Sq, int Skv, const svgb_plan* plan, const char* who) {
  SVGB_REQUIRE(plan, "null pointer");
  SVGB_REQUIRE(BHq > 0 && BHkv > 0 && BHq % BHkv == 0,
               "%s: the query heads BHq=%d must be a multiple of the key/value heads BHkv=%d", who, BHq, BHkv);
  SVGB_REQUIRE(dtype == SVGB_BF16 || dtype == SVGB_F16,
               "%s takes bf16 or fp16 inputs (dtype %d; e4m3 attention has no GQA path)", who, dtype);
  SVGB_REQUIRE(plan->kind == SVGB_PLAN_VARBLOCK || plan->kind == SVGB_PLAN_BAND,
               "%s takes variable-block or band plans (kind %d; gather and key-major plans have no GQA path)", who,
               plan->kind);
  SVGB_REQUIRE(plan->kind != SVGB_PLAN_BAND || Sq == Skv, "%s: band plans need Sq == Skv (got %d, %d)", who, Sq, Skv);
  SVGB_REQUIRE(plan->items_stride == 0 || plan->BH == BHkv,
               "%s: a per-head plan is built over the BHkv=%d key/value heads (plan BH=%d)", who, BHkv, plan->BH);
  return 0;
}

struct AttnArgs;
// attention launch with independent query / key-value geometry (attn_fwd.cu); used by svgb_attn_fwd
// and by sample_mse's split-KV passes.  Checks D and dtype; gather selects the row-gather kernel (run lists).
int attn_fwd_impl(const void* q, int Sq, long long q_rs, long long q_hs, const void* k, const void* v, int Skv,
                  long long kv_rs, long long kv_hs, int dtype, int BH, int D, const AttnArgs& a, bool gather,
                  int grid_x, cudaStream_t st);

// stable counting-sort argsort (layout_ops.cu); `offs` (optional) receives the exclusive prefix of
// counts per head; `skip_flag` (optional, device) turns the three kernels into no-ops when non-zero.
int argsort_labels_impl(const int* labels, int BH, int S, int K, int* perm, int* counts, int* offs,
                        void* ws, const int* skip_flag, cudaStream_t stream);

}  // namespace svgb
