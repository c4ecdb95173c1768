// Attention backward: the delta pre-pass and the query-major (dQ) and key-major (dK, dV) launches.  The kernels are in
// attn_bwd_kernel.cuh; the key-major plans come from the forward's planners (attn_fwd.cu).
#include "../../include/svgb200.h"
#include "attn_bwd_kernel.cuh"
#include "host_common.h"

namespace svgb {

template <int D, int DT, bool kKeyMajor>
static int launch_bwd(const CUtensorMap& xm, const CUtensorMap& ym, const CUtensorMap& um, const CUtensorMap& wm,
                      const AttnBwdArgs& a, dim3 grid, cudaStream_t st) {
  constexpr int smem = AttnBwdCfg<D>::kSmemBytes;
  auto kern = attn_bwd_kernel<D, DT, kKeyMajor>;
  SVGB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  kern<<<grid, AttnBwdCfg<D>::kThreads, smem, st>>>(xm, ym, um, wm, a);
  SVGB_LAUNCH_OK();
  return 0;
}

template <int D, int DT>
static int launch_bwd_pair(const CUtensorMap& qm, const CUtensorMap& km, const CUtensorMap& vm, const CUtensorMap& dom,
                           const AttnBwdArgs& aq, dim3 gq, const AttnBwdArgs& ak, dim3 gk, cudaStream_t st) {
  if (launch_bwd<D, DT, true>(km, vm, qm, dom, ak, gk, st)) return -1;
  return launch_bwd<D, DT, false>(qm, dom, km, vm, aq, gq, st);
}

static AttnBwdArgs bwd_args(const svgb_plan* p, const void* ws) {
  const char* w = static_cast<const char*>(ws);
  AttnBwdArgs a;
  a.items = reinterpret_cast<const int4*>(w + p->items_off);
  a.item_count = reinterpret_cast<const int*>(w + p->counts_off);
  a.chunks = reinterpret_cast<const int2*>(w + p->chunks_off);
  a.items_stride = p->items_stride;
  a.mask_mode = p->mask_mode;
  a.m0 = p->m0;
  a.m1 = p->m1;
  a.m2 = p->m2;
  if (p->kind == SVGB_PLAN_SEG || p->kind == SVGB_PLAN_SEG_T)
    a.segs = reinterpret_cast<const int*>(w + SVGB_PLAN_SEG_BOUNDS_OFF);
  return a;
}

// One backward call: q, o, dO, dq over Sq rows and Hq heads in B batch elements, k, v, dk, dv over Skv rows and Hkv
// heads, each tensor with its own strides.
struct AttnBwdCall {
  const void *q, *k, *v, *o, *dout;
  const float* lse;
  void *dq, *dk, *dv;
  int dtype, B, Hq, Hkv, Sq, Skv, D;
  Strides qs, ks, vs, os, dos, dqs, dks, dvs;
  float sm_scale;
  const svgb_plan* plan;
  const void* plan_ws;
  const svgb_plan* plan_t;
  const void* plan_t_ws;
  void* ws;
  size_t ws_bytes;
  void* stream;
};

// what one backward entry accepts: its name and the forward plan kinds (bit k: kind k)
struct AttnBwdRule {
  const char* who;
  unsigned kinds;
  const char* kinds_text;
};
enum { BWD, BWD_KV, BWD_GQA, BWD_STRIDED };
constexpr unsigned kBandOrSeg = 1u << SVGB_PLAN_VARBLOCK | 1u << SVGB_PLAN_BAND | 1u << SVGB_PLAN_SEG;
static constexpr AttnBwdRule kBwdRules[] = {
    {"svgb_attn_bwd", kBandOrSeg, "variable-block, band or segment plans"},
    {"svgb_attn_bwd_kv", 1u << SVGB_PLAN_VARBLOCK | 1u << SVGB_PLAN_SEG, "segment plans and variable-block plans"},
    {"svgb_attn_bwd_gqa", kBandOrSeg, "variable-block, band or segment plans"},
    {"svgb_attn_bwd_strided", kBandOrSeg, "variable-block, band or segment plans"},
};

// Every rule of the backward, in one order, before any device work.
static int attn_bwd_check(const AttnBwdCall& c, const AttnBwdRule& r) {
  const char* who = r.who;
  const svgb_plan *plan = c.plan, *plan_t = c.plan_t;
  SVGB_REQUIRE(c.q && c.k && c.v && c.o && c.dout && c.lse && c.dq && c.dk && c.dv && plan && c.plan_ws && plan_t &&
                   c.plan_t_ws && c.ws,
               "null pointer");
  // KV-cache plans run forward only, as FlashAttention's flash_attn_with_kvcache
  SVGB_REQUIRE(plan->kind != SVGB_PLAN_KVCACHE,
               "%s: a KV-cache plan (svgb_attn_plan_kvcache) has no backward; it runs forward only", who);
  SVGB_REQUIRE(plan->kind != SVGB_PLAN_KVCACHE_SPLIT,
               "%s: a split KV-cache plan (svgb_attn_plan_kvcache_split) has no backward; it runs forward only, on "
               "svgb_attn_fwd_kvcache_split", who);
  SVGB_REQUIRE(plan->kind >= 1 && plan->kind <= 8 && (r.kinds >> plan->kind & 1),
               "%s takes %s only (kind %d; gather plans have no backward, key-major plans go in plan_t)", who,
               r.kinds_text, plan->kind);
  SVGB_REQUIRE(c.dtype == SVGB_BF16 || c.dtype == SVGB_F16,
               "%s takes bf16 or fp16 inputs (dtype %d; e4m3 attention has no backward)", who, c.dtype);
  SVGB_REQUIRE(c.D == 64 || c.D == 128, "head_dim %d unsupported (64 or 128)", c.D);
  SVGB_REQUIRE(c.B > 0 && c.Hq > 0 && c.Hkv > 0 && c.Hq % c.Hkv == 0,
               "%s: the query heads Hq=%d must be a multiple of the key/value heads Hkv=%d (B=%d)", who, c.Hq, c.Hkv, c.B);
  SVGB_REQUIRE(plan->kind != SVGB_PLAN_BAND || c.Sq == c.Skv, "%s: band plans need Sq == Skv (got %d, %d)", who, c.Sq,
               c.Skv);
  const int kind_t = plan->kind == SVGB_PLAN_BAND  ? SVGB_PLAN_BAND_T
                     : plan->kind == SVGB_PLAN_SEG ? SVGB_PLAN_SEG_T
                                                   : SVGB_PLAN_VARBLOCK;
  SVGB_REQUIRE(plan_t->kind == kind_t, "plan_t (kind %d) is not the key-major companion of a kind-%d plan",
               plan_t->kind, plan->kind);
  SVGB_REQUIRE((plan->mask_mode >= MASK_NONE && plan->mask_mode <= MASK_COG) || plan->mask_mode == MASK_LOCAL ||
                   plan->mask_mode == MASK_BLOCK_CAUSAL,
               "attention backward supports the executed band masks NONE / HY / WAN / COG / LOCAL / BLOCK_CAUSAL (mask "
               "mode %d)", plan->mask_mode);
  // a variable-block plan's m0 is its Skv (svgb200.h), checked with the lengths below
  SVGB_REQUIRE(plan->kind == SVGB_PLAN_VARBLOCK ||
                   (plan_t->mask_mode == plan->mask_mode && plan_t->m0 == plan->m0 && plan_t->m1 == plan->m1 &&
                    plan_t->m2 == plan->m2),
               "plan_t was built for another mask than plan");
  // a segment plan's layout is a function of (nseg, Sq, Skv), so equal layouts mean equal segment counts
  SVGB_REQUIRE(plan->kind != SVGB_PLAN_SEG || (plan_t->items_off == plan->items_off &&
                                               plan_t->chunks_off == plan->chunks_off && plan_t->bytes == plan->bytes),
               "plan_t was built for another segmentation than plan (nseg, Sq or Skv)");
  // both plans are per key/value head; the key-major plan has the keys as rows: its S is Skv and its Skv is Sq
  const int BHkv = c.B * c.Hkv;
  SVGB_REQUIRE(plan->items_stride == 0 || plan->BH == BHkv,
               "%s: a per-head plan is built over the BHkv=%d key/value heads (plan BH=%d)", who, BHkv, plan->BH);
  SVGB_REQUIRE(plan_t->items_stride == 0 || plan_t->BH == BHkv,
               "%s: a per-head plan_t is built over the B*Hkv=%d key/value heads (plan_t BH=%d)", who, BHkv, plan_t->BH);
  SVGB_REQUIRE(plan->S == c.Sq && plan_kv_len(plan) == c.Skv,
               "plan was built for BH=%d Sq=%d Skv=%d, called with BH=%d Sq=%d Skv=%d", plan->BH, plan->S,
               plan_kv_len(plan), BHkv, c.Sq, c.Skv);
  SVGB_REQUIRE(plan_t->S == c.Skv && plan_kv_len(plan_t) == c.Sq,
               "plan_t was built for BH=%d S=%d Skv=%d; the key-major plan of this call has BH=%d S=%d Skv=%d",
               plan_t->BH, plan_t->S, plan_kv_len(plan_t), BHkv, c.Skv, c.Sq);
  size_t need = 0;
  if (svgb_attn_bwd_bytes(c.B * c.Hq, c.Sq, &need)) return -1;
  SVGB_REQUIRE(c.ws_bytes >= need, "backward workspace too small: %zu < %zu", c.ws_bytes, need);
  for (const void* t : {c.dq, c.dk, c.dv})
    SVGB_REQUIRE((reinterpret_cast<uintptr_t>(t) & 15) == 0, "gradients must be 16-byte aligned");
  SVGB_REQUIRE((reinterpret_cast<uintptr_t>(c.o) & 15) == 0 && (reinterpret_cast<uintptr_t>(c.dout) & 15) == 0,
               "o / dO must be 16-byte aligned with strides multiple of 8 elements");
  for (const Strides& s : {c.qs, c.ks, c.vs, c.os, c.dos, c.dqs, c.dks, c.dvs})
    SVGB_REQUIRE(s.r % 8 == 0 && s.h % 8 == 0 && s.b % 8 == 0,
                 "every stride must be a multiple of 8 elements (got %lld, %lld, %lld)", s.b, s.h, s.r);
  return 0;
}

// The delta pre-pass, then the dK / dV launch over the key-major plan (X / Y = K / V, U / W = Q / dO, one CTA row per
// key/value head) and the dQ launch over the forward plan (X / Y = Q / dO, U / W = K / V, one CTA row per query head);
// lse and delta are per query row in both.
static int attn_bwd(const AttnBwdCall& c, int row) {
  if (attn_bwd_check(c, kBwdRules[row])) return -1;
  const int B = c.B, Hq = c.Hq, Hkv = c.Hkv, Sq = c.Sq, Skv = c.Skv, D = c.D, dtype = c.dtype;
  const int BH = B * Hq, BHkv = B * Hkv;
  cudaStream_t st = static_cast<cudaStream_t>(c.stream);
  float* delta = static_cast<float*>(c.ws);

  const long long rows = static_cast<long long>(BH) * Sq;
  const unsigned blocks = static_cast<unsigned>((rows + 7) / 8);
  auto delta_kernel = dtype == SVGB_BF16 ? attn_bwd_delta_kernel<true> : attn_bwd_delta_kernel<false>;
  delta_kernel<<<blocks, 256, 0, st>>>(static_cast<const uint16_t*>(c.o), static_cast<const uint16_t*>(c.dout), c.os.b,
                                       c.os.h, c.os.r, c.dos.b, c.dos.h, c.dos.r, BH, Hq, Sq, D, delta);
  SVGB_LAUNCH_OK();

  CUtensorMap qm, km, vm, dom;
  if (encode_tmap_bhsd(&qm, c.q, dtype, B, Hq, Sq, D, c.qs)) return -1;
  if (encode_tmap_bhsd(&km, c.k, dtype, B, Hkv, Skv, D, c.ks)) return -1;
  if (encode_tmap_bhsd(&vm, c.v, dtype, B, Hkv, Skv, D, c.vs)) return -1;
  if (encode_tmap_bhsd(&dom, c.dout, dtype, B, Hq, Sq, D, c.dos)) return -1;
  AttnBwdArgs aq = bwd_args(c.plan, c.plan_ws), ak = bwd_args(c.plan_t, c.plan_t_ws);
  for (AttnBwdArgs* a : {&aq, &ak}) {
    a->lse = c.lse;
    a->delta = delta;
    a->scale_log2 = c.sm_scale * 1.4426950408889634f;
    a->sm_scale = c.sm_scale;
    a->S = Sq;
    a->kv_group = Hq / Hkv;
  }
  aq.Hx = Hq;
  ak.Hx = Hkv;
  aq.g0 = c.dq;
  aq.g0_bs = c.dqs.b, aq.g0_hs = c.dqs.h, aq.g0_rs = c.dqs.r;
  ak.g0 = c.dk;
  ak.g0_bs = c.dks.b, ak.g0_hs = c.dks.h, ak.g0_rs = c.dks.r;
  ak.g1 = c.dv;
  ak.g1_bs = c.dvs.b, ak.g1_hs = c.dvs.h, ak.g1_rs = c.dvs.r;
  const dim3 gq(c.plan->max_items, BH), gk(c.plan_t->max_items, BHkv);
  if (D == 128)
    return dtype == SVGB_BF16 ? launch_bwd_pair<128, DT_BF16>(qm, km, vm, dom, aq, gq, ak, gk, st)
                              : launch_bwd_pair<128, DT_F16>(qm, km, vm, dom, aq, gq, ak, gk, st);
  return dtype == SVGB_BF16 ? launch_bwd_pair<64, DT_BF16>(qm, km, vm, dom, aq, gq, ak, gk, st)
                            : launch_bwd_pair<64, DT_F16>(qm, km, vm, dom, aq, gq, ak, gk, st);
}

}  // namespace svgb

using namespace svgb;

extern "C" {

int svgb_attn_bwd_bytes(int BH, int S, size_t* bytes) {
  SVGB_REQUIRE(BH > 0 && S > 0 && bytes, "bad arguments");
  *bytes = align_up(sizeof(float) * static_cast<size_t>(BH) * S, 256);
  return 0;
}

int svgb_attn_bwd(const void* q, const void* k, const void* v, const void* o, const void* dout, const float* lse,
                  void* dq, void* dk, void* dv, int dtype, int BH, int S, int D, long long row_stride,
                  long long head_stride, float sm_scale, const svgb_plan* plan, const void* plan_ws,
                  const svgb_plan* plan_t, const void* plan_t_ws, void* ws, size_t ws_bytes, void* stream) {
  const Strides x = flat_strides(row_stride, head_stride, BH);
  return attn_bwd({q, k, v, o, dout, lse, dq, dk, dv, dtype, 1, BH, BH, S, S, D, x, x, x, x, x, x, x, x, sm_scale, plan,
                   plan_ws, plan_t, plan_t_ws, ws, ws_bytes, stream},
                  BWD);
}

int svgb_attn_bwd_kv_bytes(int BH, int Sq, int Skv, size_t* bytes) {
  SVGB_REQUIRE(Skv > 0, "bad arguments");
  return svgb_attn_bwd_bytes(BH, Sq, bytes);  // the per-query-row delta
}

int svgb_attn_bwd_kv(const void* q, const void* k, const void* v, const void* o, const void* dout, const float* lse,
                     void* dq, void* dk, void* dv, int dtype, int BH, int Sq, int Skv, int D, long long q_row_stride,
                     long long q_head_stride, long long kv_row_stride, long long kv_head_stride, float sm_scale,
                     const svgb_plan* plan, const void* plan_ws, const svgb_plan* plan_t, const void* plan_t_ws,
                     void* ws, size_t ws_bytes, void* stream) {
  const Strides x = flat_strides(q_row_stride, q_head_stride, BH), y = flat_strides(kv_row_stride, kv_head_stride, BH);
  return attn_bwd({q, k, v, o, dout, lse, dq, dk, dv, dtype, 1, BH, BH, Sq, Skv, D, x, y, y, x, x, x, y, y, sm_scale,
                   plan, plan_ws, plan_t, plan_t_ws, ws, ws_bytes, stream},
                  BWD_KV);
}

int svgb_attn_bwd_gqa_bytes(int BHq, int BHkv, int Sq, int Skv, size_t* bytes) {
  SVGB_REQUIRE(BHkv > 0 && Skv > 0, "bad arguments");
  return svgb_attn_bwd_bytes(BHq, Sq, bytes);  // the per-query-row delta
}

int svgb_attn_bwd_gqa(const void* q, const void* k, const void* v, const void* o, const void* dout, const float* lse,
                      void* dq, void* dk, void* dv, int dtype, int BHq, int BHkv, int Sq, int Skv, int D,
                      long long q_row_stride, long long q_head_stride, long long kv_row_stride,
                      long long kv_head_stride, float sm_scale, const svgb_plan* plan, const void* plan_ws,
                      const svgb_plan* plan_t, const void* plan_t_ws, void* ws, size_t ws_bytes, void* stream) {
  const Strides x = flat_strides(q_row_stride, q_head_stride, BHq), y = flat_strides(kv_row_stride, kv_head_stride, BHkv);
  return attn_bwd({q, k, v, o, dout, lse, dq, dk, dv, dtype, 1, BHq, BHkv, Sq, Skv, D, x, y, y, x, x, x, y, y, sm_scale,
                   plan, plan_ws, plan_t, plan_t_ws, ws, ws_bytes, stream},
                  BWD_GQA);
}

int svgb_attn_bwd_strided_bytes(int B, int Hq, int Hkv, int Sq, int Skv, size_t* bytes) {
  SVGB_REQUIRE(B > 0 && Hq > 0 && Hkv > 0 && Skv > 0, "bad arguments");
  return svgb_attn_bwd_bytes(B * Hq, Sq, bytes);  // the per-query-row delta
}

int svgb_attn_bwd_strided(const void* q, const void* k, const void* v, const void* o, const void* dout,
                          const float* lse, void* dq, void* dk, void* dv, int dtype, int B, int Hq, int Hkv, int Sq,
                          int Skv, int D, const long long* q_strides, const long long* k_strides,
                          const long long* v_strides, const long long* o_strides, const long long* do_strides,
                          const long long* dq_strides, const long long* dk_strides, const long long* dv_strides,
                          float sm_scale, const svgb_plan* plan, const void* plan_ws, const svgb_plan* plan_t,
                          const void* plan_t_ws, void* ws, size_t ws_bytes, void* stream) {
  Strides st[8];
  if (attn_strided_check(B, Hq, Hkv, {q, k, v, o, dout, dq, dk, dv},
                         {q_strides, k_strides, v_strides, o_strides, do_strides, dq_strides, dk_strides, dv_strides},
                         st, kBwdRules[BWD_STRIDED].who))
    return -1;
  return attn_bwd({q, k, v, o, dout, lse, dq, dk, dv, dtype, B, Hq, Hkv, Sq, Skv, D, st[0], st[1], st[2], st[3], st[4],
                   st[5], st[6], st[7], sm_scale, plan, plan_ws, plan_t, plan_t_ws, ws, ws_bytes, stream},
                  BWD_STRIDED);
}

}  // extern "C"
