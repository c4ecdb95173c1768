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
  return a;
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
  SVGB_REQUIRE(q && k && v && o && dout && lse && dq && dk && dv && plan && plan_ws && plan_t && plan_t_ws && ws,
               "null pointer");
  SVGB_REQUIRE(dtype == SVGB_BF16 || dtype == SVGB_F16,
               "attention backward takes bf16 or fp16 inputs (dtype %d; e4m3 attention has no backward)", dtype);
  SVGB_REQUIRE(D == 64 || D == 128, "head_dim %d unsupported (64 or 128)", D);
  SVGB_REQUIRE(plan->kind == SVGB_PLAN_VARBLOCK || plan->kind == SVGB_PLAN_BAND,
               "attention backward needs a variable-block or band plan (kind %d; gather plans have no backward)",
               plan->kind);
  SVGB_REQUIRE(plan_t->kind == (plan->kind == SVGB_PLAN_BAND ? SVGB_PLAN_BAND_T : SVGB_PLAN_VARBLOCK),
               "plan_t (kind %d) is not the key-major companion of a kind-%d plan", plan_t->kind, plan->kind);
  SVGB_REQUIRE(plan->mask_mode >= MASK_NONE && plan->mask_mode <= MASK_COG,
               "attention backward supports the executed band masks NONE / HY / WAN / COG (mask mode %d)",
               plan->mask_mode);
  SVGB_REQUIRE(plan_t->mask_mode == plan->mask_mode && plan_t->m0 == plan->m0 && plan_t->m1 == plan->m1 &&
                   plan_t->m2 == plan->m2,
               "plan_t was built for another mask than plan");
  for (const svgb_plan* p : {plan, plan_t})
    SVGB_REQUIRE(p->S == S && (p->items_stride == 0 || p->BH == BH),
                 "plan was built for BH=%d S=%d, called with BH=%d S=%d", p->BH, p->S, BH, S);
  size_t need = 0;
  if (svgb_attn_bwd_bytes(BH, S, &need)) return -1;
  SVGB_REQUIRE(ws_bytes >= need, "backward workspace too small: %zu < %zu", ws_bytes, need);
  for (const void* t : {dq, dk, dv})
    SVGB_REQUIRE((reinterpret_cast<uintptr_t>(t) & 15) == 0, "gradients must be 16-byte aligned");
  SVGB_REQUIRE((reinterpret_cast<uintptr_t>(o) & 15) == 0 && (reinterpret_cast<uintptr_t>(dout) & 15) == 0 &&
                   row_stride % 8 == 0 && head_stride % 8 == 0,
               "o / dO must be 16-byte aligned with strides multiple of 8 elements");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  float* delta = static_cast<float*>(ws);

  const long long rows = static_cast<long long>(BH) * S;
  const unsigned blocks = static_cast<unsigned>((rows + 7) / 8);
  if (dtype == SVGB_BF16)
    attn_bwd_delta_kernel<true><<<blocks, 256, 0, st>>>(static_cast<const uint16_t*>(o),
                                                        static_cast<const uint16_t*>(dout), row_stride, head_stride,
                                                        BH, S, D, delta);
  else
    attn_bwd_delta_kernel<false><<<blocks, 256, 0, st>>>(static_cast<const uint16_t*>(o),
                                                         static_cast<const uint16_t*>(dout), row_stride, head_stride,
                                                         BH, S, D, delta);
  SVGB_LAUNCH_OK();

  CUtensorMap qm, km, vm, dom;
  if (encode_tmap_hsd(&qm, q, dtype, BH, S, D, row_stride, head_stride)) return -1;
  if (encode_tmap_hsd(&km, k, dtype, BH, S, D, row_stride, head_stride)) return -1;
  if (encode_tmap_hsd(&vm, v, dtype, BH, S, D, row_stride, head_stride)) return -1;
  if (encode_tmap_hsd(&dom, dout, dtype, BH, S, D, row_stride, head_stride)) return -1;
  AttnBwdArgs aq = bwd_args(plan, plan_ws), ak = bwd_args(plan_t, plan_t_ws);
  for (AttnBwdArgs* a : {&aq, &ak}) {
    a->lse = lse;
    a->delta = delta;
    a->row_stride = row_stride;
    a->head_stride = head_stride;
    a->scale_log2 = sm_scale * 1.4426950408889634f;
    a->sm_scale = sm_scale;
    a->S = S;
  }
  aq.g0 = dq;
  ak.g0 = dk;
  ak.g1 = dv;
  const dim3 gq(plan->max_items, BH), gk(plan_t->max_items, BH);
  if (D == 128)
    return dtype == SVGB_BF16 ? launch_bwd_pair<128, DT_BF16>(qm, km, vm, dom, aq, gq, ak, gk, st)
                              : launch_bwd_pair<128, DT_F16>(qm, km, vm, dom, aq, gq, ak, gk, st);
  return dtype == SVGB_BF16 ? launch_bwd_pair<64, DT_BF16>(qm, km, vm, dom, aq, gq, ak, gk, st)
                            : launch_bwd_pair<64, DT_F16>(qm, km, vm, dom, aq, gq, ak, gk, st);
}

}  // extern "C"
