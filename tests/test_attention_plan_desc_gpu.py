"""Every planner writes every field of the plan descriptor: a C caller's svgb_plan need not be zeroed.

Each planner runs twice on the same device inputs, once into a descriptor filled with 0xFF bytes and once into a zeroed
one, and the two descriptors must agree field by field."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

S, SKV, BH, QC, KC = 640, 384, 2, 5, 3


def _p(t):
    return C.c_void_p(t.data_ptr())


def _cases(cuda):
    i32 = dict(dtype=torch.int32, device=cuda)
    blk = torch.ones(BH, QC, KC, dtype=torch.uint8, device=cuda)
    row, col = torch.full((BH, QC), S // QC, **i32), torch.full((BH, KC), SKV // KC, **i32)
    col_sq = torch.full((BH, KC), S // KC + 1, **i32)
    col_sq[:, -1] = S - 2 * (S // KC + 1)
    cu_q, cu_k = torch.tensor([0, 300, S], **i32), torch.tensor([0, 100, SKV], **i32)
    seqlens, cu_new = torch.tensor([200, 0], **i32), torch.tensor([0, 1, 3], **i32)
    vb = (_p(blk), _p(row), _p(col))
    return {
        "svgb_attn_plan_varblock": ("svgb_attn_plan_varblock_bytes", (BH, S, QC, KC), (_p(blk), _p(row), _p(col_sq), BH,
                                                                                       S, QC, KC)),
        "svgb_attn_plan_varblock_kv": ("svgb_attn_plan_varblock_kv_bytes", (BH, S, SKV, QC, KC),
                                       (*vb, BH, S, SKV, QC, KC)),
        "svgb_attn_plan_varblock_gather": ("svgb_attn_plan_varblock_bytes", (BH, S, QC, KC),
                                           (_p(blk), _p(row), _p(col_sq), BH, S, QC, KC)),
        "svgb_attn_plan_band": ("svgb_attn_plan_band_bytes", (S,), (10, 0, 100, 0, BH, S)),
        "svgb_attn_plan_band_t": ("svgb_attn_plan_band_t_bytes", (S,), (10, 0, 100, 0, BH, S)),
        "svgb_attn_plan_local_varlen": ("svgb_attn_plan_local_varlen_bytes", (2, S, SKV),
                                        (_p(cu_q), _p(cu_k), 2, S, SKV, 4, 64, 0)),
        "svgb_attn_plan_local_varlen_t": ("svgb_attn_plan_local_varlen_bytes", (2, S, SKV),
                                          (_p(cu_q), _p(cu_k), 2, S, SKV, 4, 64, 0)),
        "svgb_attn_plan_block_varlen": ("svgb_attn_plan_local_varlen_bytes", (2, S, SKV),
                                        (_p(cu_q), _p(cu_k), 2, S, SKV, 0, 96, 32, 16)),
        "svgb_attn_plan_block_varlen_t": ("svgb_attn_plan_local_varlen_bytes", (2, S, SKV),
                                          (_p(cu_q), _p(cu_k), 2, S, SKV, 0, 96, 32, 16)),
        "svgb_attn_plan_kvcache": ("svgb_attn_plan_kvcache_bytes", (2, 3, 512, 0, 100, 0),
                                   (_p(seqlens), None, None, 2, 3, 3, 2, 512, 0, 0, 100, 0)),
        "svgb_attn_plan_kvcache_split": ("svgb_attn_plan_kvcache_split_bytes", (2, 3, 512, 0, 100, 0, 2),
                                         (_p(seqlens), None, None, 2, 3, 3, 2, 512, 0, 0, 100, 0, 2)),
        "svgb_attn_plan_kvcache_block": ("svgb_attn_plan_kvcache_block_bytes", (2, 3, 512, 0, 96, 32, 16, 1),
                                         (_p(seqlens), None, None, 2, 3, 3, 2, 512, 0, 0, 96, 32, 16, 1)),
        "svgb_attn_plan_kvcache_varlen": ("svgb_attn_plan_kvcache_varlen_bytes", (2, 3, 2, 512, 0, 100, 0, 0, 0, 0, 2),
                                          (_p(torch.tensor([0, 1, 3], **i32)), _p(seqlens), _p(cu_new), None, None, 2, 3,
                                           2, 2, 512, 0, 0, 100, 0, 0, 0, 0, 2)),
    }, (blk, row, col, col_sq, cu_q, cu_k, seqlens, cu_new)


def test_every_planner_writes_every_field(cuda):
    from svgb200._lib import Plan, lib

    handle = lib()
    cases, keep = _cases(cuda)
    fields = [f for f, _ in Plan._fields_]
    for name, (bytes_fn, bytes_args, args) in cases.items():
        need = C.c_size_t(0)
        assert getattr(handle, bytes_fn)(*bytes_args, C.byref(need)) == 0, (name, handle.svgb_last_error())
        descs = []
        for fill in (0xFF, 0):
            ws = torch.empty(need.value, dtype=torch.uint8, device=cuda)
            plan = Plan()
            C.memset(C.byref(plan), fill, C.sizeof(plan))
            rc = getattr(handle, name)(*args, _p(ws), need.value, C.byref(plan), None)
            assert rc == 0, (name, handle.svgb_last_error())
            descs.append({f: getattr(plan, f) for f in fields})
        torch.cuda.synchronize()
        assert descs[0] == descs[1], (name, {f: (descs[0][f], descs[1][f]) for f in fields if descs[0][f] != descs[1][f]})
    del keep
