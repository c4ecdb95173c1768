"""FP8 mode without a GPU: argument errors of svgb_attn_fwd for e4m3 inputs and row gathers, the head-dim check of the
cores, and which operators patch.install(..., fp8=) puts in place."""
import ctypes as C
import types
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent


@pytest.fixture(scope="module")
def lib():
    import importlib.util

    spec = importlib.util.spec_from_file_location("svgb200_build", ROOT / "sparse-videogen_b200" / "build.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.build_lib()
    from svgb200 import _lib

    return _lib.lib()


SVGB_BF16, SVGB_E4M3 = 0, 2


def _call(lib, plan, scales=True, rows=False, dtype=SVGB_E4M3):
    p = C.c_void_p(4096)  # never dereferenced: the arguments are rejected first
    s = p if scales else None
    r = p if rows else None
    return lib.svgb_attn_fwd(p, p, p, s, s, s, p, None, r, r, None, dtype, 1, 1024, 128, 128, 1024 * 128,
                             128, 1024 * 128, 0.088, C.byref(plan), p, None)


def test_attn_fwd_e4m3_argument_errors(lib):
    from svgb200._lib import Plan
    from svgb200.core import PLAN_BAND, PLAN_GATHER, PLAN_VARBLOCK

    plan = Plan(kind=PLAN_GATHER, BH=1, S=1024, max_items=4, items_stride=4)
    assert _call(lib, plan, scales=False, rows=True) < 0
    assert b"scale" in lib.svgb_last_error()
    for kind in (PLAN_VARBLOCK, PLAN_BAND):
        plan.kind = kind
        assert _call(lib, plan, rows=True) < 0
        assert b"svgb_attn_plan_varblock_gather" in lib.svgb_last_error()


def test_scales_are_rejected_with_16bit_inputs(lib):
    from svgb200._lib import Plan
    from svgb200.core import PLAN_VARBLOCK

    plan = Plan(kind=PLAN_VARBLOCK, BH=1, S=1024, max_items=4, items_stride=4)
    assert _call(lib, plan, dtype=SVGB_BF16) < 0
    assert b"scale" in lib.svgb_last_error()


def test_cores_reject_head_dim_64_in_fp8():
    import torch

    from svgb200 import core
    from svgb200.models import wan
    from svgb200.models.common import sparse_flex_attention_fp8

    q = torch.zeros(1, 2, 256, 64, dtype=torch.bfloat16)
    sap = wan.WanSAPCore(4, 64, num_q_centroids=4, num_k_centroids=8, top_p_kmeans=0.9, min_kc_ratio=0.1,
                         kmeans_iter_init=2, kmeans_iter_step=1, fp8=True)
    with pytest.raises(core.SvgbError, match="head_dim 128"):
        sap.sparse_core(q, q, q)
    with pytest.raises(core.SvgbError, match="head_dim 128"):
        sparse_flex_attention_fp8(q, q, q, None)


def _stand_in():
    m = types.ModuleType("svg.models.hyvideo.attention")
    for name in ("flex_attention", "dynamic_block_sparse_fwd_flashinfer", "dynamic_block_sparse_fwd_triton"):
        setattr(m, name, None)
    return m


def test_install_selects_the_fp8_operators():
    from svgb200 import kmeans_utils as ku
    from svgb200 import patch

    m = _stand_in()
    patch.install(m)
    assert m.flex_attention is patch.flex_attention
    assert m.dynamic_block_sparse_fwd_flashinfer is ku.dynamic_block_sparse_fwd_flashinfer
    assert m.dynamic_block_sparse_fwd_triton is ku.dynamic_block_sparse_fwd_triton
    m = _stand_in()
    done = patch.install(m, fp8=True)
    assert m.flex_attention is patch.flex_attention_fp8
    assert m.dynamic_block_sparse_fwd_flashinfer is ku.dynamic_block_sparse_fwd_flashinfer_fp8
    assert m.dynamic_block_sparse_fwd_triton is ku.dynamic_block_sparse_fwd_triton_fp8
    assert {"flex_attention", "dynamic_block_sparse_fwd_flashinfer", "dynamic_block_sparse_fwd_triton"} <= set(done)
