"""Host side of the attention backward without a GPU: the key-major band planner's ABI, the argument checks of
svgb_attn_bwd (every rejection happens before any device work), and the Python routing that keeps paths without a
backward from returning results detached from the autograd graph."""
import ctypes as C
from pathlib import Path

import pytest
import torch

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


def test_band_t_workspace_matches_band(lib):
    """The key-major band plan has the query-major plan's shape (items x chunk lists over S), so the same workspace."""
    a, b = C.c_size_t(), C.c_size_t()
    for S in (1, 127, 344, 4096, 119056):
        assert lib.svgb_attn_plan_band_bytes(S, C.byref(a)) == 0
        assert lib.svgb_attn_plan_band_t_bytes(S, C.byref(b)) == 0
        assert a.value == b.value
    assert lib.svgb_attn_plan_band_t_bytes(0, C.byref(b)) < 0


def _plan(kind, mode=0, S=512, BH=2):
    from svgb200._lib import Plan

    p = Plan()
    p.kind, p.BH, p.S, p.max_items, p.items_stride, p.mask_mode = kind, BH, S, 4, 0, mode
    return p


def _bwd(lib, plan, plan_t, dtype=0, D=128, S=512, ws_bytes=1 << 20):
    ptr = C.c_void_p(1 << 20)  # never dereferenced: every call here fails its argument checks
    return lib.svgb_attn_bwd(ptr, ptr, ptr, ptr, ptr, ptr, ptr, ptr, ptr, dtype, 2, S, D, D, S * D, 0.1,
                             C.byref(plan), ptr, C.byref(plan_t), ptr, ptr, ws_bytes, None)


@pytest.mark.parametrize("case,needle", [
    (dict(dtype=2), b"e4m3"),
    (dict(D=96), b"head_dim"),
    (dict(kinds=(3, 1)), b"gather"),
    (dict(kinds=(2, 2)), b"key-major"),
    (dict(kinds=(1, 4)), b"key-major"),
    (dict(mode=4), b"mask mode"),
    (dict(S_call=1024), b"plan was built"),
    (dict(ws_bytes=16), b"workspace too small"),
])
def test_bwd_argument_errors(lib, case, needle):
    kinds = case.get("kinds", (2, 4))
    mode = case.get("mode", 1)
    rc = _bwd(lib, _plan(kinds[0], mode), _plan(kinds[1], mode), dtype=case.get("dtype", 0), D=case.get("D", 128),
              S=case.get("S_call", 512), ws_bytes=case.get("ws_bytes", 1 << 20))
    assert rc < 0
    assert needle in lib.svgb_last_error(), lib.svgb_last_error()


def test_bwd_bytes(lib):
    n = C.c_size_t()
    assert lib.svgb_attn_bwd_bytes(24, 119056, C.byref(n)) == 0 and n.value >= 4 * 24 * 119056
    assert lib.svgb_attn_bwd_bytes(0, 10, C.byref(n)) < 0


def test_paths_without_backward_raise_under_grad():
    """FP8 attention, the SVG2 core (permutations, fused o_rows store) and gather / profiling plans raise SvgbError when
    an input requires grad, before any device work; without grad nothing changes (needs_grad is False)."""
    from svgb200 import core
    from svgb200._lib import Plan
    from svgb200.models import common

    x = [torch.zeros(1, 2, 256, 128, dtype=torch.bfloat16, requires_grad=True) for _ in range(3)]
    assert core.needs_grad(*x)
    with torch.no_grad():
        assert not core.needs_grad(*x)
    assert not core.needs_grad(*[t.detach() for t in x])
    with pytest.raises(core.SvgbError, match="fp8"):
        common.fp8_attention(*x, None)
    with pytest.raises(core.SvgbError, match="fp8"):
        common.sparse_flex_attention_fp8(*x, None)
    sap = common.SAPCore(0, 2, 128, 4, 8, 0.9, 0.1, 1, 1)
    with pytest.raises(core.SvgbError, match="SVG2"):
        sap.sparse_core(*x)
    for kind, mode, needle in ((core.PLAN_GATHER, 0, "gather"), (core.PLAN_BAND, core.MASK_PROF_WAN_T, "profiling")):
        d = Plan()
        d.kind, d.mask_mode = kind, mode
        with pytest.raises(core.SvgbError, match=needle):
            core.attention(*x, core.AttnPlan(d, torch.empty(0)))


def test_forward_rejects_key_major_band_plan(lib):
    """A key-major band plan holds key items and query chunk lists: the forward refuses it instead of running it."""
    ptr = C.c_void_p(1 << 20)
    rc = lib.svgb_attn_fwd(ptr, ptr, ptr, None, None, None, ptr, None, None, None, None, 0, 2, 512, 128, 128,
                           512 * 128, 128, 512 * 128, 0.1, C.byref(_plan(4, 1)), ptr, None)
    assert rc < 0
    assert b"key-major" in lib.svgb_last_error(), lib.svgb_last_error()


def test_key_major_plan_refuses_an_edited_map():
    """The key-major plan is built at the first backward from the map the plan was built from: if that map was
    modified in place since, key_major() raises instead of planning dK / dV under another mask than the forward's."""
    from svgb200 import core
    from svgb200._lib import Plan

    m = torch.ones(1, 2, 2, dtype=torch.uint8)
    r = c = torch.full((1, 2), 64, dtype=torch.int32)
    d = Plan()
    d.kind, d.BH, d.S, d.items_stride = core.PLAN_VARBLOCK, 1, 128, 0
    plan = core.AttnPlan(d, torch.empty(0), (m, r, c, (m._version, r._version, c._version)))
    m[0, 0, 1] = 0
    with pytest.raises(core.SvgbError, match="modified in place"):
        plan.key_major()
