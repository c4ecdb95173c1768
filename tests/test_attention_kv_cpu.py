"""Host side of attention with a key/value length Skv other than the query length Sq, without a GPU: the rectangular
planner's workspace, the argument checks of svgb_attn_fwd_kv / svgb_attn_bwd_kv and of the square entries against a
rectangular plan (every rejection happens before any device work), and the Python routing of lengths and segments."""
import ctypes as C
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent
PTR = C.c_void_p(1 << 20)  # never dereferenced: every call here fails its argument checks


@pytest.fixture(scope="module")
def lib():
    import importlib.util

    spec = importlib.util.spec_from_file_location("svgb200_build", ROOT / "sparse-videogen_b200" / "build.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.build_lib()
    from svgb200 import _lib

    return _lib.lib()


def _plan(kind=1, S=300, S_kv=0, BH=2, mode=0):
    from svgb200._lib import Plan

    p = Plan()
    p.kind, p.BH, p.S, p.m0, p.max_items, p.items_stride, p.mask_mode = kind, BH, S, S_kv, 4, 4, mode
    return p


def test_plan_workspace(lib):
    """The rectangular planner's workspace is the square planner's at Sq == Skv; its items grow with Sq and its chunk
    lists with Skv; zero lengths are bad arguments."""
    a, b = C.c_size_t(), C.c_size_t()
    for BH, S, QC, KC in ((1, 1, 1, 1), (24, 119056, 402, 1002), (40, 75600, 21, 3)):
        assert lib.svgb_attn_plan_varblock_bytes(BH, S, QC, KC, C.byref(a)) == 0
        assert lib.svgb_attn_plan_varblock_kv_bytes(BH, S, S, QC, KC, C.byref(b)) == 0
        assert a.value == b.value
    lib.svgb_attn_plan_varblock_kv_bytes(40, 75600, 512, 1, 1, C.byref(a))
    lib.svgb_attn_plan_varblock_kv_bytes(40, 75600, 75600, 1, 1, C.byref(b))
    assert a.value < b.value
    lib.svgb_attn_plan_varblock_kv_bytes(40, 512, 75600, 100, 1, C.byref(a))
    lib.svgb_attn_plan_varblock_kv_bytes(40, 75600, 75600, 100, 1, C.byref(b))
    assert a.value < b.value
    for args in ((2, 100, 0, 1, 1), (2, 0, 100, 1, 1)):
        assert lib.svgb_attn_plan_varblock_kv_bytes(*args, C.byref(a)) < 0
        assert b"bad arguments" in lib.svgb_last_error()
    n = C.c_size_t()
    assert lib.svgb_attn_bwd_kv_bytes(40, 75600, 512, C.byref(n)) == 0 and n.value >= 4 * 40 * 75600
    assert lib.svgb_attn_bwd_kv_bytes(40, 75600, 0, C.byref(n)) < 0


def _fwd_kv(lib, plan, dtype=0, Sq=300, Skv=500, D=128, q=PTR, k=PTR, q_rs=128, kv_rs=128, kv_hs=500 * 128):
    return lib.svgb_attn_fwd_kv(q, k, PTR, PTR, None, dtype, 2, Sq, Skv, D, q_rs, Sq * 128, kv_rs, kv_hs, 128,
                                Sq * 128, 0.1, C.byref(plan), PTR, None)


@pytest.mark.parametrize("case,needle", [
    (dict(plan=_plan(kind=2)), b"variable-block plans only"),          # band
    (dict(plan=_plan(kind=3)), b"variable-block plans only"),          # gather
    (dict(plan=_plan(kind=4)), b"variable-block plans only"),          # key-major band
    (dict(plan=_plan(kind=2, mode=6)), b"variable-block plans only"),  # profiling
    (dict(dtype=2), b"e4m3"),
    (dict(plan=_plan(S_kv=600)), b"plan was built"),                  # recorded Skv differs from the call's
    (dict(plan=_plan(S=200, S_kv=500)), b"plan was built"),
    (dict(plan=_plan(S_kv=0)), b"plan was built"),                    # a square plan for S = 300
    (dict(kv_rs=100), b"multiple of 8"),
    (dict(kv_hs=500 * 128 + 4), b"multiple of 8"),
    (dict(q_rs=132), b"multiple of 8"),
    (dict(k=C.c_void_p((1 << 20) + 2)), b"16-byte aligned"),
])
def test_fwd_kv_argument_errors(lib, case, needle):
    plan = case.pop("plan", _plan(S_kv=500))
    assert _fwd_kv(lib, plan, **case) < 0
    assert needle in lib.svgb_last_error(), lib.svgb_last_error()


def test_square_entries_reject_a_rectangular_plan(lib):
    """svgb_attn_fwd / svgb_attn_bwd at S = Sq with a plan that records another Skv refuse it (they would read k, v
    over the wrong length)."""
    rc = lib.svgb_attn_fwd(PTR, PTR, PTR, None, None, None, PTR, None, None, None, None, 0, 2, 300, 128, 128, 300 * 128,
                           128, 300 * 128, 0.1, C.byref(_plan(S_kv=500)), PTR, None)
    assert rc < 0 and b"plan was built" in lib.svgb_last_error()
    rc = lib.svgb_attn_bwd(PTR, PTR, PTR, PTR, PTR, PTR, PTR, PTR, PTR, 0, 2, 300, 128, 128, 300 * 128, 0.1,
                           C.byref(_plan(S_kv=500)), PTR, C.byref(_plan(S=500, S_kv=300)), PTR, PTR, 1 << 20, None)
    assert rc < 0 and b"plan was built" in lib.svgb_last_error()


def _bwd_kv(lib, plan, plan_t, dtype=0, Sq=300, Skv=500, D=128, kv_rs=128, ws_bytes=1 << 20):
    return lib.svgb_attn_bwd_kv(PTR, PTR, PTR, PTR, PTR, PTR, PTR, PTR, PTR, dtype, 2, Sq, Skv, D, 128, Sq * 128, kv_rs,
                                Skv * 128, 0.1, C.byref(plan), PTR, C.byref(plan_t), PTR, PTR, ws_bytes, None)


@pytest.mark.parametrize("case,needle", [
    (dict(plans=(_plan(kind=2, mode=1), _plan(kind=4, mode=1))), b"variable-block plans only"),
    (dict(plans=(_plan(kind=3, S_kv=500), _plan(S=500, S_kv=300))), b"variable-block plans only"),
    (dict(dtype=2), b"e4m3"),
    (dict(D=96), b"head_dim"),
    (dict(plans=(_plan(S_kv=500), _plan(kind=4, S=500))), b"key-major"),
    (dict(Skv=600), b"plan was built"),
    # the key-major plan built with the lengths swapped: its rows must be the Skv keys, its chunks the Sq queries
    (dict(plans=(_plan(S_kv=500), _plan(S=300, S_kv=500))), b"plan_t was built"),
    (dict(plans=(_plan(S_kv=500), _plan(S=500, S_kv=0))), b"plan_t was built"),
    (dict(kv_rs=100), b"multiple of 8"),
    (dict(ws_bytes=16), b"workspace too small"),
])
def test_bwd_kv_argument_errors(lib, case, needle):
    plan, plan_t = case.pop("plans", (_plan(S_kv=500), _plan(S=500, S_kv=300)))
    assert _bwd_kv(lib, plan, plan_t, **case) < 0
    assert needle in lib.svgb_last_error(), lib.svgb_last_error()


def test_key_major_plan_swaps_the_lengths(monkeypatch):
    """AttnPlan.key_major() of a rectangular plan plans the transposed map with the sizes and the lengths swapped:
    (map^T, col_sz, row_sz, S = Skv, S_kv = Sq)."""
    from svgb200 import core

    m = torch.ones(2, 3, 4, dtype=torch.uint8)
    r, c = torch.full((2, 3), 100, dtype=torch.int32), torch.full((2, 4), 128, dtype=torch.int32)
    plan = core.AttnPlan(_plan(S=300, S_kv=512), torch.empty(0), (m, r, c, (m._version, r._version, c._version)))
    assert plan.S == 300 and plan.S_kv == 512
    assert core.AttnPlan(_plan(S=300), torch.empty(0)).S_kv == 300
    seen = {}

    def fake(bm, rs, cs, S, gather=False, *, S_kv=None):
        seen.update(bm=bm, rs=rs, cs=cs, S=S, S_kv=S_kv)
        return core.AttnPlan(_plan(S=S, S_kv=S_kv), torch.empty(0))

    monkeypatch.setattr(core, "plan_varblock", fake)
    plan.key_major()
    assert seen["S"] == 512 and seen["S_kv"] == 300
    assert seen["rs"] is c and seen["cs"] is r and torch.equal(seen["bm"], m.transpose(1, 2))


def test_segments_must_pair_up():
    """dense_attention and the varlen mirrors check what the host can see: one key segment per query segment, and
    segment sums equal to the lengths, before any device work."""
    from svgb200 import core, patch
    from svgb200.models import common

    q = torch.zeros(1, 2, 300, 64, dtype=torch.bfloat16)
    k = torch.zeros(1, 2, 100, 64, dtype=torch.bfloat16)
    with pytest.raises(core.SvgbError, match="need kv_seg_lens"):
        common.dense_attention(q, k, k, [100, 200])
    with pytest.raises(core.SvgbError, match="must sum"):
        common.dense_attention(q, k, k, [100, 200], [50, 40])
    with pytest.raises(core.SvgbError, match="must sum"):
        common.dense_attention(q, k, k, [100, 100], [50, 50])
    with pytest.raises(core.SvgbError, match="one key segment per query segment"):
        common.dense_attention(q, k, k, [100, 200], [100])
    with pytest.raises(core.SvgbError, match="must sum"):  # equal lists, but the keys are 100 long
        common.dense_attention(q, k, k, [100, 200], [100, 200])
    cu_q = torch.tensor([0, 100, 300], dtype=torch.int32)
    qs, ks = q[0].transpose(0, 1).contiguous(), k[0].transpose(0, 1).contiguous()  # [S, H, D]
    for cu_kv in (cu_q, cu_q.clone(), torch.tensor([0, 50, 150], dtype=torch.int32)):
        with pytest.raises(core.SvgbError, match="must sum"):
            patch.flash_attn_varlen_func(qs, ks, ks, cu_q, cu_kv, 200, 200)
        with pytest.raises(core.SvgbError, match="must sum"):
            patch.flashinfer_varlen_func(q, k, k, cu_q, cu_kv, 200, 200)
    with pytest.raises(core.SvgbError, match="same number of segments"):
        patch.flashinfer_varlen_func(q, k, k, cu_q, torch.tensor([0, 100], dtype=torch.int32), 200, 100)
    assert patch._varlen_segments(cu_q, cu_q.clone()) == ([100, 200], [100, 200])
    assert patch._varlen_segments(torch.tensor([0, 0, 100, 300]), torch.tensor([0, 0, 40, 40])) == ([100, 200], [40, 0])

