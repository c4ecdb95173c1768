"""Host side of grouped-query attention (fewer key/value heads than query heads) without a GPU: the argument checks
of svgb_attn_fwd_gqa / svgb_attn_bwd_gqa (every rejection happens before any device work), the Python refusals and
head routing, and the fp64 oracle the GPU tests compare against."""
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


def _plan(kind=1, S=300, S_kv=0, BH=2, mode=0, stride=4):
    from svgb200._lib import Plan

    p = Plan()
    p.kind, p.BH, p.S, p.m0, p.max_items, p.items_stride, p.mask_mode = kind, BH, S, S_kv, 4, stride, mode
    return p


def _fwd(lib, plan, dtype=0, BHq=8, BHkv=2, Sq=300, Skv=300):
    return lib.svgb_attn_fwd_gqa(PTR, PTR, PTR, PTR, None, dtype, BHq, BHkv, Sq, Skv, 128, 128, Sq * 128, 128,
                                 Skv * 128, 128, Sq * 128, 0.1, C.byref(plan), PTR, None)


def _bwd(lib, plan, plan_t, dtype=0, BHq=8, BHkv=2, Sq=300, Skv=300):
    return lib.svgb_attn_bwd_gqa(PTR, PTR, PTR, PTR, PTR, PTR, PTR, PTR, PTR, dtype, BHq, BHkv, Sq, Skv, 128, 128,
                                 Sq * 128, 128, Skv * 128, 0.1, C.byref(plan), PTR, C.byref(plan_t), PTR, PTR, 1 << 20,
                                 None)


ERRORS = [
    (dict(BHq=8, BHkv=3), b"multiple of the key/value heads"),
    (dict(BHkv=0), b"multiple of the key/value heads"),
    (dict(plan=_plan(BH=8)), b"built over the BHkv=2"),          # a plan over the query heads
    (dict(dtype=2), b"e4m3"),
    (dict(plan=_plan(kind=3)), b"gather"),
    (dict(plan=_plan(kind=4, stride=0)), b"key-major"),
    (dict(plan=_plan(kind=2, stride=0), Skv=500), b"band plans need Sq == Skv"),
    (dict(plan=_plan(S_kv=500)), b"plan was built"),            # a rectangular plan called at Sq == Skv
]


@pytest.mark.parametrize("case,needle", ERRORS)
def test_fwd_gqa_argument_errors(lib, case, needle):
    case = dict(case)
    plan = case.pop("plan", _plan())
    assert _fwd(lib, plan, **case) < 0
    assert needle in lib.svgb_last_error(), lib.svgb_last_error()


@pytest.mark.parametrize("case,needle", ERRORS + [
    (dict(plans=(_plan(), _plan(BH=8))), b"plan_t BH=8"),         # key-major plan over the query heads
    (dict(plans=(_plan(kind=2, mode=6, stride=0), _plan(kind=4, mode=6, stride=0))), b"mask mode 6"),
])
def test_bwd_gqa_argument_errors(lib, case, needle):
    case = dict(case)
    plan, plan_t = case.pop("plans", (case.pop("plan", _plan()), _plan()))
    assert _bwd(lib, plan, plan_t, **case) < 0
    assert needle in lib.svgb_last_error(), lib.svgb_last_error()


def test_bwd_gqa_workspace(lib):
    """The delta covers the BHq query heads' rows, as svgb_attn_bwd_kv's does."""
    a, b = C.c_size_t(), C.c_size_t()
    assert lib.svgb_attn_bwd_gqa_bytes(40, 8, 75600, 512, C.byref(a)) == 0
    assert lib.svgb_attn_bwd_kv_bytes(40, 75600, 512, C.byref(b)) == 0
    assert a.value == b.value
    assert lib.svgb_attn_bwd_gqa_bytes(40, 0, 75600, 512, C.byref(a)) < 0


@pytest.fixture
def host_only(monkeypatch):
    """core with CPU tensors accepted and the library unreachable: a call that gets as far as device work fails."""
    from svgb200 import core

    def no_lib():
        raise AssertionError("reached the library")

    monkeypatch.setattr(core, "_need_cuda", lambda *ts: None)
    monkeypatch.setattr(core, "lib", no_lib)
    return core


def test_geometry_accepts_head_groups_only(host_only):
    core = host_only
    q = torch.zeros(2, 8, 300, 64)
    for layout, qq, kk in (("bhsd", q, torch.zeros(2, 2, 500, 64)), ("shd", q[0].transpose(0, 1),
                                                                      torch.zeros(500, 2, 64))):
        BH, Sq, Skv, D, qs, kvs = core._kv_geometry(qq, kk, layout)
        assert (BH, Sq, Skv, D, core._kv_group(qq, kk)) == ((16 if layout == "bhsd" else 8), 300, 500, 64, 4)
    for k in (torch.zeros(2, 3, 300, 64), torch.zeros(2, 16, 300, 64), torch.zeros(2, 2, 300, 128),
              torch.zeros(1, 2, 300, 64)):
        with pytest.raises(core.SvgbError, match="may differ in the sequence length only, and in a key/value head count"):
            core._kv_geometry(q, k, "bhsd")
    k3 = torch.zeros(2, 3, 300, 64, dtype=torch.bfloat16)
    with pytest.raises(core.SvgbError, match="may differ"):
        core.attn_fwd(q.bfloat16(), k3, k3, core.AttnPlan(_plan(), None))


def test_python_refusals_before_device_work(host_only):
    """Row vectors, FP8 and gather plans name GQA; a D mismatch is still refused."""
    core = host_only
    q, k = torch.zeros(1, 8, 300, 128, dtype=torch.bfloat16), torch.zeros(1, 2, 300, 128, dtype=torch.bfloat16)
    vb, gather = core.AttnPlan(_plan(BH=2), None), core.AttnPlan(_plan(kind=3, BH=2), None)
    rows = torch.zeros(8, 300, dtype=torch.int32)
    for kw in (dict(o_rows=rows), dict(q_rows=rows), dict(kv_rows=rows)):
        with pytest.raises(core.SvgbError, match="grouped-query attention .* row vectors"):
            core.attn_fwd(q, k, k, vb, **kw)
    with pytest.raises(core.SvgbError, match="grouped-query attention .* gather plan"):
        core.attn_fwd(q, k, k, gather)
    with pytest.raises(core.SvgbError, match="grouped-query attention .* gather plan"):
        core.attn_bwd(q, k, k, q, q, torch.zeros(8, 300), gather)
    q8, k8 = q.view(torch.uint8)[..., :128], k.view(torch.uint8)[..., :128]
    s = torch.ones(8)
    with pytest.raises(core.SvgbError, match="grouped-query attention .* FP8"):
        core.attn_fwd_fp8(q8, k8, k8, s, s[:2], s[:2], vb)
    k64 = torch.zeros(1, 2, 300, 64, dtype=torch.bfloat16)
    with pytest.raises(core.SvgbError, match="may differ"):
        core.attn_fwd(q, k64, k64, vb)
    with pytest.raises(core.SvgbError, match="may differ"):
        core.attn_bwd(q, torch.zeros(1, 3, 300, 128, dtype=torch.bfloat16),
                      torch.zeros(1, 3, 300, 128, dtype=torch.bfloat16), q, q, torch.zeros(8, 300), vb)


def test_segment_map_is_built_over_key_heads(monkeypatch):
    """segment_attention plans its diagonal map over k's heads, so GQA k, v reach core.attention with a plan the
    grouped launch accepts (plan BH = key/value heads), in both layouts."""
    from svgb200 import core
    from svgb200.models import common

    seen = []
    monkeypatch.setattr(core, "plan_varblock", lambda bm, r, c, S, S_kv=None: seen.append(bm.shape[0]) or "plan")
    monkeypatch.setattr(core, "attention", lambda q, k, v, plan, layout="bhsd": (q.shape, k.shape, plan))
    q, k = torch.zeros(2, 8, 300, 64), torch.zeros(2, 2, 300, 64)
    common.dense_attention(q, k, k, [100, 200])
    common.segment_attention("t", q[0].transpose(0, 1), k[0].transpose(0, 1), k[0].transpose(0, 1), [300], [300],
                             layout="shd")
    assert seen == [4, 2]


def test_oracle_group_sums():
    """gqa_grads against explicit per-query-head autograd on repeated K / V: o and dq per head, dk / dv of a key/value
    head the sum over its group's query heads, and G = 1 the plain masked softmax."""
    import gqa_fp64

    g = torch.Generator().manual_seed(0)
    Hq, Hkv, Sq, Skv, D = 6, 2, 37, 53, 16
    q, do = (torch.randn(Hq, Sq, D, generator=g, dtype=torch.float64) for _ in range(2))
    k, v = (torch.randn(Hkv, Skv, D, generator=g, dtype=torch.float64) for _ in range(2))
    masks = torch.rand(Hq, Sq, Skv, generator=g) < 0.4
    masks[:, 3] = False  # a row without keys
    o, dq, dk, dv = gqa_fp64.gqa_grads(q, k, v, do, masks, sm_scale=0.3)
    G = Hq // Hkv
    dk_sum, dv_sum = torch.zeros_like(k), torch.zeros_like(v)
    for h in range(Hq):
        x = [t.clone().requires_grad_() for t in (q[h], k[h // G], v[h // G])]
        s = (x[0] @ x[1].T * 0.3).masked_fill(~masks[h], float("-inf"))
        oh = torch.nan_to_num(torch.softmax(s, -1), nan=0.0) @ x[2]
        oh.backward(do[h])
        torch.testing.assert_close(o[h], oh.detach(), rtol=0, atol=1e-12)
        torch.testing.assert_close(dq[h], x[0].grad, rtol=0, atol=1e-12)
        dk_sum[h // G] += x[1].grad
        dv_sum[h // G] += x[2].grad
    torch.testing.assert_close(dk, dk_sum, rtol=0, atol=1e-12)
    torch.testing.assert_close(dv, dv_sum, rtol=0, atol=1e-12)
    assert float(o[:, 3].abs().max()) == 0.0 and float(dq[:, 3].abs().max()) == 0.0
    sq = masks[..., :Sq]
    o1 = gqa_fp64.gqa_attention(q, q, do, sq)  # G = 1
    s = (q @ q.transpose(1, 2) * D ** -0.5).masked_fill(~sq, float("-inf"))
    torch.testing.assert_close(o1, torch.nan_to_num(torch.softmax(s, -1), nan=0.0) @ do, rtol=0, atol=0)
