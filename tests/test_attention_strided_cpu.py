"""Host side of attention on strided views, without a GPU: the argument checks of svgb_attn_fwd_strided /
svgb_attn_bwd_strided (every rejection happens before any device work) and, with the library calls stubbed, which entry
core reaches with which pointers and strides, and which operands it copies."""
import ctypes as C
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent
PTR = 1 << 20  # never dereferenced: every call here fails its argument checks


@pytest.fixture(scope="module")
def lib():
    import importlib.util

    spec = importlib.util.spec_from_file_location("svgb200_build", ROOT / "sparse-videogen_b200" / "build.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.build_lib()
    from svgb200 import _lib

    return _lib.lib()


def _plan(kind=1, S=300, S_kv=0, BH=4, mode=0, stride=4):
    from svgb200._lib import Plan

    p = Plan()
    p.kind, p.BH, p.S, p.m0, p.max_items, p.items_stride, p.mask_mode = kind, BH, S, S_kv, 4, stride, mode
    return p


def _st(*s):
    return (C.c_longlong * 3)(*s)


GOOD = (8 * 300 * 128, 300 * 128, 128)  # contiguous [B = 2, H = 8, S = 300, D = 128]
KV = (2 * 300 * 128, 300 * 128, 128)    # contiguous [2, 2, 300, 128]


def _fwd(lib, plan=None, dtype=0, B=2, Hq=8, Hkv=2, Sq=300, Skv=300, q=PTR, k=PTR, qs=GOOD, ks=KV, os=GOOD):
    return lib.svgb_attn_fwd_strided(q, k, PTR, PTR, None, dtype, B, Hq, Hkv, Sq, Skv, 128, _st(*qs), _st(*ks),
                                     _st(*KV), _st(*os), 0.1, C.byref(plan or _plan()), PTR, None)


def _bwd(lib, plan=None, plan_t=None, dtype=0, B=2, Hq=8, Hkv=2, qs=GOOD, dos=GOOD, dks=KV, dq=PTR):
    sts = [_st(*s) for s in (qs, KV, KV, GOOD, dos, GOOD, dks, KV)]
    return lib.svgb_attn_bwd_strided(PTR, PTR, PTR, PTR, PTR, PTR, dq, PTR, PTR, dtype, B, Hq, Hkv, 300, 300, 128, *sts,
                                     0.1, C.byref(plan or _plan()), PTR, C.byref(plan_t or _plan()), PTR, PTR, 1 << 30,
                                     None)


@pytest.mark.parametrize("case,needle", [
    (dict(qs=(0, 300 * 128, 128)), b"nonzero multiple of 8"),           # zero batch stride
    (dict(ks=(KV[0], 0, 128)), b"nonzero multiple of 8"),               # zero head stride
    (dict(os=(GOOD[0], GOOD[1], 132)), b"nonzero multiple of 8"),       # row stride not a multiple of 8
    (dict(qs=(GOOD[0] + 4, GOOD[1], 128)), b"nonzero multiple of 8"),   # batch stride not a multiple of 8
    (dict(k=PTR + 2), b"16-byte aligned"),
    (dict(plan=_plan(BH=8)), b"built over the BHkv=4"),                 # a plan over B * Hq heads
    (dict(plan=_plan(BH=2)), b"built over the BHkv=4"),                 # a plan over Hkv heads, not B * Hkv
    (dict(Hkv=3), b"multiple of the key/value heads"),
    (dict(B=0), b"bad head counts"),
    (dict(dtype=2), b"e4m3"),
    (dict(plan=_plan(kind=3)), b"gather"),
    (dict(plan=_plan(kind=2, stride=0), Skv=500), b"band plans need Sq == Skv"),
])
def test_fwd_argument_errors(lib, case, needle):
    assert _fwd(lib, **case) < 0
    assert needle in lib.svgb_last_error(), lib.svgb_last_error()


@pytest.mark.parametrize("case,needle", [
    (dict(dos=(0, 0, 0)), b"nonzero multiple of 8"),                    # the expanded dO of o.sum()
    (dict(dks=(KV[0], KV[1], 100)), b"nonzero multiple of 8"),
    (dict(dq=PTR + 8), b"16-byte aligned"),
    (dict(plan=_plan(BH=8)), b"built over the BHkv=4"),
    (dict(plan_t=_plan(BH=2)), b"plan_t is built over the B*Hkv=4"),
    (dict(dtype=2), b"e4m3"),
])
def test_bwd_argument_errors(lib, case, needle):
    assert _bwd(lib, **case) < 0
    assert needle in lib.svgb_last_error(), lib.svgb_last_error()


def test_bwd_workspace(lib):
    """The delta covers the B * Hq query heads' rows, as svgb_attn_bwd_gqa's does."""
    a, b = C.c_size_t(), C.c_size_t()
    assert lib.svgb_attn_bwd_strided_bytes(2, 40, 8, 75600, 512, C.byref(a)) == 0
    assert lib.svgb_attn_bwd_gqa_bytes(80, 16, 75600, 512, C.byref(b)) == 0
    assert a.value == b.value
    assert lib.svgb_attn_bwd_strided_bytes(0, 40, 8, 75600, 512, C.byref(a)) < 0


class _Recorder:
    """Stands in for the library: records (entry, arguments) with stride triples as tuples and returns success."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def call(*args):
            if not name.endswith("_bytes"):
                self.calls.append((name, [tuple(a) if isinstance(a, C.Array) else a for a in args]))
            return 0

        return call


@pytest.fixture
def stubbed(monkeypatch):
    from svgb200 import core

    rec = _Recorder()
    monkeypatch.setattr(core, "_need_cuda", lambda *ts: None)
    monkeypatch.setattr(core, "_stream", lambda t: 0)
    monkeypatch.setattr(core, "lib", lambda: rec)
    plan = core.AttnPlan(_plan(), torch.empty(0))
    plan._key_major = core.AttnPlan(_plan(), torch.empty(0))
    return core, rec, plan


def test_views_reach_the_strided_entries_with_their_own_strides(stubbed):
    core, rec, plan = stubbed
    B, S, H, D = 2, 300, 8, 64
    qkv = torch.zeros(B, S, 3, H, D, dtype=torch.bfloat16)
    q, k, v = (t.transpose(1, 2) for t in qkv.unbind(2))
    o, lse = core.attn_fwd(q, k, v, plan, return_lse=True)
    assert o.transpose(1, 2).is_contiguous()  # empty_like keeps the [B, S, H, D] memory order
    name, args = rec.calls[-1]
    assert name == "svgb_attn_fwd_strided"
    assert args[:4] == [q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr()]
    assert args[6:12] == [B, H, H, S, S, D]
    row = 3 * H * D
    assert args[12:15] == [(S * row, D, row)] * 3
    assert args[15] == (S * H * D, D, H * D)
    do = torch.zeros(B, S, H, D, dtype=torch.bfloat16).transpose(1, 2)
    out = tuple(torch.zeros(B, S, H, D, dtype=torch.bfloat16).transpose(1, 2) for _ in range(3))
    got = core.attn_bwd(q, k, v, o, do, lse, plan, out=out)
    assert all(g is x for g, x in zip(got, out))
    name, args = rec.calls[-1]
    assert name == "svgb_attn_bwd_strided"
    ts = (q, k, v, o, do, lse) + out
    assert args[:9] == [t.data_ptr() for t in ts]
    assert args[10:16] == [B, H, H, S, S, D]
    assert args[16:24] == [(S * row, D, row)] * 3 + [(S * H * D, D, H * D)] * 5


def test_every_other_head_and_batch_slice(stubbed):
    core, rec, plan = stubbed
    S, D = 300, 128
    x = torch.zeros(4, 16, S, D, dtype=torch.float16)
    q, k = x[:2, ::2], x[::2, :8]
    core.attn_fwd(q, k, k, plan)
    name, args = rec.calls[-1]
    assert name == "svgb_attn_fwd_strided" and args[6:9] == [2, 8, 8]
    assert args[12] == (16 * S * D, 2 * S * D, D) and args[13] == args[14] == (32 * S * D, S * D, D)


def test_copies_exactly_for_unsupported_strides(stubbed, monkeypatch):
    """Only operands the strided entry cannot address are copied: a zero stride, a last stride other than 1, a
    misaligned base; an addressable view is never copied"""
    core, rec, plan = stubbed
    copied = []
    real = torch.Tensor.clone

    def spy(t, *a, **kw):
        copied.append(tuple(t.stride()))
        return real(t, *a, **kw)

    monkeypatch.setattr(torch.Tensor, "clone", spy)
    B, H, S, D = 2, 8, 300, 128
    tr = torch.zeros(B, S, H, D, dtype=torch.bfloat16).transpose(1, 2)
    zero = torch.zeros((), dtype=torch.bfloat16).expand(B, H, S, D)
    last_s = torch.zeros(B, H, D, S, dtype=torch.bfloat16).transpose(2, 3)
    misaligned = torch.zeros(B * H * S * D + 4, dtype=torch.bfloat16)[4:].view(B, H, S, D)
    assert misaligned.data_ptr() % 16 and misaligned.is_contiguous()
    for t, want in ((tr, []), (zero, [zero.stride()]), (last_s, [last_s.stride()]), (misaligned, [misaligned.stride()])):
        copied.clear()
        core.attn_fwd(tr, t, tr, plan)
        assert copied == want
        assert rec.calls[-1][0] == "svgb_attn_fwd_strided"
        assert rec.calls[-1][1][1] != t.data_ptr() or not want
    copied.clear()
    o, lse = core.attn_fwd(tr, tr, tr, plan, return_lse=True)
    core.attn_bwd(tr, tr, tr, o, zero, lse, plan)
    assert copied == [zero.stride()]
    assert rec.calls[-1][0] == "svgb_attn_bwd_strided" and rec.calls[-1][1][4] != zero.data_ptr()


def test_contiguous_calls_keep_the_flat_entries(stubbed):
    """Contiguous operands reach svgb_attn_fwd / _kv / _gqa and svgb_attn_bwd / _kv / _gqa with the arguments they
    took before the strided entries existed"""
    core, rec, plan = stubbed
    q = torch.zeros(2, 8, 300, 128, dtype=torch.bfloat16)
    k2 = torch.zeros(2, 2, 300, 128, dtype=torch.bfloat16)
    kl = torch.zeros(2, 8, 500, 128, dtype=torch.bfloat16)
    plan_kv = core.AttnPlan(_plan(S_kv=500, BH=16), torch.empty(0))
    plan_kv._key_major = plan_kv
    for kk, p, fwd, bwd in ((q, plan, "svgb_attn_fwd", "svgb_attn_bwd"), (k2, plan, "svgb_attn_fwd_gqa",
                                                                         "svgb_attn_bwd_gqa"),
                            (kl, plan_kv, "svgb_attn_fwd_kv", "svgb_attn_bwd_kv")):
        o, lse = core.attn_fwd(q, kk, kk, p, return_lse=True)
        assert o.is_contiguous() and rec.calls[-1][0] == fwd
        args = rec.calls[-1][1]
        assert (300 * 128) in args and 128 in args and not any(isinstance(a, tuple) for a in args)
        core.attn_bwd(q, kk, kk, o, q, lse, p)
        assert rec.calls[-1][0] == bwd
        assert not any(isinstance(a, tuple) for a in rec.calls[-1][1])
    # the square forward's exact argument list: the (row, head) pair of q, k / v and o
    core.attn_fwd(q, q, q, plan)
    args = rec.calls[-1][1]
    assert args[11:19] == [0, 16, 300, 128, 128, 300 * 128, 128, 300 * 128]


def test_row_vectors_and_gather_plans_refuse_views(stubbed):
    core, rec, plan = stubbed
    tr = torch.zeros(1, 300, 8, 128, dtype=torch.bfloat16).transpose(1, 2)
    rows = torch.zeros(8, 300, dtype=torch.int32)
    with pytest.raises(core.SvgbError, match="q, k, v must be contiguous"):
        core.attn_fwd(tr, tr, tr, plan, o_rows=rows)
    gather = core.AttnPlan(_plan(kind=3, BH=8), torch.empty(0))
    with pytest.raises(core.SvgbError, match="q, k, v must be contiguous"):
        core.attn_fwd(tr, tr, tr, gather)
    c = tr.contiguous()
    with pytest.raises(core.SvgbError, match="out must be contiguous"):
        core.attn_fwd(c, c, c, plan, o_rows=rows, out=tr)
