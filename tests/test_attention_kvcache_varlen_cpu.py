"""Variable-length KV-cache plans and appends without a GPU: the workspace formula and the item bound over adversarial
length mixes, the ABI refusals by name, the Python refusals before any launch, and the drop-in's mapping of
FlashAttention 3's cu_seqlens_q / cu_seqlens_k_new / max_seqlen_q to core calls."""
import ctypes as C
import random

import pytest
import torch

from test_attention_local_cpu import PTR, lib  # noqa: F401  (lib: the module-scoped library fixture)


def _align16(x):
    return (x + 15) // 16 * 16


def _items(B, total_q, max_q):
    """the host bound I of include/svgb200.h, svgb_attn_plan_kvcache_varlen"""
    return min(B * -(-max_q // 256), (total_q + 255 * B) // 256)


def _want_bytes(B, total_q, max_q, cap, sink, left, right, n):
    I = _items(B, total_q, max_q)
    slots = min(-(-cap // 128), -(-sink // 128) + (255 + left + right) // 128 + 2)
    return 16 + _align16(4 * (2 * B + 3)) + 32 * n * I + 8 * n * I * -(-slots // n)


def _bytes(lib, *a):
    nb = C.c_size_t()
    assert lib.svgb_attn_plan_kvcache_varlen_bytes(*a, C.byref(nb)) == 0, lib.svgb_last_error()
    return nb.value


def test_workspace_formula(lib):
    for B, Tq, mq, cap, sink, left, right, n in [(4, 4 * 257, 257, 32760, 0, 40000, 0, 1),
                                                  (5, 1, 1, 1300, 70, 300, 0, 3), (1, 4680, 4680, 37440, 1560, 14040, 0, 2),
                                                  (64, 64, 1, 131072, 0, 131072, 0, 10), (3, 1000, 900, 128, 0, 0, 0, 1)]:
        assert _bytes(lib, B, Tq, mq, cap, sink, left, right, 0, 0, 0, n) == \
            _want_bytes(B, Tq, mq, cap, sink, left, right, n), (B, Tq, mq)
    # block-causal: the slot bound of left = W - 1, right = C - 1
    assert _bytes(lib, 3, 900, 600, 5000, 30, 0, 0, 320, 96, 40, 2) == _want_bytes(3, 900, 600, 5000, 30, 319, 95, 2)


def test_item_bound_holds_on_adversarial_mixes():
    """sum over streams of ceil(Lq_b / 256) never exceeds I, whatever the mix with that total and longest stream; both
    terms of the min are reached."""
    rng = random.Random(0)
    mixes = [[257] * 8, [256] * 8, [1] * 300, [0] * 7 + [4680], [255, 257] * 5, [1, 256, 257, 0, 513]]
    for _ in range(2000):
        B = rng.randint(1, 40)
        mixes.append([rng.choice([0, 1, 255, 256, 257, 511, 512, 513, rng.randint(0, 3000)]) for _ in range(B)])
    for lq in mixes:
        if not sum(lq):
            continue
        need = sum(-(-x // 256) for x in lq)
        assert need <= _items(len(lq), sum(lq), max(lq)), lq
    assert _items(8, 8 * 257, 257) == 16 == sum(-(-257 // 256) for _ in range(8))  # every stream at 257: tight
    assert _items(4, 1024, 256) == 4 < (1024 + 255 * 4) // 256  # the longest stream bounds it
    assert _items(8, 4680, 4680) == (4680 + 255 * 8) // 256 < 8 * 19  # the total bounds it


def _plan_args(**kw):
    a = dict(cu_q=PTR, seqlens=PTR, cu_new=None, bi=None, bt=None, B=3, Tq=100, mq=50, nb=4, rows=512, mp=0, sink=0,
             left=10, right=0, W=0, Cb=0, F=0, n=1, ws=PTR, wsb=1 << 30)
    a.update(kw)
    return a


def _plan_call(lib, **kw):
    a = _plan_args(**kw)
    plan = __import__("svgb200._lib", fromlist=["Plan"]).Plan()
    rc = lib.svgb_attn_plan_kvcache_varlen(a["cu_q"], a["seqlens"], a["cu_new"], a["bi"], a["bt"], a["B"], a["Tq"],
                                           a["mq"], a["nb"], a["rows"], a["mp"], a["sink"], a["left"], a["right"],
                                           a["W"], a["Cb"], a["F"], a["n"], a["ws"], a["wsb"], C.byref(plan), None)
    return rc, lib.svgb_last_error().decode()


@pytest.mark.parametrize("kw,needle", [
    (dict(cu_q=None), "null pointer"), (dict(seqlens=None), "null pointer"),
    (dict(B=0), "bad arguments"), (dict(Tq=0, mq=0), "bad arguments"),
    (dict(mq=0), "max_q"), (dict(mq=101), "max_q"), (dict(n=0), "num_splits"),
    (dict(W=5), "window and first_block must be 0"), (dict(F=3), "window and first_block must be 0"),
    (dict(left=-1), "must be >= 0"), (dict(sink=-2), "must be >= 0"),
    (dict(Cb=96, F=40, W=320), "left and right must be 0"),
    (dict(Cb=96, F=97, W=320, left=0), "first_block"), (dict(Cb=96, F=40, W=50, left=0), "window W"),
    (dict(Cb=70000, F=1, W=70000, left=0), "block C"),
    (dict(wsb=64), "workspace too small"), (dict(nb=0), "bad cache geometry"),
    (dict(bt=PTR, rows=500, mp=4), "multiple of 128"),
])
def test_planner_refusals(lib, kw, needle):
    rc, msg = _plan_call(lib, **kw)
    assert rc < 0 and needle in msg, msg
    assert "svgb_attn_plan_kvcache_varlen" in msg or needle in ("null pointer", "workspace too small")


def test_bytes_refusals(lib):
    nb = C.c_size_t()
    assert lib.svgb_attn_plan_kvcache_varlen_bytes(2, 10, 11, 1000, 0, 5, 0, 0, 0, 0, 1, C.byref(nb)) < 0
    assert b"svgb_attn_plan_kvcache_varlen_bytes: max_q" in lib.svgb_last_error()
    assert lib.svgb_attn_plan_kvcache_varlen_bytes(2, 10, 5, 1000, 0, 5, 0, 0, 96, 40, 1, C.byref(nb)) < 0
    assert b"left and right must be 0" in lib.svgb_last_error()


def _append_call(lib, cu_new=PTR, ks=None, vs=None, rows=0, B=2, T=10, D=128, nrows=512):
    st = (C.c_longlong * 3)(1024, 128, 256)
    return lib.svgb_kvcache_append_varlen(PTR, PTR, PTR, PTR, cu_new, PTR, None, None, 0, B, T, 2, D, 4, nrows, 0, st,
                                          st, st, st, ks, vs, rows, None), lib.svgb_last_error().decode()


@pytest.mark.parametrize("kw,needle", [
    (dict(cu_new=None), "needs cu_new"), (dict(B=0), "bad stream count"), (dict(T=0), "no new rows"),
    (dict(ks=PTR), "both scale vectors"), (dict(rows=1), "per-row scale tensors"),
    (dict(ks=PTR, vs=PTR, rows=1, nrows=510), "multiple of 4"), (dict(D=96), "head_dim 96"),
])
def test_append_refusals(lib, kw, needle):
    rc, msg = _append_call(lib, **kw)
    assert rc < 0 and "svgb_kvcache_append_varlen" in msg and needle in msg, msg


class _T:
    """a stand-in CUDA tensor: what the Python layer inspects before a launch"""
    is_cuda = True
    dtype = torch.int32
    device = "cuda:0"

    def __init__(self, *shape, requires_grad=False):
        self.shape = torch.Size(shape)
        self.requires_grad = requires_grad

    def dim(self):
        return len(self.shape)

    def numel(self):
        n = 1
        for x in self.shape:
            n *= x
        return n

    def is_floating_point(self):
        return False

    def to(self, *a, **kw):
        return self

    def contiguous(self):
        return self

    def data_ptr(self):
        return 0


@pytest.mark.parametrize("kw,needle", [
    (dict(q_len=4, cu_seqlens_q=_T(4)), "exactly one"), (dict(), "exactly one"),
    (dict(q_len=4, cu_seqlens_new=_T(4)), "goes with cu_seqlens_q"),
    (dict(cu_seqlens_q=_T(4)), "needs total_q"),
    (dict(cu_seqlens_q=_T(4), total_q=9, cu_seqlens_new=_T(4), new_len=2), "both give the appended rows"),
    (dict(cu_seqlens_q=_T(4), total_q=0), "total_q=0"),
    (dict(cu_seqlens_q=_T(4), total_q=9, max_seqlen_q=10), "max_seqlen_q=10"),
    (dict(cu_seqlens_q=_T(1), total_q=9), r"B \+ 1 >= 2"),
    (dict(cu_seqlens_q=_T(4), total_q=9, block=4, causal=True), "causal=True"),
])
def test_plan_refusals_before_launch(monkeypatch, kw, needle):
    from svgb200 import core
    from svgb200._lib import SvgbError

    calls = []
    monkeypatch.setattr(core, "lib", lambda: calls.append(1))
    monkeypatch.setattr(core, "_cu_seqlens", lambda who, name, cu, B, dev: _check_len(who, name, cu, B))
    with pytest.raises(SvgbError, match=needle):
        core.plan_kvcache(5, num_blocks=4, cache_len=1000, **kw)
    assert calls == []


def _check_len(who, name, cu, B):
    from svgb200._lib import SvgbError

    if cu.numel() < 2 or (B is not None and cu.numel() != B + 1):
        raise SvgbError(f"{who}: {name} must be a 1-D int tensor of B + 1 >= 2 entries")
    return cu


def test_cpu_bounds_refused_by_name():
    from svgb200 import core
    from svgb200._lib import SvgbError

    with pytest.raises(SvgbError, match="cu_seqlens_q is on the CPU"):
        core.plan_kvcache(5, cu_seqlens_q=torch.tensor([0, 3, 5], dtype=torch.int32), total_q=5, num_blocks=2,
                          cache_len=512)
    with pytest.raises(SvgbError, match="cu_seqlens is on the CPU"):
        core._cu_seqlens("kvcache_append", "cu_seqlens", torch.tensor([0, 3]), None, None)
    with pytest.raises(SvgbError, match="must be a device int tensor"):
        core._cu_seqlens("kvcache_append", "cu_seqlens", [0, 3], None, None)


def test_attn_fwd_refusals_before_launch(monkeypatch):
    """q whose rows differ from the plan's total_q, and grad, are refused before any launch."""
    from svgb200 import core
    from svgb200._lib import Plan, SvgbError

    calls = []
    monkeypatch.setattr(core, "lib", lambda: calls.append(1))
    monkeypatch.setattr(core, "_need_cuda", lambda *ts: None)
    desc = Plan(kind=core.PLAN_KVCACHE, BH=1024, S=12, max_items=4, varlen_items=4)
    plan = core.AttnPlan(desc, torch.empty(0), (1, 12))
    kc = torch.zeros(4, 256, 2, 64, dtype=torch.bfloat16)
    with pytest.raises(SvgbError, match="total_q=12"):
        core.attn_fwd(torch.zeros(11, 4, 64, dtype=torch.bfloat16), kc, kc, plan)
    with pytest.raises(SvgbError, match="total_q=12"):
        core.attn_fwd(torch.zeros(1, 12, 4, 64, dtype=torch.bfloat16), kc, kc, plan)
    with pytest.raises(SvgbError, match="no backward"):
        core.attn_fwd(torch.zeros(12, 4, 64, dtype=torch.bfloat16, requires_grad=True), kc, kc, plan)
    with pytest.raises(SvgbError, match="out"):
        core.attn_fwd(torch.zeros(12, 4, 64, dtype=torch.bfloat16), kc, kc, plan,
                      out=torch.zeros(12, 4, 32, dtype=torch.bfloat16))
    assert calls == []


@pytest.fixture
def dropin(monkeypatch):
    """flash_attn_with_kvcache with core's append, plan and forward recorded instead of run"""
    from svgb200 import core, patch

    calls = []
    monkeypatch.setattr(core, "_seqlens", lambda s, B, dev: ("lens", s if isinstance(s, int) else "t", B))
    monkeypatch.setattr(core, "_cu_seqlens", lambda who, name, cu, B, dev: _check_len(who, name, cu, B))
    monkeypatch.setattr(core, "kvcache_append", lambda *a, **kw: calls.append(("append", a, kw)))
    monkeypatch.setattr(core, "plan_kvcache", lambda *a, **kw: calls.append(("plan", a, kw)) or "plan")
    monkeypatch.setattr(core, "attn_fwd", lambda *a, **kw: calls.append(("fwd", a, kw)) or "out")
    return patch, calls


def test_dropin_varlen_mapping(dropin):
    patch, calls = dropin
    q, kc, vc, table = _T(9, 8, 128), _T(40, 256, 2, 128), _T(40, 256, 2, 128), _T(3, 9)
    k, v, cu_q, cu_k = _T(6, 2, 128), _T(6, 2, 128), _T(4), _T(4)
    assert patch.flash_attn_with_kvcache(q, kc, vc, k, v, cache_seqlens=_T(3), block_table=table, causal=True,
                                         softmax_scale=0.5, return_softmax_lse=True, cu_seqlens_q=cu_q,
                                         cu_seqlens_k_new=cu_k, max_seqlen_q=5) == "out"
    ap, pp, fp = calls
    assert ap[0] == "append" and ap[1] == (kc, vc, k, v, ("lens", "t", 3))
    assert ap[2] == dict(block_table=table, cache_batch_idx=None, cu_seqlens=cu_k)
    assert pp[0] == "plan" and pp[1] == (("lens", "t", 3),)
    assert pp[2] == dict(cu_seqlens_q=cu_q, total_q=9, max_seqlen_q=5, cu_seqlens_new=cu_k, num_blocks=40,
                         cache_len=None, block_table=table, page_size=256, cache_batch_idx=None, causal=True,
                         window_size=(-1, -1))
    assert fp[0] == "fwd" and fp[1] == (q, kc, vc, "plan") and fp[2] == dict(return_lse=True, sm_scale=0.5)
    calls.clear()
    # no new rows: plan and forward only; a contiguous cache defaults to its whole length
    patch.flash_attn_with_kvcache(q, _T(3, 512, 2, 128), _T(3, 512, 2, 128), cu_seqlens_q=cu_q)
    pp, fp = calls
    assert pp[1] == (("lens", 512, 3),) and pp[2]["cu_seqlens_new"] is None and pp[2]["cache_len"] == 512


@pytest.mark.parametrize("kw,needle", [
    (dict(cu_seqlens_k_new=_T(4)), "go with cu_seqlens_q"), (dict(max_seqlen_q=3), "go with cu_seqlens_q"),
    (dict(cu_seqlens_q=_T(4), k=_T(6, 2, 64), v=_T(6, 2, 64)), "come with cu_seqlens_k_new"),
    (dict(cu_seqlens_q=_T(4), cu_seqlens_k_new=_T(4)), "come with cu_seqlens_k_new"),
    (dict(cu_seqlens_q=_T(4), k=_T(6, 2, 64), v=_T(6, 2, 64), cu_seqlens_k_new=_T(3)), "B \\+ 1"),
    (dict(cu_seqlens_q=_T(4), max_seqlen_q=10), "max_seqlen_q=10"),
    (dict(cu_seqlens_q=_T(4), rotary_cos=_T(4, 32)), "rotary_cos"),
])
def test_dropin_varlen_refusals(dropin, kw, needle):
    from svgb200._lib import SvgbError

    patch, calls = dropin
    with pytest.raises(SvgbError, match=needle):
        patch.flash_attn_with_kvcache(_T(9, 8, 64), _T(2, 512, 2, 64), _T(2, 512, 2, 64), **kw)
    assert calls == []


def test_dropin_varlen_q_shape(dropin):
    from svgb200._lib import SvgbError

    patch, calls = dropin
    with pytest.raises(SvgbError, match=r"\[total_q, Hq, D\]"):
        patch.flash_attn_with_kvcache(_T(2, 5, 8, 64), _T(2, 512, 2, 64), _T(2, 512, 2, 64), cu_seqlens_q=_T(3))
    assert calls == []
