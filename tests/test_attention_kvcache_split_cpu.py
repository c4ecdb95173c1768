"""Split KV-cache attention (svgb_attn_plan_kvcache_split, svgb_attn_fwd_kvcache_split, plan_kvcache(num_splits=))
without a GPU: the ABI refusals, the split plan's workspace against the single plan's, the automatic split count at the
decode and chunk shapes with a patched SM count, and that num_splits=1 reaches exactly the single-pass planner."""
import ctypes as C

import pytest

from test_attention_kvcache_cpu import _kv_plan, _Ptr, _T
from test_attention_local_cpu import PTR, lib  # noqa: F401  (lib: the module-scoped library fixture)

BIG = 10 ** 6
SPLIT = 8  # SVGB_PLAN_KVCACHE_SPLIT


def _bytes(lib, B, Sq, cap, sink=0, left=BIG, right=0, n=None):
    out = C.c_size_t()
    if n is None:
        assert lib.svgb_attn_plan_kvcache_bytes(B, Sq, cap, sink, left, right, C.byref(out)) == 0
    else:
        assert lib.svgb_attn_plan_kvcache_split_bytes(B, Sq, cap, sink, left, right, n, C.byref(out)) == 0
    return out.value


def _split_plan(B=2, Sq=100, rows=4 * 512, n=3):
    p = _kv_plan(B, Sq, rows)
    p.kind, p.max_items = SPLIT, n * B * -(-Sq // 256)
    return p


def test_split_plan_workspace_against_the_single_plan(lib):
    """16 + align16(4 (B + 2)) + 32 n I + 8 n I ceil(slots / n): the header of the single plan, n times its items, and
    chunk storage between the single plan's I slots and I (slots + n - 1)."""
    def slots(cap, sink, left, right):
        return min(-(-cap // 128), -(-sink // 128) + (255 + left + right) // 128 + 2)

    for B, Sq, cap, sink, left, right in [(1, 1, 32768, 1560, 14040, 0), (1, 1560, 32768, 1560, 14040, 0),
                                          (3, 300, 1000, 70, 300, 0), (2, 1, 128, 0, 0, 0), (64, 1, 131072, 0, BIG, 0)]:
        single = _bytes(lib, B, Sq, cap, sink, left, right)
        items = B * -(-Sq // 256)
        head = 16 + -(-4 * (B + 2) // 16) * 16
        sl = slots(cap, sink, left, right)
        assert single == head + 32 * items + 8 * items * sl
        assert _bytes(lib, B, Sq, cap, sink, left, right, n=1) == single
        for n in (2, 3, 7, 32, 200):
            got = _bytes(lib, B, Sq, cap, sink, left, right, n=n)
            per = -(-sl // n)
            assert got == head + 32 * n * items + 8 * n * items * per, (B, Sq, n)
            assert items * sl <= n * items * per < items * (sl + n)


def test_split_forward_workspace_bytes(lib):
    out = C.c_size_t()
    assert lib.svgb_attn_fwd_kvcache_split_bytes(3, 1560, 12, 128, C.byref(out)) == 0
    assert out.value == 3 * 1560 * 12 * 128 * 4 + 3 * 12 * 1560 * 4  # about 29 MB for the one-frame chunk
    for args in [(0, 10, 2, 128), (2, 0, 2, 128), (2, 10, 0, 128), (2, 10, 2, 96)]:
        assert lib.svgb_attn_fwd_kvcache_split_bytes(*args, C.byref(out)) < 0, args
        assert b"bad arguments" in lib.svgb_last_error()


def test_split_planner_refusals(lib):
    from svgb200._lib import Plan

    out = C.c_size_t()
    assert lib.svgb_attn_plan_kvcache_split_bytes(2, 100, 1024, 0, 10, 0, 0, C.byref(out)) < 0
    assert b"num_splits (0) must be >= 1" in lib.svgb_last_error()

    def call(n=3, ws=1 << 20, seqlens=PTR):
        return lib.svgb_attn_plan_kvcache_split(seqlens, None, None, 2, 100, 0, 4, 512, 0, 0, 10, 0, n, PTR, ws,
                                                C.byref(Plan()), None)

    for kw, needle in [(dict(n=0), b"num_splits (0) must be >= 1"), (dict(n=-2), b"num_splits (-2)"),
                       (dict(ws=64), b"workspace too small"), (dict(seqlens=None), b"null pointer")]:
        assert call(**kw) < 0, kw
        assert needle in lib.svgb_last_error(), (kw, lib.svgb_last_error())


def test_every_other_entry_refuses_the_split_plan_by_name(lib):
    plan = _split_plan(Sq=100, rows=200)
    s = (C.c_longlong * 3)(8, 8, 8)
    s16 = (C.c_longlong * 3)(16, 16, 16)
    name = b"split KV-cache plan (svgb_attn_plan_kvcache_split)"
    calls = {
        "svgb_attn_fwd": lambda: lib.svgb_attn_fwd(PTR, PTR, PTR, None, None, None, PTR, None, None, None, None, 0, 2,
                                                   200, 128, 128, 200 * 128, 128, 200 * 128, 0.1, C.byref(plan), PTR,
                                                   None),
        "svgb_attn_fwd_kv": lambda: lib.svgb_attn_fwd_kv(PTR, PTR, PTR, PTR, None, 0, 2, 200, 200, 128, 128,
                                                         200 * 128, 128, 200 * 128, 128, 200 * 128, 0.1,
                                                         C.byref(plan), PTR, None),
        "svgb_attn_fwd_gqa": lambda: lib.svgb_attn_fwd_gqa(PTR, PTR, PTR, PTR, None, 0, 4, 2, 200, 200, 128, 128,
                                                           200 * 128, 128, 200 * 128, 128, 200 * 128, 0.1,
                                                           C.byref(plan), PTR, None),
        "svgb_attn_fwd_strided": lambda: lib.svgb_attn_fwd_strided(PTR, PTR, PTR, PTR, None, 0, 1, 2, 2, 200, 200, 128,
                                                                   s, s, s, s, 0.1, C.byref(plan), PTR, None),
        "svgb_attn_fwd_strided_e4m3": lambda: lib.svgb_attn_fwd_strided_e4m3(
            PTR, PTR, PTR, PTR, PTR, PTR, PTR, None, 1, 2, 2, 200, 200, 128, s16, s16, s16, s, 0.1, C.byref(plan), PTR,
            None),
        "svgb_attn_fwd_kvcache_e4m3_rows": lambda: lib.svgb_attn_fwd_kvcache_e4m3_rows(
            PTR, PTR, PTR, PTR, PTR, PTR, PTR, None, 2, 2, 200, 1, 200, 128, s16, s16, s16, s, 0.1, C.byref(plan), PTR,
            None),
        "svgb_attn_bwd": lambda: lib.svgb_attn_bwd(PTR, PTR, PTR, PTR, PTR, PTR, PTR, PTR, PTR, 0, 2, 200, 128, 128,
                                                   200 * 128, 0.1, C.byref(plan), PTR, C.byref(plan), PTR, PTR, 1 << 20,
                                                   None),
        "svgb_attn_bwd_strided": lambda: lib.svgb_attn_bwd_strided(
            PTR, PTR, PTR, PTR, PTR, PTR, PTR, PTR, PTR, 0, 1, 2, 2, 200, 200, 128, *([s] * 8), 0.1, C.byref(plan), PTR,
            C.byref(plan), PTR, PTR, 1 << 20, None),
    }
    for who, call in calls.items():
        assert call() < 0, who
        assert name in lib.svgb_last_error(), (who, lib.svgb_last_error())
        want = b"has no backward" if "bwd" in who else b"runs on svgb_attn_fwd_kvcache_split only"
        assert want in lib.svgb_last_error(), (who, lib.svgb_last_error())


def _split_fwd(lib, plan, *, scales=(None, None, None), dtype=0, row_scales=0, B=2, Sq=100, Hq=4, Hkv=2, D=128,
               nb=4, rows=512, ws=1 << 30, st=(8, 8, 8), st8=(16, 16, 16)):
    s = (C.c_longlong * 3)(*st)
    k = (C.c_longlong * 3)(*(st8 if dtype == 2 else st))
    return lib.svgb_attn_fwd_kvcache_split(PTR, PTR, PTR, *scales, PTR, None, dtype, row_scales, B, Hq, Hkv, Sq, nb,
                                           rows, D, k, k, k, s, 0.1, C.byref(plan), PTR, PTR, ws, None)


def test_split_forward_refusals(lib):
    split = _split_plan(B=2, Sq=100, rows=4 * 512, n=3)
    for kw, needle in [
        (dict(scales=(PTR, PTR, PTR)), b"16-bit inputs (dtype 0) take no scales"),
        (dict(scales=(None, PTR, None), dtype=1), b"16-bit inputs (dtype 1) take no scales"),
        (dict(row_scales=1), b"take no scales"),
        (dict(dtype=2), b"needs the three scale tensors"),
        (dict(dtype=2, scales=(PTR, PTR, PTR), D=64), b"head_dim 128"),
        (dict(dtype=2, scales=(PTR, PTR, PTR), row_scales=1, rows=510), b"multiple of 4"),
        (dict(dtype=2, scales=(PTR, PTR, PTR), st8=(8, 8, 8)), b"multiple of 16 bytes"),
        (dict(dtype=7), b"dtype 7 unsupported"),
        (dict(ws=1000), b"workspace too small"),
        (dict(Sq=50), b"built for 200 query rows"),
        (dict(Hq=3), b"multiple of the key/value heads"),
        (dict(nb=0), b"bad cache geometry"),
    ]:
        assert _split_fwd(lib, split, **kw) < 0, kw
        assert needle in lib.svgb_last_error(), (kw, lib.svgb_last_error())
    # the split count is the plan's items over B ceil(Sq / 256): a plan built for other streams is refused
    odd = _split_plan(B=2, Sq=100, n=3)
    odd.max_items = 5
    assert _split_fwd(lib, odd) < 0
    assert b"no whole number of splits" in lib.svgb_last_error()
    assert _split_fwd(lib, _kv_plan(B=2, Sq=100, rows=4 * 512)) < 0
    assert b"takes split KV-cache plans (svgb_attn_plan_kvcache_split) only (kind 7)" in lib.svgb_last_error()


# --------------------------------------------------------------------------------------------
# the automatic split count
# --------------------------------------------------------------------------------------------
WAN_SLOTS = -(-1560 // 128) + (255 + 14040) // 128 + 2  # sink 1 560, 14 040 back: 126 chunk slots per item


@pytest.mark.parametrize("ctas,want", [
    (12, 10),   # decode, Wan 1.3B: 10 x 12 = 120 of 132 SMs
    (40, 3),    # decode, Wan 14B: 120 of 132
    (84, 3),    # one-frame chunk (1 560 queries), 12 heads: 252 CTAs, 1.9 waves
    (228, 1),   # three-frame chunk, 12 heads: already 1.7 waves
    (760, 1),   # three-frame chunk, 40 heads
    (132, 1), (133, 1),
])
def test_automatic_split_count(ctas, want):
    from svgb200 import core

    assert core.kvcache_num_splits(ctas, WAN_SLOTS, 132) == want


def test_automatic_split_count_bounds():
    from svgb200 import core

    # 6 chunk slots (the 3-page caches of the launch-count tests) leave no split its 4 slots
    assert core.kvcache_num_splits(4, 6, 132) == 1
    assert core.kvcache_num_splits(1, 8, 132) == 2  # 8 slots: two splits of 4 at most
    assert core.kvcache_num_splits(1, 10 ** 4, 132) == 32  # the cap
    assert core.kvcache_num_splits(1, 10 ** 4, 16) == 14  # 14 of 16 SMs
    for ctas in range(1, 300):
        n = core.kvcache_num_splits(ctas, WAN_SLOTS, 132)
        assert n == 1 or (ctas < 132 and 2 <= n <= 31)


class _Lib:
    """The planner entries, recorded."""

    def __init__(self):
        self.seen = []

    def __getattr__(self, name):
        def call(*a):
            self.seen.append((name, a))
            return 0
        return call


@pytest.fixture
def fake(monkeypatch):
    from svgb200 import core

    lib_ = _Lib()
    monkeypatch.setattr(core, "_seqlens", lambda s, B, dev: _Ptr())
    monkeypatch.setattr(core, "_cache_layout", lambda *a: (None, None, 0))
    monkeypatch.setattr(core, "check", lambda rc, what: None)
    monkeypatch.setattr(core.torch, "empty", lambda *a, **kw: _Ptr())
    monkeypatch.setattr(core, "lib", lambda: lib_)
    monkeypatch.setattr(core.torch.cuda, "current_stream", lambda d: type("S", (), {"cuda_stream": 0})())
    monkeypatch.setattr(core, "_sm_count", lambda: 132)
    return core, lib_.seen


def test_one_split_is_exactly_the_single_plan(fake):
    core, seen = fake
    bi = _T(3)
    kw = dict(q_len=40, num_blocks=4, cache_len=1000, cache_batch_idx=bi, causal=True, sink=9)
    core.plan_kvcache(5, **kw)
    default = list(seen)
    seen.clear()
    core.plan_kvcache(5, num_splits=1, **kw)

    def plain(calls):  # a byref() is a new object per call
        return [(n, tuple("byref" if type(x).__name__ == "CArgObject" else x for x in a)) for n, a in calls]

    assert plain(seen) == plain(default)
    assert [n for n, _ in default] == ["svgb_attn_plan_kvcache_bytes", "svgb_attn_plan_kvcache"]
    assert default[1][1][3:12] == (3, 40, 0, 4, 1000, 0, 9, 1040, 0)


def test_split_and_automatic_planner_calls(fake):
    from svgb200._lib import SvgbError

    core, seen = fake
    bi = _T(1)
    kw = dict(q_len=1, num_blocks=1, cache_len=32768, cache_batch_idx=bi, causal=True, window_size=(14040, 0),
              sink=1560)
    core.plan_kvcache(5, num_splits=4, **kw)
    (b, ba), (p, pa) = seen
    assert (b, ba[:7]) == ("svgb_attn_plan_kvcache_split_bytes", (1, 1, 32768, 1560, 14040, 0, 4))
    assert (p, pa[3:13]) == ("svgb_attn_plan_kvcache_split", (1, 1, 0, 1, 32768, 0, 1560, 14040, 0, 4))
    seen.clear()
    core.plan_kvcache(5, num_splits=0, num_heads=12, **kw)  # decode at 12 heads: 10 splits on 132 SMs
    assert seen[0][1][:7] == (1, 1, 32768, 1560, 14040, 0, 10)
    seen.clear()
    core.plan_kvcache(5, num_splits=0, num_heads=12, **{**kw, "q_len": 4680})  # 228 CTAs: no split
    assert [n for n, _ in seen] == ["svgb_attn_plan_kvcache_bytes", "svgb_attn_plan_kvcache"]
    with pytest.raises(SvgbError, match="needs num_heads"):
        core.plan_kvcache(5, num_splits=0, **kw)
    with pytest.raises(SvgbError, match="num_splits=-1"):
        core.plan_kvcache(5, num_splits=-1, **kw)


def test_no_backward_by_name():
    from svgb200 import core
    from svgb200._lib import SvgbError

    plan = core.AttnPlan(_split_plan(), None, (2, 100))
    with pytest.raises(SvgbError, match=r"split KV-cache plan \(plan_kvcache\(num_splits=\)\) has no backward"):
        plan.key_major()
    assert plan.S_kv == 4 * 512
