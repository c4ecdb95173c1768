"""Host side of the block-causal mask (SVGB_MASK_BLOCK_CAUSAL: chunk-wise causal attention of autoregressive video),
without a GPU: the kernel's predicate against the definition on every pair, block = 1 against the causal sliding window,
the host mirrors of its band items and KV-cache lists and the slot bound, the C ABI's refusals, and core's argument
translation."""
import ctypes as C
import random

import pytest
import torch

import block_causal_mask as bm
import local_mask as lm
from test_attention_local_cpu import S_GRID, _grid, _item_work, lib, probe  # noqa: F401  (fixtures)

PTR = 1 << 20  # never dereferenced: every plan call here fails its argument checks

# (block C, first_block F, window W (-1: unbounded), sink): C = 1 / 127 / 128 / 129 / 300 and C not a multiple of 128,
# a shorter first block, W = C, W > C, unbounded W, sinks below, across and past a block boundary
CASES = [(1, 1, -1, 0), (1, 1, 5, 0), (1, 1, 1, 3), (127, 127, -1, 0), (128, 128, -1, 0), (129, 129, -1, 0),
         (300, 300, -1, 0), (300, 300, 300, 0), (300, 300, 450, 0), (129, 40, -1, 0), (129, 1, 129, 0),
         (300, 77, 600, 37), (128, 128, 256, 100), (129, 129, 258, 200), (300, 300, 300, 650), (200, 13, 201, 900),
         (700, 700, -1, 0), (1000, 1000, -1, 0), (500, 499, 500, 1)]


def _W(window, block):
    return S_GRID + block if window == -1 else window  # what plan_block_causal passes for an unbounded window


def test_mask_allowed_matches_definition(probe):  # noqa: F811
    got = probe([(bm.MASK_BLOCK_CAUSAL, sink, bm.m1_of(C_, F), _W(W, C_)) for C_, F, W, sink in CASES])
    for i, (C_, F, W, sink) in enumerate(CASES):
        want = _grid(bm.block_causal_mask_fn(C_, F, W, sink))
        assert torch.equal(got[i], want), f"BLOCK{(C_, F, W, sink)}: {int((got[i] != want).sum())} pairs differ"
        assert bool(want.diagonal().all()), "every row keeps its diagonal key"


def test_block_one_is_the_causal_sliding_window(probe):  # noqa: F811
    """block = 1 is MASK_LOCAL(sink, W - 1, 0) on every pair, in the kernel's predicate and in the definition."""
    cases = [(1, 0), (5, 0), (S_GRID, 0), (64, 37), (129, 300), (1, 800)]
    got = probe([(bm.MASK_BLOCK_CAUSAL, sink, bm.m1_of(1, 1), W) for W, sink in cases] +
                [(lm.MASK_LOCAL, sink, W - 1, 0) for W, sink in cases])
    n = len(cases)
    for i, (W, sink) in enumerate(cases):
        want = _grid(lm.local_mask_fn(sink, W - 1, 0))
        assert torch.equal(got[i], want), f"BLOCK(1, W={W}, sink={sink}) kernel vs LOCAL"
        assert torch.equal(got[n + i], want)
        assert torch.equal(_grid(bm.block_causal_mask_fn(1, 1, W, sink)), want)


def test_block_covering_the_sequence_is_dense():
    assert bool(_grid(bm.block_causal_mask_fn(S_GRID, S_GRID, -1, 0)).all())


def test_block_end_rounding():
    """e(p) - 1 is the engine's rounding: the last position of p's block (negative positions: the first block)."""
    for C_, F in [(1, 1), (7, 3), (128, 128), (4680, 1560)]:
        for p in list(range(-20, 3 * C_ + 20)) + [10 ** 6 + 3]:
            e = bm.block_end(p, C_, F)
            assert e > p and (e - F) % C_ == 0 and e >= F and (e - C_ <= p or e == F)


@pytest.mark.parametrize("S", [1000, 4096 + 77])
@pytest.mark.parametrize("C_,F,W,sink", [(300, 300, -1, 0), (129, 40, 258, 0), (1, 1, 300, 0), (300, 300, 600, 130)])
def test_band_items(S, C_, F, W, sink):
    """The mirror's items: every row in one item, the sink keys first key-major, and query-major the segment issued from
    its last rows when W > 1 (heaviest first: list work counted from the predicate)."""
    mod = bm.block_causal_mask_fn(C_, F, W, sink)
    Wp = S + C_ if W == -1 else W
    for transposed in (False, True):
        items = bm.band_items(sink, Wp, S, transposed)
        cov = torch.zeros(S, dtype=torch.int32)
        for r0, nr in items:
            assert 0 < nr <= 256
            cov[r0: r0 + nr] += 1
        assert bool((cov == 1).all())
        starts = [r for r, _ in items]
        if transposed:
            n_sink = (sink + 255) // 256 if 0 < sink < S else 0
            assert starts[:n_sink] == list(range(0, n_sink * 256, 256))
            assert starts[n_sink:] == sorted(starts[n_sink:])
        else:
            assert starts == sorted(starts, reverse=Wp > 1)
            work = [_item_work(mod, S, r, nr) for r, nr in items if nr == 256]
            assert Wp == 1 or work[0] >= work[-1]


# KV-cache mirror cases: (seqlens, Sq, new_len, block, first_block, window, sink, page)
KV_CASES = [
    ([900, 0, 1300], 300, 0, 300, 300, -1, 0, 128),
    ([1000, 1500], 256, 40, 256, 100, 512, 64, 256),
    ([777, 129], 1, 0, 200, 200, 450, 130, 128),
    ([2000, 5], 500, 0, 129, 1, 129, 0, 384),
    ([3000], 700, 0, 700, 700, 1400, 300, 256),
]


@pytest.mark.parametrize("case", range(len(KV_CASES)))
def test_kv_mirror_against_definition_and_slot_bound(case):
    """The mirror's lists hold exactly the chunks with an allowed pair, classified from the definition, and never more
    chunks per item than the planner's slot bound."""
    seqlens, Sq, Snew, C_, F, W, sink, page = KV_CASES[case]
    g = random.Random(case)
    max_pages = -(-(max(seqlens) + Snew) // page)
    nblocks = len(seqlens) * max_pages + 2
    tab = [g.sample(range(nblocks), max_pages) for _ in seqlens]
    items, Ls = bm.kv_plan(seqlens, Sq=Sq, new_len=Snew, nblocks=nblocks, block_rows=page, table=tab, sink=sink,
                           block=C_, first_block=F, window=W)
    cap = max_pages * page
    Wc = min(cap + Sq + C_, 2 ** 31 - 1) if W == -1 else W
    slots = bm.kv_slots(cap, sink, Wc, C_)
    for b, r0, nr, chunks in items:
        L = Ls[b]
        assert len(chunks) <= slots, (b, r0, len(chunks), slots)
        for row, valid, elem, j in chunks:
            pairs = [bm.allowed(L - Sq + (i - b * Sq), 128 * j + c, sink, C_, F, W)
                     for i in range(r0, r0 + nr) for c in range(valid)]
            assert any(pairs) and elem == (not all(pairs))
        kept = {j for *_, j in chunks}
        for j in range(-(-L // 128)):
            if j not in kept:
                assert not any(bm.allowed(L - Sq + (i - b * Sq), 128 * j + c, sink, C_, F, W)
                               for i in range(r0, r0 + nr) for c in range(min(128, L - 128 * j)))


def test_one_block_call_attends_the_cache_tail():
    """Sq queries that form one block (a block ends at L) all attend [L - W, L) plus the sinks."""
    L, Sq, C_, W, sink = 4680 * 7, 4680, 4680, 3 * 4680, 1560
    for i in range(0, Sq, 97):
        e = bm.block_end(L - Sq + i, C_, C_)
        assert e == L
        assert bm.allowed(L - Sq + i, L - W, sink, C_, C_, W) and not bm.allowed(L - Sq + i, L - W - 1, sink, C_, C_, W)
        assert bm.allowed(L - Sq + i, L - 1, sink, C_, C_, W) and bm.allowed(L - Sq + i, sink - 1, sink, C_, C_, W)


def test_renumbered_first_block_keeps_the_blocks():
    """Lowering every position by d keys with first_block = ((F - d - 1) mod C) + 1 keeps every (query, key) pair."""
    for C_, F, d in [(300, 300, 256), (300, 77, 1000), (4680, 4680, 1560), (129, 1, 128), (128, 128, 128)]:
        F2 = (F - d - 1) % C_ + 1
        assert 1 <= F2 <= C_
        for p in range(d, d + 3 * C_, 7):
            assert bm.block_end(p, C_, F) - d == bm.block_end(p - d, C_, F2)


# --------------------------------------------------------------------------------------------
# C ABI
# --------------------------------------------------------------------------------------------
def _band_call(lib, entry, m0, m1, m2, S=1000):  # noqa: F811
    from svgb200._lib import Plan

    nbytes = C.c_size_t()
    assert lib.svgb_attn_plan_band_bytes(S, C.byref(nbytes)) == 0
    plan = Plan()
    assert getattr(lib, entry)(bm.MASK_BLOCK_CAUSAL, m0, m1, m2, 2, S, PTR, nbytes.value, C.byref(plan), None) < 0
    return lib.svgb_last_error()


@pytest.mark.parametrize("entry", ["svgb_attn_plan_band", "svgb_attn_plan_band_t"])
@pytest.mark.parametrize("args,needle", [
    ((0, 0, 10), b"block C = 0 must be >= 1"),
    ((0, bm.m1_of(100, 0), 100), b"first_block F = 0 must lie in [1, C = 100]"),
    ((0, 100 | 200 << 16, 100), b"first_block F = -100 must lie in [1, C = 100]"),
    ((0, bm.m1_of(100, 100), 99), b"window W = 99 must be >= the block C = 100"),
    ((-1, bm.m1_of(100, 100), 100), b"sink = -1 must be >= 0"),
    ((0, -5, 100), b"m1 = -5 is not C | (C - F) << 16"),
])
def test_band_plan_refusals(lib, entry, args, needle):  # noqa: F811
    msg = _band_call(lib, entry, *args)
    assert needle in msg and entry.encode() in msg, msg


def test_mode_11_stays_unknown(lib):  # noqa: F811
    from svgb200._lib import Plan

    nbytes = C.c_size_t()
    assert lib.svgb_attn_plan_band_bytes(1000, C.byref(nbytes)) == 0
    for mode in (11, 13):
        assert lib.svgb_attn_plan_band(mode, 0, 0, 0, 2, 1000, PTR, nbytes.value, C.byref(Plan()), None) < 0
        assert f"unknown mask mode {mode}".encode() in lib.svgb_last_error()


@pytest.mark.parametrize("args,needle", [
    ((0, 100, 0, 100), b"block C = 0 must lie in [1, 2^16)"),
    ((0, 70000, 70000, 70000), b"block C = 70000 must lie in [1, 2^16) (it is packed in 16 bits)"),
    ((0, 100, 100, 0), b"first_block F = 0 must lie in [1, C = 100]"),
    ((0, 100, 100, 101), b"first_block F = 101 must lie in [1, C = 100]"),
    ((0, 99, 100, 100), b"window W = 99 must be >= the block C = 100"),
    ((-3, 100, 100, 100), b"sink = -3 must be >= 0"),
])
@pytest.mark.parametrize("n", [1, 3])
def test_kvcache_block_refusals(lib, args, needle, n):  # noqa: F811
    from svgb200._lib import Plan

    sink, W, C_, F = args
    nbytes = C.c_size_t()
    assert lib.svgb_attn_plan_kvcache_block_bytes(2, 300, 4096, sink, W, C_, F, n, C.byref(nbytes)) < 0
    assert needle in lib.svgb_last_error() and b"svgb_attn_plan_kvcache_block_bytes" in lib.svgb_last_error()
    lens = (C.c_int32 * 2)(100, 200)
    assert lib.svgb_attn_plan_kvcache_block(lens, None, None, 2, 300, 0, 2, 4096, 0, sink, W, C_, F, n, PTR, 1 << 30,
                                            C.byref(Plan()), None) < 0
    msg = lib.svgb_last_error()
    assert needle in msg and b"svgb_attn_plan_kvcache_block:" in msg, msg


def test_kvcache_block_refuses_zero_splits(lib):  # noqa: F811
    nbytes = C.c_size_t()
    assert lib.svgb_attn_plan_kvcache_block_bytes(2, 300, 4096, 0, 100, 100, 100, 0, C.byref(nbytes)) < 0
    assert b"num_splits (0) must be >= 1" in lib.svgb_last_error()


@pytest.mark.parametrize("n", [1, 2, 5])
@pytest.mark.parametrize("cap,sink,W,C_", [(4096, 0, 300, 300), (32760, 1560, 14040, 4680), (5000, 130, 5500, 129),
                                           (65536, 0, 2 ** 31 - 1, 4680)])
def test_kvcache_block_workspace(lib, n, cap, sink, W, C_):  # noqa: F811
    """The block entry's workspace is the split planner's (the single one's at n = 1) with left = W - 1 and
    right = C - 1: the slot bound the mirror checks."""
    B, Sq = 3, 700
    a, b = C.c_size_t(), C.c_size_t()
    assert lib.svgb_attn_plan_kvcache_block_bytes(B, Sq, cap, sink, W, C_, C_, n, C.byref(a)) == 0
    if n == 1:
        assert lib.svgb_attn_plan_kvcache_bytes(B, Sq, cap, sink, W - 1, C_ - 1, C.byref(b)) == 0
    else:
        assert lib.svgb_attn_plan_kvcache_split_bytes(B, Sq, cap, sink, W - 1, C_ - 1, n, C.byref(b)) == 0
    assert a.value == b.value
    slots = bm.kv_slots(cap, sink, W, C_)
    items = n * B * -(-Sq // 256)
    hdr = 16 + -(-4 * (B + 2) // 16) * 16
    assert a.value == hdr + 32 * items + 8 * items * -(-slots // n)


# --------------------------------------------------------------------------------------------
# Python
# --------------------------------------------------------------------------------------------
@pytest.fixture
def recorded(monkeypatch):
    from svgb200 import core

    calls = []
    monkeypatch.setattr(core, "plan_band", lambda *a: calls.append(a) or "plan")
    return calls


@pytest.mark.parametrize("kw,expect", [
    (dict(block=300), (0, 300, 1300)),
    (dict(block=300, window=600, sink=37), (37, 300, 600)),
    (dict(block=300, first_block=77), (0, 300 | 223 << 16, 1300)),
    (dict(block=2000), (0, 2000, 3000)),
    (dict(block=1, window=1), (0, 1, 1)),
])
def test_plan_block_causal_mapping(recorded, kw, expect):
    from svgb200 import core

    assert core.plan_block_causal(3, 1000, "dev", **kw) == "plan"
    assert recorded == [(core.MASK_BLOCK_CAUSAL, *expect, 3, 1000, "dev")]


@pytest.mark.parametrize("kw,needle", [
    (dict(block=0), "block=0 must lie in"),
    (dict(block=1 << 16), "block=65536 must lie in"),
    (dict(block=300, first_block=0), "first_block=0 must lie in"),
    (dict(block=300, first_block=301), "first_block=301 must lie in"),
    (dict(block=300, window=299), "window=299 must be -1"),
    (dict(block=300, sink=-1), "sink=-1 must be >= 0"),
])
def test_plan_block_causal_refusals(recorded, kw, needle):
    from svgb200 import core

    with pytest.raises(core.SvgbError, match=needle.replace("(", r"\(")):
        core.plan_block_causal(3, 1000, "dev", **kw)
    assert recorded == []


@pytest.mark.parametrize("kw,needle", [
    (dict(window_size=(600, 0)), r"window_size\[1\] = 0 must be -1"),
    (dict(window_size=(600, 5)), r"window_size\[1\] = 5 must be -1"),
    (dict(causal=True), "causal=True is redundant with block="),
    (dict(window_size=(100, -1)), "window=100 must be -1"),
    (dict(first_block=400), "first_block=400 must lie in"),
])
def test_plan_kvcache_block_refusals(kw, needle):
    """Refused before any device work: the cache arguments here are CPU tensors the planner never reaches."""
    from svgb200 import core

    with pytest.raises(core.SvgbError, match=needle):
        core.plan_kvcache(torch.zeros(2, dtype=torch.int32), q_len=300, num_blocks=2, cache_len=4096, block=300, **kw)


def test_varlen_refuses_the_block_form():
    from svgb200 import core

    cu = torch.tensor([0, 100, 300], dtype=torch.int32)
    with pytest.raises(core.SvgbError, match="block-causal masks inside packed segments are not supported"):
        core.plan_local_varlen(cu, total_q=300, block=100)


def _band_plan(mode, m1=300):
    from svgb200 import core
    from svgb200._lib import Plan

    d = Plan()
    d.kind, d.BH, d.S, d.mask_mode, d.m0, d.m1, d.m2 = core.PLAN_BAND, 2, 500, mode, 1, m1, 600
    return core.AttnPlan(d, torch.empty(0, dtype=torch.uint8))


def test_block_plans_have_a_backward(monkeypatch):
    """Under grad a block-causal plan reaches the autograd Function, and key_major() is the band planner's transpose
    with the same parameters."""
    from svgb200 import core

    calls = []
    monkeypatch.setattr(core, "plan_band_t", lambda *a: calls.append(a) or "plan_t")

    class Fn:
        @staticmethod
        def apply(*a):
            return "ran"

    monkeypatch.setattr(core, "_Attention", Fn)
    x = [torch.zeros(1, 2, 500, 64, dtype=torch.bfloat16, requires_grad=True) for _ in range(3)]
    plan = _band_plan(core.MASK_BLOCK_CAUSAL)
    assert core.attention(*x, plan) == "ran"
    assert plan.key_major() == "plan_t"
    assert calls == [(core.MASK_BLOCK_CAUSAL, 1, 300, 600, 2, 500, torch.device("cpu"))]
