"""Which arguments every attention entry of the C ABI accepts, without a GPU: a census of refusals.

Each cell is one call with host-built descriptors and fake device pointers.  It records one of two outcomes: "R", the
call was refused (rc = -1 with an argument message), or "P", it passed every check.  Without a CUDA driver a pass ends
at the TMA encode ("cuTensorMapEncodeTiled unavailable"), at a failed launch, or, for a `_bytes` entry, at rc = 0.
The expected outcomes are pinned per entry as a hex bitmask ("P" = 1) in cell order; `PYTHONPATH=.:sparse-videogen_b200
python tests/test_attention_entry_rules_cpu.py` prints the table for the library as built.

Axes:
- forward: every forward entry x plan kinds 1-8 and an unknown kind x bf16 / fp16 / e4m3 x scales absent, per head or
  per row x row vectors absent or present x Sq == Skv or not x G = Hq / Hkv = 1 or 2;
- backward: every backward entry x (kind, kind_t) x Sq == Skv or not x G = 1 or 2;
- KV-cache planners and their `_bytes` twins: good and bad (sink, left, right, W, C, F, n, max_q) x contiguous, paged
  and bad cache geometry;
- KV-cache appends: every append x dtype x head_dim x scale pointers x row flag x block_rows x cache strides.

On a machine with a CUDA device a passing cell would launch kernels on fake pointers, so the file skips itself there."""
import ctypes as C
import itertools

import pytest
import torch

from test_attention_local_cpu import lib  # noqa: F401  (lib: the module-scoped library fixture)

pytestmark = pytest.mark.skipif(torch.cuda.is_available(),
                                reason="a passing cell would launch kernels on fake pointers on a real device")

PTR = 1 << 20  # 16-byte aligned, never dereferenced
BIG = 1 << 40  # workspace bytes: never the reason for a refusal
D = 128
PASS_MARKS = (b"cuTensorMapEncodeTiled unavailable", b"kernel launch failed")
KINDS = (1, 2, 3, 4, 5, 6, 7, 8, 99)


def _plan(kind, S, Skv, BHkv):
    """A well-formed descriptor of `kind` for S query rows over Skv keys and BHkv key/value heads."""
    from svgb200._lib import Plan

    p = Plan()
    p.kind, p.S = kind, S
    p.items_off, p.chunks_off, p.bytes = 48, 112, 4096
    p.max_items = 2
    if kind in (5, 6, 7, 8):  # one list for every head: BH holds the key length
        p.BH, p.items_stride = Skv, 0
        p.mask_mode, p.m0, p.m1, p.m2 = 10, 0, 10, 0
        if kind == 8:
            p.max_items = 2 * ((S + 255) // 256)  # two splits
    elif kind in (2, 4):  # band: Skv = S
        p.BH, p.items_stride = BHkv, 0
    else:  # variable-block and gather plans record Skv in m0; an unknown kind looks like them
        p.BH, p.items_stride, p.m0 = BHkv, p.max_items, Skv
    return p


def _st(*x):
    return (C.c_longlong * 3)(*x)


def _outcome(lib, rc):
    assert rc in (0, -1, -2, -3), rc
    if rc == -1:
        err = lib.svgb_last_error()
        if not any(m in err for m in PASS_MARKS):
            assert err, "a refusal names its reason"
            return "R"
    return "P"


# --------------------------------------------------------------------------------------------
# forward
# --------------------------------------------------------------------------------------------
FWD = ("svgb_attn_fwd", "svgb_attn_fwd_kv", "svgb_attn_fwd_gqa", "svgb_attn_fwd_strided", "svgb_attn_fwd_strided_e4m3",
       "svgb_attn_fwd_kvcache_e4m3_rows", "svgb_attn_fwd_kvcache_split")
FWD_AXES = (KINDS, (0, 1, 2), ("none", "head", "row"), (False, True), (True, False), (1, 2))


def _fwd(lib, name, kind, dtype, scales, rowvec, square, G):
    Sq, Skv, Hq = (256, 256, 2) if square else (128, 256, 2)
    Hkv = Hq // G
    plan = _plan(kind, Sq, Skv, Hkv)
    sc = (None, None, None) if scales == "none" else (PTR, PTR, PTR)
    rows = (PTR, PTR, PTR) if rowvec else (None, None, None)
    qst, kst, ost = _st(Hq * Sq * D, Sq * D, D), _st(Hkv * Skv * D, Skv * D, D), _st(Hq * Sq * D, Sq * D, D)
    tail = (0.1, C.byref(plan), PTR, None)
    f = getattr(lib, name)
    if name == "svgb_attn_fwd":
        return f(PTR, PTR, PTR, *sc, PTR, None, *rows, dtype, Hq, Sq, D, D, Sq * D, D, Sq * D, *tail)
    if name == "svgb_attn_fwd_kv":
        return f(PTR, PTR, PTR, PTR, None, dtype, Hq, Sq, Skv, D, D, Sq * D, D, Skv * D, D, Sq * D, *tail)
    if name == "svgb_attn_fwd_gqa":
        return f(PTR, PTR, PTR, PTR, None, dtype, Hq, Hkv, Sq, Skv, D, D, Sq * D, D, Skv * D, D, Sq * D, *tail)
    if name == "svgb_attn_fwd_strided":
        return f(PTR, PTR, PTR, PTR, None, dtype, 1, Hq, Hkv, Sq, Skv, D, qst, kst, kst, ost, *tail)
    if name == "svgb_attn_fwd_strided_e4m3":
        return f(PTR, PTR, PTR, *sc, PTR, None, 1, Hq, Hkv, Sq, Skv, D, qst, kst, kst, ost, *tail)
    if name == "svgb_attn_fwd_kvcache_e4m3_rows":
        return f(PTR, PTR, PTR, *sc, PTR, None, Hq, Hkv, Sq, Skv // 128, 128, D, qst, kst, kst, ost, *tail)
    assert name == "svgb_attn_fwd_kvcache_split"
    return f(PTR, PTR, PTR, *sc, PTR, None, dtype, int(scales == "row"), 1, Hq, Hkv, Sq, Skv // 128, 128, D, qst, kst,
             kst, ost, 0.1, C.byref(plan), PTR, PTR, BIG, None)


# --------------------------------------------------------------------------------------------
# backward
# --------------------------------------------------------------------------------------------
BWD = ("svgb_attn_bwd", "svgb_attn_bwd_kv", "svgb_attn_bwd_gqa", "svgb_attn_bwd_strided")
BWD_AXES = (KINDS, KINDS, (True, False), (1, 2))


def _bwd(lib, name, kind, kind_t, square, G):
    Sq, Skv, Hq = (256, 256, 2) if square else (128, 256, 2)
    Hkv = Hq // G
    plan, plan_t = _plan(kind, Sq, Skv, Hkv), _plan(kind_t, Skv, Sq, Hkv)
    ptrs = (PTR,) * 9
    tail = (0.1, C.byref(plan), PTR, C.byref(plan_t), PTR, PTR, BIG, None)
    f = getattr(lib, name)
    if name == "svgb_attn_bwd":
        return f(*ptrs, 0, Hq, Sq, D, D, Sq * D, *tail)
    if name == "svgb_attn_bwd_kv":
        return f(*ptrs, 0, Hq, Sq, Skv, D, D, Sq * D, D, Skv * D, *tail)
    if name == "svgb_attn_bwd_gqa":
        return f(*ptrs, 0, Hq, Hkv, Sq, Skv, D, D, Sq * D, D, Skv * D, *tail)
    q, kv = _st(Hq * Sq * D, Sq * D, D), _st(Hkv * Skv * D, Skv * D, D)
    return f(*ptrs, 0, 1, Hq, Hkv, Sq, Skv, D, q, kv, kv, q, q, q, kv, kv, *tail)


# --------------------------------------------------------------------------------------------
# KV-cache planners
# --------------------------------------------------------------------------------------------
# (num_blocks, block_rows, max_pages, paged) and the capacity a `_bytes` call takes for it
GEOMETRY = ((4, 512, 0, False), (8, 256, 4, True), (8, 200, 4, True))
CAP = (512, 1024, 0)
SINK, LEFT, RIGHT, W, BLOCK, FIRST, NSPLIT, MAXQ = (0, 5, -1), (0, 300, -1), (0, -1), (0, 8, 2), (0, 4), (0, 1, 5), \
    (1, 3, 0), (100, 0, 1000)
# the parameters each planner takes, in its argument order
PLAN = {
    "svgb_attn_plan_kvcache": (SINK, LEFT, RIGHT),
    "svgb_attn_plan_kvcache_split": (SINK, LEFT, RIGHT, NSPLIT),
    "svgb_attn_plan_kvcache_block": (SINK, W, BLOCK, FIRST, NSPLIT),
    "svgb_attn_plan_kvcache_varlen": (SINK, LEFT, RIGHT, W, BLOCK, FIRST, NSPLIT),
}
B, TOTAL_Q = 2, 200


def _planner(lib, name, g, maxq, *params):
    """The planner at geometry g; its query bound is max_q for the variable-length planner and Sq for the others."""
    nb, br, mp, paged = GEOMETRY[g]
    from svgb200._lib import Plan

    plan = Plan()
    table = PTR if paged else None
    tail = (PTR, BIG, C.byref(plan), None)
    if name == "svgb_attn_plan_kvcache_varlen":
        return lib.svgb_attn_plan_kvcache_varlen(PTR, PTR, PTR, None, table, B, TOTAL_Q, maxq, nb, br, mp, *params,
                                                 *tail)
    return getattr(lib, name)(PTR, None, table, B, maxq, 1, nb, br, mp, *params, *tail)


def _planner_bytes(lib, name, g, maxq, *params):
    out = C.c_size_t(0)
    if name == "svgb_attn_plan_kvcache_varlen":
        return lib.svgb_attn_plan_kvcache_varlen_bytes(B, TOTAL_Q, maxq, CAP[g], *params, C.byref(out))
    return getattr(lib, name + "_bytes")(B, maxq, CAP[g], *params, C.byref(out))


# --------------------------------------------------------------------------------------------
# KV-cache appends
# --------------------------------------------------------------------------------------------
APPEND = ("svgb_kvcache_append", "svgb_kvcache_append_e4m3", "svgb_kvcache_append_e4m3_rows",
          "svgb_kvcache_append_varlen")
APPEND_AXES = ((0, 1, 2), (64, 128), ((None, None), (PTR, None), (PTR, PTR)), (0, 1), (512, 130), (16, 8))


def _append(lib, name, dtype, d, scales, row_flag, block_rows, cache_stride):
    kc = _st(cache_stride * 64, cache_stride * 32, cache_stride * 2)
    new = _st(4 * 2 * d, 2 * d, 8 * d)
    geo = (4, block_rows, 0)
    if name == "svgb_kvcache_append_varlen":
        return lib.svgb_kvcache_append_varlen(PTR, PTR, PTR, PTR, PTR, PTR, None, None, dtype, 2, 8, 2, d, *geo, kc, kc,
                                              new, new, *scales, row_flag, None)
    f = getattr(lib, name)
    head = (PTR, PTR, PTR, PTR, PTR, None, None, dtype, 2, 4, 2, d, *geo, kc, kc, new, new)
    return f(*head, None) if name == "svgb_kvcache_append" else f(*head, *scales, None)


# --------------------------------------------------------------------------------------------
# the census
# --------------------------------------------------------------------------------------------
def _groups():
    """(group name, call, cells): the cells of one entry in a fixed order"""
    for name in FWD:
        yield name, lambda lib, c, n=name: _fwd(lib, n, *c), list(itertools.product(*FWD_AXES))
    for name in BWD:
        yield name, lambda lib, c, n=name: _bwd(lib, n, *c), list(itertools.product(*BWD_AXES))
    for name, axes in PLAN.items():
        cells = list(itertools.product(range(len(GEOMETRY)), MAXQ, *axes))
        yield name, lambda lib, c, n=name: _planner(lib, n, *c), cells
        yield name + "_bytes", lambda lib, c, n=name: _planner_bytes(lib, n, *c), cells
    for name in APPEND:
        yield name, lambda lib, c, n=name: _append(lib, n, *c), list(itertools.product(*APPEND_AXES))


def _census(lib, call, cells):
    return "".join(_outcome(lib, call(lib, c)) for c in cells)


def _hex(outcomes):
    return format(int("1" + outcomes.replace("R", "0").replace("P", "1"), 2), "x")


def _unhex(h):
    return bin(int(h, 16))[3:].replace("0", "R").replace("1", "P")


EXPECTED = {
    "svgb_attn_fwd": (
        "1800000800000008080f00000f0000000f0f0aa0000aa000000aaaa000000000000000000c00000c00000000000000000000"
        "000000000c00000c00000000000000000000000000000a00000a0000000a0a0"
    ),
    "svgb_attn_fwd_kv": (
        "1aaaaaaaaaaaa000000000000000000000000000000000000000000000000000000000000ffffffffffff000000000000000"
        "000000000000000000000000000000000000000000000000000000000000000"
    ),
    "svgb_attn_fwd_gqa": (
        "1ffffffffffff000000cccccccccccc000000000000000000000000000000000000000000ffffffffffff000000000000000"
        "000000000ffffffffffff000000000000000000000000000000000000000000"
    ),
    "svgb_attn_fwd_strided": (
        "1ffffffffffff000000cccccccccccc000000000000000000000000000000000000000000ffffffffffff000000000000000"
        "000000000ffffffffffff000000000000000000000000000000000000000000"
    ),
    "svgb_attn_fwd_strided_e4m3": (
        "100ffff00ffff00ffff00cccc00cccc00cccc000000000000000000000000000000000000000000000000000000000000000"
        "00000000000ffff00ffff00ffff000000000000000000000000000000000000"
    ),
    "svgb_attn_fwd_kvcache_e4m3_rows": (
        "1000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000"
        "00000000000ffff00ffff00ffff000000000000000000000000000000000000"
    ),
    "svgb_attn_fwd_kvcache_split": (
        "1000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000"
        "000000000000000000000000000ff0000ff000000ffff000000000000000000"
    ),
    "svgb_attn_bwd": (
        "1800000000000c0000000000000000000000000000c000000000000000000000000000000000000000"
    ),
    "svgb_attn_bwd_kv": (
        "1a0000000000000000000000000000000000000000f000000000000000000000000000000000000000"
    ),
    "svgb_attn_bwd_gqa": (
        "1f00000000000c0000000000000000000000000000f000000000000000000000000000000000000000"
    ),
    "svgb_attn_bwd_strided": (
        "1f00000000000c0000000000000000000000000000f000000000000000000000000000000000000000"
    ),
    "svgb_attn_plan_kvcache": (
        "68a00000028a00a28000000a28000000000000000"
    ),
    "svgb_attn_plan_kvcache_bytes": (
        "68a00000028a00a28000000a28000000000000000"
    ),
    "svgb_attn_plan_kvcache_split": (
        "70c00c30000000000000000000030c00c30000000c30030c00000000000000000000c30030c0000000000000000000000000"
        "0000000000000000000000"
    ),
    "svgb_attn_plan_kvcache_split_bytes": (
        "70c00c30000000000000000000030c00c30000000c30030c00000000000000000000c30030c0000000000000000000000000"
        "0000000000000000000000"
    ),
    "svgb_attn_plan_kvcache_block": (
        "40000000c00000000000030000000000000000000000000000000000000000000000000000000000000000000c0000000000"
        "0030000000000000000000000000030000000000000c00000000000000000000000000000000000000000000000000000000"
        "000000000030000000000000c000000000000000000000000000000000000000000000000000000000000000000000000000"
        "00000000000000000000000000000000000000000000000000000000000000000"
    ),
    "svgb_attn_plan_kvcache_block_bytes": (
        "40000000c00000000000030000000000000000000000000000000000000000000000000000000000000000000c0000000000"
        "0030000000000000000000000000030000000000000c00000000000000000000000000000000000000000000000000000000"
        "000000000030000000000000c000000000000000000000000000000000000000000000000000000000000000000000000000"
        "00000000000000000000000000000000000000000000000000000000000000000"
    ),
    "svgb_attn_plan_kvcache_varlen": (
        "1c00000030000000000000000000c00000000000000000000000000000000000000000000000000000c00000030000000000"
        "000000000c000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000"
        "0000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000"
        "0000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000"
        "0000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000"
        "0000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000"
        "0000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000"
        "000000000000000000000000000000c00000030000000000000000000c000000000000000000000000000000000000000000"
        "00000000000c00000030000000000000000000c0000000000000000000000000000000000000000000000000000000000000"
        "0000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000"
        "0000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000"
        "0000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000"
        "0000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000"
        "0000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000"
        "0000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000"
        "0000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000"
        "0000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000"
        "0000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000"
        "0000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000"
        "0000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000"
        "0000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000"
        "0000000000000000000000000000000000000000000000000000000000000000000000000000000000000000"
    ),
    "svgb_attn_plan_kvcache_varlen_bytes": (
        "1c00000030000000000000000000c00000000000000000000000000000000000000000000000000000c00000030000000000"
        "000000000c000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000"
        "0000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000"
        "0000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000"
        "0000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000"
        "0000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000"
        "0000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000"
        "000000000000000000000000000000c00000030000000000000000000c000000000000000000000000000000000000000000"
        "00000000000c00000030000000000000000000c0000000000000000000000000000000000000000000000000000000000000"
        "0000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000"
        "0000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000"
        "0000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000"
        "0000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000"
        "0000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000"
        "0000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000"
        "0000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000"
        "0000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000"
        "0000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000"
        "0000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000"
        "0000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000"
        "0000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000000"
        "0000000000000000000000000000000000000000000000000000000000000000000000000000000000000000"
    ),
    "svgb_kvcache_append": (
        "1ffffffffffffffffffffffff000000000000"
    ),
    "svgb_kvcache_append_e4m3": (
        "10000ff0000ff0000ff0000ff000000000000"
    ),
    "svgb_kvcache_append_e4m3_rows": (
        "10000000000cc0000000000cc000000000000"
    ),
    "svgb_kvcache_append_varlen": (
        "1f000f0f000fcf000f0f000fc000000000000"
    ),
}


@pytest.mark.parametrize("name,call,cells", list(_groups()), ids=[g[0] for g in _groups()])
def test_entry_rules(lib, name, call, cells):
    got = _census(lib, call, cells)
    want = _unhex(EXPECTED[name])
    assert len(want) == len(cells)
    diff = [(c, w, g) for c, w, g in zip(cells, want, got) if w != g]
    assert not diff, f"{len(diff)} of {len(cells)} cells changed outcome (cell, expected, got): {diff[:12]}"
    assert "R" in got and "P" in got, "every entry both refuses and passes some cells"


if __name__ == "__main__":
    from svgb200 import _lib

    handle = _lib.lib()
    for name, call, cells in _groups():
        h = _hex(_census(handle, call, cells))
        print(f'    "{name}": (')
        for i in range(0, len(h), 100):
            print(f'        "{h[i:i + 100]}"')
        print("    ),")
