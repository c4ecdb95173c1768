"""Host side of the local mask inside packed variable-length segments (svgb_attn_plan_local_varlen), without a GPU: the
kernels' predicate and chunk classification compiled for the host against the issue's semantics, the planner mirror's
structure and its clamping of malformed bounds, the C ABI's refusals and workspace bound, core.plan_local_varlen's
translation of FlashAttention's conventions, and which path the flash_attn_varlen_func drop-in takes."""
import ctypes as C
import os
import random
import shutil
import subprocess

import numpy as np
import pytest
import torch

import local_mask as lm
import varlen_local_mask as vm
from test_attention_local_cpu import ROOT, CSRC, PTR, lib  # noqa: F401  (lib: the module-scoped library fixture)

# the kernels' view of the mask, compiled for the host.  Per case (stdin "nseg sink left right" then the sanitised
# cu_q and cu_k): the Sq x Skv grid as the query-major kernel sees it (seg_origin of the query row) and as the key-major
# kernel sees it (seg_origin of the key row), each restricted to the row's segment as the plan's chunks are; then, per
# line "key_major r0 r1 c0 c1", seg_chunk_kind.
PROBE = r"""
#include <cstdio>
#include <vector>
#include "attn_common.cuh"
using namespace svgb;
static int seg_of(const int* b, int nseg, int x) { int i = 0; while (i + 1 < nseg && b[i + 1] <= x) ++i; return i; }
int main() {
  int nseg, sink, left, right;
  while (std::scanf("%d %d %d %d", &nseg, &sink, &left, &right) == 4) {
    std::vector<int> segs(2 * (nseg + 1) + 1);  // the plan's bounds copy {nseg, cq, ck}
    segs[0] = nseg;
    for (size_t i = 1; i < segs.size(); ++i) std::scanf("%d", &segs[i]);
    const int* cq = segs.data() + 1; const int* ck = cq + nseg + 1;
    const int Sq = cq[nseg], Skv = ck[nseg];
    for (int km = 0; km < 2; ++km) {
      std::vector<unsigned char> out(static_cast<size_t>(Sq) * Skv);
      for (int q = 0; q < Sq; ++q)
        for (int kv = 0; kv < Skv; ++kv) {
          const int i = seg_of(cq, nseg, q), j = seg_of(ck, nseg, kv);
          bool a = false;
          if (i == j && q >= cq[i] && q < cq[i + 1] && kv >= ck[j] && kv < ck[j + 1]) {
            const SegOrigin o = seg_origin(segs.data(), km ? kv : q, km, sink);
            a = mask_allowed(MASK_LOCAL, q - o.shift, kv, o.sink_end, left, right);
          }
          out[static_cast<size_t>(q) * Skv + kv] = a;
        }
      std::fwrite(out.data(), 1, out.size(), stdout);
    }
    int n;
    std::scanf("%d", &n);
    std::vector<unsigned char> kinds(n);
    for (int t = 0; t < n; ++t) {
      int km, r0, r1, c0, c1;
      std::scanf("%d %d %d %d %d", &km, &r0, &r1, &c0, &c1);
      kinds[t] = seg_chunk_kind(km, r0, r1, c0, c1, seg_origin(segs.data(), r0, km, sink), left, right);
    }
    std::fwrite(kinds.data(), 1, kinds.size(), stdout);
  }
  return 0;
}
"""

# (cu_q, cu_k, sink, left, right): equal and unequal segments, Lq > Lk (rows without keys under causal), Lq < Lk (a
# KV-cache shape), empty and 1-token segments, bounds off 8 and 128, sinks longer than a segment, windows (l, 0),
# (l, r), (0, r)
BIG = 10 ** 6
CASES = [
    ([0, 300], [0, 300], 0, BIG, 0),
    ([0, 100, 357, 358, 700], [0, 100, 357, 358, 700], 0, BIG, 0),
    ([0, 200, 201, 460], [0, 77, 300, 300], 0, BIG, 0),
    ([0, 130, 130, 400], [0, 390, 391, 650], 5, 100, 0),
    ([0, 259, 500], [0, 259, 500], 3, 40, 17),
    ([0, 1, 257, 513], [0, 500, 501, 513], 300, 0, 60),
    ([0, 0, 129, 129, 390], [0, 1, 1, 400, 401], 2, 129, 0),
    ([0, 520], [0, 1100], 260, 255, 0),
]


def _case_id(c):
    return f"n{len(c[0]) - 1}-q{c[0][-1]}-k{c[1][-1]}-s{c[2]}-l{min(c[3], 9999)}-r{c[4]}"


@pytest.fixture(scope="module")
def probe(tmp_path_factory):
    nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    d = tmp_path_factory.mktemp("varlen_probe")
    (d / "probe.cu").write_text(PROBE)
    subprocess.run([nvcc, "-std=c++17", "-I", str(CSRC), str(d / "probe.cu"), "-o", str(d / "probe")], check=True,
                   capture_output=True)

    def run(cu_q, cu_k, sink, left, right, queries):
        text = f"{len(cu_q) - 1} {sink} {left} {right}\n{' '.join(map(str, cu_q + cu_k))}\n{len(queries)}\n"
        text += "".join(" ".join(map(str, x)) + "\n" for x in queries)
        out = subprocess.run([str(d / "probe")], input=text.encode(), capture_output=True, check=True).stdout
        Sq, Skv = cu_q[-1], cu_k[-1]
        g = np.frombuffer(out[: 2 * Sq * Skv], np.uint8).reshape(2, Sq, Skv).astype(bool)
        return torch.from_numpy(g.copy()), list(out[2 * Sq * Skv:])

    return run


def _all_chunks(cu_q, cu_k, sink, transposed):
    """(r0, r1, c0, c1) of every item and every chunk of its segment, omitted ones included."""
    out = []
    for r0, nr, _ in vm.items(cu_q, cu_k, sink, 0, 0, transposed):
        rb = cu_k if transposed else cu_q
        cb = cu_q if transposed else cu_k
        i = max(j for j in range(len(rb) - 1) if rb[j] <= r0)
        out += [(r0, r0 + nr - 1, c, min(c + 128, cb[i + 1]) - 1) for c in range(cb[i], cb[i + 1], 128)]
    return out


@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_kernel_predicate_and_chunk_kinds(probe, case):
    """The kernels' predicate (seg_origin + mask_allowed, both directions) equals the semantics on every pair, and
    seg_chunk_kind classifies every chunk of every item exactly (0 none, 1 all, 2 some allowed pairs)."""
    cu_q, cu_k, sink, left, right = case
    want = vm.dense(cu_q, cu_k, sink, left, right)
    qs = [(0, *x) for x in _all_chunks(cu_q, cu_k, sink, False)] + [(1, *x) for x in _all_chunks(cu_q, cu_k, sink, True)]
    grids, kinds = probe(cu_q, cu_k, sink, left, right, qs)
    for km in (0, 1):
        assert torch.equal(grids[km], want), f"key_major={km}: {int((grids[km] != want).sum())} pairs differ"
    for (km, r0, r1, c0, c1), kind in zip(qs, kinds):
        blk = (want.T if km else want)[r0: r1 + 1, c0: c1 + 1]
        exp = 0 if not bool(blk.any()) else 1 if bool(blk.all()) else 2
        assert kind == exp, f"key_major={km} rows {r0}..{r1} cols {c0}..{c1}: kind {kind}, expected {exp}"


def test_one_segment_is_the_local_band():
    """nseg = 1, Sq == Skv: the semantics are MASK_LOCAL(sink, left, right) on every pair."""
    for sink, left, right in [(0, 700, 0), (37, 129, 0), (0, 0, 256), (130, 77, 200)]:
        idx = torch.arange(700)
        band = lm.local_mask_fn(sink, left, right)(idx.view(-1, 1), idx.view(1, -1))
        q, kv = idx.view(-1, 1), idx.view(1, -1)
        # the general path of mask_fn (two segments, one empty) must agree with the band
        assert torch.equal(vm.mask_fn([0, 700, 700], [0, 700, 700], sink, left, right)(q, kv), band)


@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_mirror_structure(case):
    """Items in launch order: every row in exactly one item, no item across a segment (key-major: across its sink keys),
    chunks at the segment start + 128 j cut at the segment end, FULL chunks with no disallowed pair and no allowed
    pair outside the lists, items in row order."""
    cu_q, cu_k, sink, left, right = case
    m = vm.dense(cu_q, cu_k, sink, left, right)
    for transposed in (False, True):
        mm = m.T if transposed else m
        rb, cb = (cu_k, cu_q) if transposed else (cu_q, cu_k)
        its = vm.items(cu_q, cu_k, sink, left, right, transposed)
        cov = torch.zeros(rb[-1], dtype=torch.int32)
        covered = torch.zeros_like(mm)
        for r0, nr, lst in its:
            assert 0 < nr <= 256
            cov[r0: r0 + nr] += 1
            i = max(j for j in range(len(rb) - 1) if rb[j] <= r0)
            assert r0 + nr <= rb[i + 1], "item across a segment"
            if transposed:
                s = rb[i] + min(sink, rb[i + 1] - rb[i])
                assert r0 + nr <= s or r0 >= s, "key-major item across the sink keys"
            for c0, valid, elem in lst:
                assert (c0 - cb[i]) % 128 == 0 and valid == min(128, cb[i + 1] - c0)
                blk = mm[r0: r0 + nr, c0: c0 + valid]
                assert bool(blk.any()) and (elem or bool(blk.all()))
                covered[r0: r0 + nr, c0: c0 + valid] = True
        assert bool((cov == 1).all())
        assert not bool((mm & ~covered).any()), "an allowed pair in an omitted chunk"
        starts = [r0 for r0, _, _ in its]
        assert starts == sorted(starts)


@pytest.mark.parametrize("cu,total,want", [
    ([0, 5, 3, 9], 9, [0, 5, 5, 9]),           # out of order: running maximum
    ([4, -7, 20, 6], 12, [0, 0, 12, 12]),        # first 0, clamped to [0, total], last = total
    ([0, 100], 40, [0, 40]),                     # last bound past the total
    ([0, 3, 3, 3, 8], 8, [0, 3, 3, 3, 8]),       # empty segments kept
])
def test_mirror_clamps_malformed_bounds(cu, total, want):
    assert vm.sanitize(cu, total) == want
    # the planned state of a malformed call stays in bounds: every item and chunk inside the totals
    cu_q = vm.sanitize(cu, total)
    for transposed in (False, True):
        for r0, nr, lst in vm.items(cu_q, cu_q, 1, 3, 0, transposed):
            assert 0 <= r0 and r0 + nr <= total
            assert all(0 <= c0 and c0 + v <= total for c0, v, _ in lst)


# --------------------------------------------------------------------------------------------
# C ABI
# --------------------------------------------------------------------------------------------
def _bytes(lib, nseg, Sq, Skv):
    n = C.c_size_t()
    assert lib.svgb_attn_plan_local_varlen_bytes(nseg, Sq, Skv, C.byref(n)) == 0, lib.svgb_last_error()
    return n.value


def test_workspace_bound(lib):
    """At nseg = 1 and Sq == Skv the workspace never exceeds the band plan's; it covers the plan's own layout for
    any segmentation (checked on the mirror: sum of items x segment chunks)."""
    for S in [1, 2, 127, 128, 129, 255, 256, 257, 1000, 4096, 32760, 75600, 119056]:
        band = C.c_size_t()
        assert lib.svgb_attn_plan_band_bytes(S, C.byref(band)) == 0
        assert _bytes(lib, 1, S, S) <= band.value, S
    rng = random.Random(0)
    for _ in range(200):
        nseg = rng.randint(1, 12)
        lq = [rng.choice([0, 1, rng.randint(0, 700)]) for _ in range(nseg)]
        lk = [rng.choice([0, 1, rng.randint(0, 700)]) for _ in range(nseg)]
        Sq, Skv = max(sum(lq), 1), max(sum(lk), 1)
        need = 0
        for a, b, sk in [(lq, lk, 0), (lk, lq, rng.randint(0, 300))]:
            n_items = sum((min(sk, x) + 255) // 256 + (x - min(sk, x) + 255) // 256 for x in a)
            n_chunks = sum(((min(sk, x) + 255) // 256 + (x - min(sk, x) + 255) // 256) * ((y + 127) // 128)
                           for x, y in zip(a, b))
            need = max(need, 32 * n_items + 8 * n_chunks)
        assert _bytes(lib, nseg, Sq, Skv) >= need + 16 * (nseg + 1)


def _seg_plan(kind=5, Sq=600, Skv=600, params=(0, 600, 0), layout=(256, 1024, 2048)):
    """A segment plan's host descriptor: S = Sq, BH = Skv (key-major: swapped); layout = (items_off, chunks_off, bytes)"""
    from svgb200._lib import Plan

    p = Plan()
    p.kind, p.S, p.BH = kind, Sq, Skv
    p.mask_mode, (p.m0, p.m1, p.m2) = lm.MASK_LOCAL, params
    p.max_items, (p.items_off, p.chunks_off, p.bytes) = 8, layout
    return p


@pytest.mark.parametrize("args,needle", [((-1, 10, 0), b"sink (-1)"), ((0, -1, 0), b"left (-1)"),
                                         ((0, 5, -2), b"right (-2)")])
@pytest.mark.parametrize("entry", ["svgb_attn_plan_local_varlen", "svgb_attn_plan_local_varlen_t"])
def test_planner_refuses_negative_parameters(lib, entry, args, needle):
    from svgb200._lib import Plan

    nbytes = _bytes(lib, 3, 600, 700)
    plan = Plan()
    assert getattr(lib, entry)(PTR, PTR, 3, 600, 700, *args, PTR, nbytes, C.byref(plan), None) < 0
    msg = lib.svgb_last_error()
    assert needle in msg and b">= 0" in msg, msg


def test_planner_refuses_small_workspace_and_bad_lengths(lib):
    from svgb200._lib import Plan

    plan = Plan()
    nbytes = _bytes(lib, 3, 600, 700)
    assert lib.svgb_attn_plan_local_varlen(PTR, PTR, 3, 600, 700, 0, 5, 0, PTR, nbytes - 1, C.byref(plan), None) < 0
    assert b"workspace too small" in lib.svgb_last_error()
    for nseg, Sq, Skv in [(0, 600, 700), (3, 0, 700), (3, 600, 0)]:
        n = C.c_size_t()
        assert lib.svgb_attn_plan_local_varlen_bytes(nseg, Sq, Skv, C.byref(n)) < 0
        assert b"bad arguments" in lib.svgb_last_error()


def _fwd(lib, plan, dtype=0, scales=(None, None, None), rows=(None, None, None), S=600):
    return lib.svgb_attn_fwd(PTR, PTR, PTR, *scales, PTR, None, *rows, dtype, 2, S, 128, 128, S * 128, 128, S * 128,
                             0.1, C.byref(plan), PTR, None)


def test_forward_refusals(lib):
    """e4m3 inputs, row vectors and the key-major plan are refused by name before any device work."""
    assert _fwd(lib, _seg_plan(), dtype=2, scales=(PTR, PTR, PTR)) < 0
    assert b"not e4m3" in lib.svgb_last_error()
    for rows in [(PTR, None, None), (None, PTR, None), (None, None, PTR)]:
        assert _fwd(lib, _seg_plan(), rows=rows) < 0
        msg = lib.svgb_last_error()
        assert b"row vectors" in msg or b"row gathers" in msg, msg
    assert _fwd(lib, _seg_plan(kind=6)) < 0
    assert b"svgb_attn_plan_local_varlen_t) is for the backward" in lib.svgb_last_error()
    assert _fwd(lib, _seg_plan(Skv=700)) < 0  # svgb_attn_fwd is Sq == Skv: the plan's Skv does not match
    assert b"Skv=700" in lib.svgb_last_error()


def test_fwd_kv_and_gqa_take_segment_plans_only_in_16_bit(lib):
    plan = _seg_plan(Skv=700)
    assert lib.svgb_attn_fwd_kv(PTR, PTR, PTR, PTR, None, 2, 2, 600, 700, 128, 128, 600 * 128, 128, 700 * 128, 128,
                                600 * 128, 0.1, C.byref(plan), PTR, None) < 0
    assert b"bf16 or fp16" in lib.svgb_last_error()
    assert lib.svgb_attn_fwd_gqa(PTR, PTR, PTR, PTR, None, 0, 4, 2, 600, 700, 128, 128, 600 * 128, 128, 700 * 128, 128,
                                 600 * 128, 0.1, C.byref(_seg_plan(kind=6, Skv=700)), PTR, None) < 0
    assert b"key-major plans have no GQA" in lib.svgb_last_error()


def _bwd(lib, plan, plan_t, S=600):
    return lib.svgb_attn_bwd(PTR, PTR, PTR, PTR, PTR, PTR, PTR, PTR, PTR, 0, 2, S, 128, 128, S * 128, 0.1,
                             C.byref(plan), PTR, C.byref(plan_t), PTR, PTR, 1 << 20, None)


def test_backward_refusals(lib):
    """The backward takes the segment plan with its own key-major companion, built for the same parameters."""
    assert _bwd(lib, _seg_plan(), _seg_plan(kind=4)) < 0  # a band key-major plan
    assert b"plan_t (kind 4) is not the key-major companion of a kind-5 plan" in lib.svgb_last_error()
    assert _bwd(lib, _seg_plan(kind=6), _seg_plan(kind=6)) < 0
    assert b"key-major plans go in plan_t" in lib.svgb_last_error()
    for params in [(1, 600, 0), (0, 600, 1), (0, 599, 0)]:
        assert _bwd(lib, _seg_plan(), _seg_plan(kind=6, params=params)) < 0
        assert b"plan_t was built for another mask than plan" in lib.svgb_last_error()
    # another segment count gives another workspace layout
    assert _bwd(lib, _seg_plan(), _seg_plan(kind=6, layout=(272, 1040, 2064))) < 0
    assert b"another segmentation than plan" in lib.svgb_last_error()


# --------------------------------------------------------------------------------------------
# Python
# --------------------------------------------------------------------------------------------
@pytest.fixture
def recorded(monkeypatch):
    from svgb200 import core

    calls = []
    monkeypatch.setattr(core, "_plan_local_varlen", lambda *a: calls.append(a) or "plan")
    monkeypatch.setattr(core, "_need_cuda", lambda *ts: None)
    return calls


@pytest.mark.parametrize("kw,expect", [
    (dict(causal=True), (0, 700, 0)),
    (dict(causal=True, sink=4), (4, 700, 0)),
    (dict(causal=True, window_size=(128, -1)), (0, 128, 0)),
    (dict(causal=True, window_size=(128, 0)), (0, 128, 0)),
    (dict(window_size=(128, 64)), (0, 128, 64)),
    (dict(window_size=(-1, 3)), (0, 700, 3)),
    (dict(window_size=(0, -1)), (0, 0, 700)),
    (dict(), (0, 700, 700)),
    (dict(window_size=(255, 0), sink=130), (130, 255, 0)),
])
def test_plan_local_varlen_mapping(recorded, kw, expect):
    """FlashAttention's conventions: -1 is unbounded (the larger total covers every segment), causal sets right = 0;
    the bounds go to the planner as int32 with nseg = numel - 1 and are never read on the host."""
    from svgb200 import core

    cu_q = torch.tensor([0, 100, 500])
    cu_k = torch.tensor([0, 300, 700], dtype=torch.int32)
    assert core.plan_local_varlen(cu_q, cu_k, total_q=500, total_k=700, **kw) == "plan"
    (name, pq, pk, nseg, Sq, Skv, *params, dev), = recorded
    assert name == "svgb_attn_plan_local_varlen" and (nseg, Sq, Skv) == (2, 500, 700) and tuple(params) == expect
    assert pq != pk


def test_plan_local_varlen_defaults_and_conflicts(recorded):
    from svgb200 import core

    cu = torch.tensor([0, 3, 9], dtype=torch.int32)
    core.plan_local_varlen(cu, total_q=9, causal=True)
    (_, pq, pk, nseg, Sq, Skv, *params, _), = recorded
    assert pq == pk == cu.data_ptr() and (nseg, Sq, Skv) == (2, 9, 9) and params == [0, 9, 0]
    with pytest.raises(core.SvgbError, match=r"causal=True.*window_size\[1\] = 2"):
        core.plan_local_varlen(cu, total_q=9, causal=True, window_size=(-1, 2))
    with pytest.raises(core.SvgbError, match="same nseg"):
        core.plan_local_varlen(cu, torch.tensor([0, 9], dtype=torch.int32), total_q=9)


def test_segment_plans_know_their_lengths_and_companion(monkeypatch):
    from svgb200 import core

    calls = []
    monkeypatch.setattr(core, "_plan_local_varlen", lambda *a: calls.append(a) or "plan_t")
    p = core.AttnPlan(_seg_plan(Sq=500, Skv=700, params=(2, 30, 0)), torch.zeros(4096, dtype=torch.uint8), (3,))
    assert (p.S, p.S_kv) == (500, 700)
    assert p.key_major() == "plan_t"
    (name, pq, pk, nseg, Sq, Skv, sink, left, right, _), = calls
    base = p.ws.data_ptr() + 16 + 4  # the bounds copy {nseg, cu_q, cu_k}
    assert name == "svgb_attn_plan_local_varlen_t" and (pq, pk) == (base, base + 4 * 4)
    assert (nseg, Sq, Skv, sink, left, right) == (3, 500, 700, 2, 30, 0)


# the drop-in, with the planners and the attention stubbed
@pytest.fixture
def dropin(monkeypatch):
    from svgb200 import core, patch
    from svgb200.models import common

    calls = []
    monkeypatch.setattr(core, "plan_local_varlen", lambda *a, **k: calls.append(("plan_local_varlen", a, k)) or "P")
    monkeypatch.setattr(core, "attention", lambda *a, **k: calls.append(("attention", a[3], k)) or "O")
    monkeypatch.setattr(common, "segment_attention", lambda *a, **k: calls.append(("segment_attention", a[4:6], k))
                        or "S")
    return patch.flash_attn_varlen_func, calls


def _varlen_args():
    q = torch.zeros(500, 4, 64)
    k = torch.zeros(700, 4, 64)
    return q, k, k, torch.tensor([0, 100, 500], dtype=torch.int32), torch.tensor([0, 300, 700], dtype=torch.int32), 400, 400


def test_dropin_default_keywords_take_the_dense_path(dropin):
    fn, calls = dropin
    assert fn(*_varlen_args()) == "S"
    assert fn(*_varlen_args(), causal=False, window_size=(-1, -1), deterministic=True) == "S"
    assert fn(*_varlen_args(), softmax_scale=0.5) == "S"
    assert [c[0] for c in calls] == ["segment_attention"] * 3
    assert calls[0][1] == ([100, 400], [300, 400]) and calls[0][2] == dict(layout="shd", sm_scale=None)
    assert calls[2][2] == dict(layout="shd", sm_scale=0.5)


@pytest.mark.parametrize("kw,plan_kw", [
    (dict(causal=True), dict(causal=True, window_size=(-1, -1))),
    (dict(window_size=(64, 0)), dict(causal=False, window_size=(64, 0))),
    (dict(window_size=(-1, 5), softmax_scale=0.25), dict(causal=False, window_size=(-1, 5))),
    (dict(causal=True, window_size=(100, -1)), dict(causal=True, window_size=(100, -1))),
])
def test_dropin_masks_take_the_segment_plan(dropin, kw, plan_kw):
    fn, calls = dropin
    args = _varlen_args()
    assert fn(*args, **kw) == "O"
    (n1, a1, k1), (n2, plan, k2) = calls
    assert n1 == "plan_local_varlen" and a1 == (args[3], args[4])
    assert k1 == dict(total_q=500, total_k=700, **plan_kw)
    assert n2 == "attention" and plan == "P" and k2 == dict(layout="shd", sm_scale=kw.get("softmax_scale"))


@pytest.mark.parametrize("kw,needle", [(dict(dropout_p=0.1), "dropout_p=0.1"), (dict(softcap=30.0), "softcap=30.0"),
                                       (dict(alibi_slopes=torch.zeros(4)), "alibi_slopes=Tensor"),
                                       (dict(return_attn_probs=True), "return_attn_probs=True"),
                                       (dict(block_table=torch.zeros(2, 2)), "block_table=Tensor")])
def test_dropin_refuses_unsupported_keywords(dropin, kw, needle):
    from svgb200.core import SvgbError

    fn, calls = dropin
    with pytest.raises(SvgbError, match=needle):
        fn(*_varlen_args(), causal=True, **kw)
    with pytest.raises(SvgbError, match=needle):
        fn(*_varlen_args(), **kw)
    assert calls == []
