"""Host side of the local band mask (SVGB_MASK_LOCAL: causal, sliding-window and sink-plus-window attention), without a
GPU: the kernel's predicate against the oracle's, the host mirror of its plan items, the C ABI's refusals,
core.plan_local's translation of FlashAttention's conventions, and which band plans have a backward."""
import ctypes as C
import os
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch

import local_mask as lm
from oracle import attention as oa

ROOT = Path(__file__).resolve().parent.parent
CSRC = ROOT / "sparse-videogen_b200" / "csrc"
PTR = 1 << 20  # never dereferenced: every plan call here fails its argument checks

# mask_allowed(mode, q, kv, m0, m1, m2) of attn_common.cuh, compiled for the host, over every (q, kv) of an S x S grid;
# one case per stdin line "mode m0 m1 m2 S", S * S bytes out per case
PROBE = r"""
#include <cstdio>
#include <vector>
#include "attn_common.cuh"
int main() {
  int mode, m0, m1, m2, S;
  while (std::scanf("%d %d %d %d %d", &mode, &m0, &m1, &m2, &S) == 5) {
    std::vector<unsigned char> out(static_cast<size_t>(S) * S);
    for (int q = 0; q < S; ++q)
      for (int kv = 0; kv < S; ++kv) out[static_cast<size_t>(q) * S + kv] = svgb::mask_allowed(mode, q, kv, m0, m1, m2);
    std::fwrite(out.data(), 1, out.size(), stdout);
  }
  return 0;
}
"""

S_GRID = 700
# (sink, left, right): causal, left- and right-only windows, widths around 256, sinks that are not multiples of 128,
# a sink past S, the diagonal alone
LOCAL_CASES = [(0, S_GRID, 0), (0, 0, S_GRID), (0, 254, 0), (0, 255, 3), (0, 0, 256), (37, 129, 0), (130, 77, 200),
               (1000, 5, 5), (0, 0, 0), (3, 700, 700)]
# (P, W) of MASK_WAN: W and P not multiples of 128
WAN_CASES = [(0, 0), (0, 77), (37, 1), (130, 254), (130, 255), (300, 256), (5, 699), (128, 128)]


@pytest.fixture(scope="module")
def probe(tmp_path_factory):
    nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    d = tmp_path_factory.mktemp("mask_probe")
    (d / "probe.cu").write_text(PROBE)
    subprocess.run([nvcc, "-std=c++17", "-I", str(CSRC), str(d / "probe.cu"), "-o", str(d / "probe")], check=True,
                   capture_output=True)

    def run(cases):
        text = "".join(f"{mode} {m0} {m1} {m2} {S_GRID}\n" for mode, m0, m1, m2 in cases)
        out = subprocess.run([str(d / "probe")], input=text.encode(), capture_output=True, check=True).stdout
        return torch.from_numpy(np.frombuffer(out, np.uint8).reshape(len(cases), S_GRID, S_GRID).astype(bool))

    return run


def _grid(mod):
    idx = torch.arange(S_GRID)
    return mod(idx.view(-1, 1), idx.view(1, -1))


def test_mask_allowed_local_matches_oracle(probe):
    got = probe([(lm.MASK_LOCAL, *c) for c in LOCAL_CASES])
    for i, c in enumerate(LOCAL_CASES):
        want = _grid(lm.local_mask_fn(*c))
        assert torch.equal(got[i], want), f"LOCAL{c}: {int((got[i] != want).sum())} pairs differ"
        assert bool(want.diagonal().all()), "every row keeps its diagonal key"


def test_local_with_equal_sides_is_wan(probe):
    """LOCAL(P, W, W) == WAN(P, W) on every pair: in the kernel's predicate, and in the oracle's two restatements."""
    got = probe([(2, P, 0, W) for P, W in WAN_CASES] + [(lm.MASK_LOCAL, P, W, W) for P, W in WAN_CASES])
    n = len(WAN_CASES)
    for i, (P, W) in enumerate(WAN_CASES):
        want = _grid(oa.generic_mask_fn(2, P, 0, W))
        assert torch.equal(got[i], want), f"WAN({P}, {W}) kernel vs oracle"
        assert torch.equal(got[n + i], want), f"LOCAL({P}, {W}, {W}) kernel vs WAN oracle"
        assert torch.equal(_grid(lm.local_mask_fn(P, W, W)), want), f"LOCAL({P}, {W}, {W}) oracle vs WAN oracle"


def _item_work(mod, S, r0, nr):
    q = torch.arange(r0, r0 + nr).view(-1, 1)
    return int(mod(q, torch.arange(S).view(1, -1)).sum())


@pytest.mark.parametrize("S", [1000, 1025, 4096 + 77])
@pytest.mark.parametrize("sink,left,right", [(0, 10 ** 6, 0), (0, 300, 0), (0, 0, 10 ** 6), (0, 40, 300),
                                             (130, 500, 0), (37, 77, 77), (0, 0, 0)])
def test_band_items_local(S, sink, left, right):
    """The mirror's LOCAL items: every row (key-major: key) in exactly one item, no item across the sink boundary
    key-major, sinks first, and the band segment issued heaviest item first (list work counted from the predicate)."""
    mod = lm.local_mask_fn(sink, left, right)
    for transposed in (False, True):
        items = lm.band_items(lm.MASK_LOCAL, sink, left, right, S, transposed)
        cov = torch.zeros(S, dtype=torch.int32)
        for r0, nr in items:
            assert 0 < nr <= 256
            cov[r0: r0 + nr] += 1
        assert bool((cov == 1).all())
        m = mod if not transposed else (lambda k, q: mod(q, k))
        band = items
        if transposed and 0 < sink < S:
            n_sink = (sink + 255) // 256
            assert [r for r, _ in items[:n_sink]] == list(range(0, sink, 256))
            assert all(r + nr <= sink for r, nr in items[:n_sink])
            band = items[n_sink:]
        one_sided = (right > left) if transposed else (left > right)
        starts = [r for r, _ in band]
        assert starts == sorted(starts, reverse=one_sided)
        work = [_item_work(m, S, r, nr) for r, nr in band if nr == 256]
        assert left == right or work[0] >= work[-1], f"transposed={transposed}: the band's first full item is not its heavy end"


@pytest.mark.parametrize("mode,m0,m1,m2,S", [(1, 900, 1000, 255, 1093), (2, 50, 0, 254, 1100), (3, 3, 130, 129, 1031),
                                             (0, 0, 0, 0, 1000)])
def test_band_items_other_modes_unchanged(mode, m0, m1, m2, S):
    from oracle import bwd_census as bc

    for transposed in (False, True):
        assert lm.band_items(mode, m0, m1, m2, S, transposed) == bc.band_items(mode, m0, m1, S, transposed)


# --------------------------------------------------------------------------------------------
# C ABI
# --------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    import importlib.util

    spec = importlib.util.spec_from_file_location("svgb200_build", ROOT / "sparse-videogen_b200" / "build.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.build_lib()
    from svgb200 import _lib

    return _lib.lib()


@pytest.mark.parametrize("entry", ["svgb_attn_plan_band", "svgb_attn_plan_band_t"])
@pytest.mark.parametrize("args,needle", [((-1, 10, 0), b"sink (m0 = -1)"), ((0, -1, 0), b"left (m1 = -1)"),
                                         ((0, 5, -2), b"right (m2 = -2)")])
def test_plan_refuses_negative_local_parameters(lib, entry, args, needle):
    from svgb200._lib import Plan

    S = 1000
    nbytes = C.c_size_t()
    assert lib.svgb_attn_plan_band_bytes(S, C.byref(nbytes)) == 0
    plan = Plan()
    assert getattr(lib, entry)(lm.MASK_LOCAL, *args, 2, S, PTR, nbytes.value, C.byref(plan), None) < 0
    msg = lib.svgb_last_error()
    assert needle in msg and b">= 0" in msg, msg


def test_plan_refuses_unknown_mode(lib):
    from svgb200._lib import Plan

    nbytes = C.c_size_t()
    assert lib.svgb_attn_plan_band_bytes(1000, C.byref(nbytes)) == 0
    plan = Plan()
    assert lib.svgb_attn_plan_band(11, 0, 0, 0, 2, 1000, PTR, nbytes.value, C.byref(plan), None) < 0
    assert b"unknown mask mode 11" in lib.svgb_last_error()


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
    (dict(causal=True), (0, 500, 0)),
    (dict(causal=True, sink=4), (4, 500, 0)),
    (dict(causal=True, window_size=(128, -1)), (0, 128, 0)),
    (dict(causal=True, window_size=(128, 0)), (0, 128, 0)),
    (dict(window_size=(128, 64)), (0, 128, 64)),
    (dict(window_size=(-1, 3)), (0, 500, 3)),
    (dict(window_size=(7, -1)), (0, 7, 500)),
    (dict(), (0, 500, 500)),
    (dict(window_size=(255, 0), sink=130), (130, 255, 0)),
])
def test_plan_local_mapping(recorded, kw, expect):
    from svgb200 import core

    assert core.plan_local(3, 500, "dev", **kw) == "plan"
    assert recorded == [(core.MASK_LOCAL, *expect, 3, 500, "dev")]


@pytest.mark.parametrize("window", [(-1, 1), (16, 16)])
def test_plan_local_causal_conflict(recorded, window):
    from svgb200 import core

    with pytest.raises(core.SvgbError, match=rf"causal=True.*window_size\[1\] = {window[1]}"):
        core.plan_local(3, 500, "dev", causal=True, window_size=window)
    assert recorded == []


def _band_plan(mode):
    from svgb200 import core
    from svgb200._lib import Plan

    d = Plan()
    d.kind, d.BH, d.S, d.mask_mode, d.m0, d.m1, d.m2 = core.PLAN_BAND, 2, 500, mode, 1, 2, 3
    return core.AttnPlan(d, torch.empty(0, dtype=torch.uint8))


@pytest.mark.parametrize("mode", range(4, 10))
def test_profiling_plans_still_refused_under_grad(mode):
    from svgb200 import core

    x = [torch.zeros(1, 2, 500, 64, dtype=torch.bfloat16, requires_grad=True) for _ in range(3)]
    with pytest.raises(core.SvgbError, match=f"profiling mask mode {mode} has no backward"):
        core.attention(*x, _band_plan(mode))
    with pytest.raises(core.SvgbError, match=f"profiling mask mode {mode} has no backward"):
        _band_plan(mode).key_major()


def test_local_plans_have_a_backward(monkeypatch):
    """Under grad a LOCAL plan reaches the autograd Function, and its key-major plan is the band planner's transpose
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
    plan = _band_plan(core.MASK_LOCAL)
    assert core.attention(*x, plan) == "ran"
    assert plan.key_major() == "plan_t"
    assert calls == [(core.MASK_LOCAL, 1, 2, 3, 2, 500, torch.device("cpu"))]
