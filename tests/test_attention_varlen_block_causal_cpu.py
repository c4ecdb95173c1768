"""Host side of the block-causal mask inside packed variable-length segments (svgb_attn_plan_block_varlen), without a
GPU: the kernels' predicates and both planners' chunk classification compiled for the host against the definition on
every pair, the host mirrors of both planners against a brute-force vote, the key-major interval against the positions
that reach each key, block = 1 against the causal sliding window, every refusal by name, and core's argument
translation."""
import ctypes as C
import os
import random
import shutil
import subprocess

import numpy as np
import pytest
import torch

import block_causal_mask as bm
import varlen_block_causal_mask as vb
import varlen_local_mask as vm
from test_attention_local_cpu import CSRC, lib  # noqa: F401  (lib: the module-scoped library fixture)

PTR = 1 << 20  # never dereferenced: every plan call here fails its argument checks

# The kernels' view of the mask, compiled for the host.  Per case (stdin "nseg sink m1 W" then the sanitised cu_q and
# cu_k): three Sq x Skv grids, each restricted to the row's segment as the plans' chunks are -- the forward's (the
# query row's seg_origin, the row rounded by seg_block_last once, then the local band (sink, W - 1, 0)), and the
# backward's (mask_allowed of the block mode on segment-relative positions) from the query row's and from the key row's
# seg_origin; then, per line "key_major r0 r1 c0 c1", the planner's chunk kind: query-major the item's first and last
# rows rounded and seg_chunk_kind on the band, key-major seg_block_chunk_kind_t.
PROBE = r"""
#include <cstdio>
#include <vector>
#include "attn_common.cuh"
using namespace svgb;
static int seg_of(const int* b, int nseg, int x) { int i = 0; while (i + 1 < nseg && b[i + 1] <= x) ++i; return i; }
int main() {
  int nseg, sink, m1, W;
  while (std::scanf("%d %d %d %d", &nseg, &sink, &m1, &W) == 4) {
    std::vector<int> segs(2 * (nseg + 1) + 1);
    segs[0] = nseg;
    for (size_t i = 1; i < segs.size(); ++i) std::scanf("%d", &segs[i]);
    const int* cq = segs.data() + 1; const int* ck = cq + nseg + 1;
    const int Sq = cq[nseg], Skv = ck[nseg];
    for (int g = 0; g < 3; ++g) {
      std::vector<unsigned char> out(static_cast<size_t>(Sq) * Skv);
      for (int q = 0; q < Sq; ++q)
        for (int kv = 0; kv < Skv; ++kv) {
          const int i = seg_of(cq, nseg, q), j = seg_of(ck, nseg, kv);
          bool a = false;
          if (i == j && q >= cq[i] && q < cq[i + 1] && kv >= ck[j] && kv < ck[j + 1]) {
            const SegOrigin o = seg_origin(segs.data(), g == 2 ? kv : q, g == 2, sink);
            if (g == 0)
              a = mask_allowed(MASK_LOCAL, seg_block_last(q - o.shift, o.key0, m1), kv, o.sink_end, W - 1, 0);
            else
              a = mask_allowed(MASK_BLOCK_CAUSAL, q - o.shift - o.key0, kv - o.key0, o.sink_end - o.key0, m1, W);
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
      const SegOrigin o = seg_origin(segs.data(), r0, km, sink);
      if (km) {
        kinds[t] = seg_block_chunk_kind_t(r0, r1, c0, c1, o, m1, W);
      } else {
        const int a0 = seg_block_last(r0 - o.shift, o.key0, m1) + o.shift;
        const int a1 = seg_block_last(r1 - o.shift, o.key0, m1) + o.shift;
        kinds[t] = seg_chunk_kind(false, a0, a1, c0, c1, o, W - 1, 0);
      }
    }
    std::fwrite(kinds.data(), 1, kinds.size(), stdout);
  }
  return 0;
}
"""

# (cu_q, cu_k, sink, block C, first_block F, window W (-1: unbounded)): one segment, equal and unequal segments, Lq > Lk
# (queries ahead of every key: the first block), Lq < Lk (a KV-cache chunk), empty and 1-token segments, F < C, C = 1,
# a block covering a whole segment, sinks inside, across and longer than a segment, W = C and W > C
CASES = [
    ([0, 300], [0, 300], 0, 128, 128, -1),
    ([0, 100, 357, 358, 700], [0, 100, 357, 358, 700], 0, 50, 20, -1),
    ([0, 200, 201, 460], [0, 77, 300, 300], 0, 64, 64, 128),
    ([0, 130, 130, 400], [0, 390, 391, 650], 5, 100, 30, 250),
    ([0, 259, 500], [0, 259, 500], 3, 40, 40, 40),
    ([0, 1, 257, 513], [0, 500, 501, 513], 300, 129, 1, 129),
    ([0, 0, 129, 129, 390], [0, 1, 1, 400, 401], 2, 7, 3, 21),
    ([0, 520], [0, 1100], 260, 300, 100, 600),
    ([0, 600, 900], [0, 300, 1200], 0, 1, 1, 5),
    ([0, 700], [0, 700], 0, 700, 700, -1),
    ([0, 333, 1000], [0, 500, 1200], 130, 150, 50, 450),
]


def _W(case):
    cu_q, cu_k, _, C_, _, W = case
    return max(cu_q[-1], cu_k[-1]) + C_ if W == -1 else W  # what plan_local_varlen passes for an unbounded window


def _id(c):
    return f"n{len(c[0]) - 1}-q{c[0][-1]}-k{c[1][-1]}-s{c[2]}-C{c[3]}-F{c[4]}-W{c[5]}"


@pytest.fixture(scope="module")
def probe(tmp_path_factory):
    nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    d = tmp_path_factory.mktemp("varlen_block_probe")
    (d / "probe.cu").write_text(PROBE)
    subprocess.run([nvcc, "-std=c++17", "-I", str(CSRC), str(d / "probe.cu"), "-o", str(d / "probe")], check=True,
                   capture_output=True)

    def run(cu_q, cu_k, sink, m1, W, queries):
        text = f"{len(cu_q) - 1} {sink} {m1} {W}\n{' '.join(map(str, cu_q + cu_k))}\n{len(queries)}\n"
        text += "".join(" ".join(map(str, x)) + "\n" for x in queries)
        out = subprocess.run([str(d / "probe")], input=text.encode(), capture_output=True, check=True).stdout
        Sq, Skv = cu_q[-1], cu_k[-1]
        g = np.frombuffer(out[: 3 * Sq * Skv], np.uint8).reshape(3, Sq, Skv).astype(bool)
        return torch.from_numpy(g.copy()), list(out[3 * Sq * Skv:])

    return run


def _all_chunks(cu_q, cu_k, sink, transposed):
    """(r0, r1, c0, c1) of every item and every chunk of its segment, omitted ones included."""
    cb = cu_q if transposed else cu_k
    return [(r0, r0 + nr - 1, c, min(c + 128, cb[i + 1]) - 1)
            for i, r0, nr in vb.item_rows(cu_q, cu_k, sink, transposed) for c in range(cb[i], cb[i + 1], 128)]


@pytest.mark.parametrize("case", CASES, ids=_id)
def test_kernel_predicates_and_chunk_kinds(probe, case):
    """The forward's rounding, the backward's relative predicate in both directions, and both planners' chunk kinds
    equal the definition on every pair and every chunk of every item (0 none, 1 all, 2 some allowed pairs)."""
    cu_q, cu_k, sink, C_, F, W = case
    want = vb.dense(cu_q, cu_k, sink, C_, F, W)
    qs = [(0, *x) for x in _all_chunks(cu_q, cu_k, sink, False)] + [(1, *x) for x in _all_chunks(cu_q, cu_k, sink, True)]
    grids, kinds = probe(cu_q, cu_k, sink, bm.m1_of(C_, F), _W(case), qs)
    for g, name in enumerate(("forward", "backward query-major", "backward key-major")):
        assert torch.equal(grids[g], want), f"{name}: {int((grids[g] != want).sum())} pairs differ"
    for (km, r0, r1, c0, c1), kind in zip(qs, kinds):
        blk = (want.T if km else want)[r0: r1 + 1, c0: c1 + 1]
        exp = 0 if not bool(blk.any()) else 1 if bool(blk.all()) else 2
        assert kind == exp, f"key_major={km} rows {r0}..{r1} cols {c0}..{c1}: kind {kind}, expected {exp}"


def test_definition_anchors_blocks_at_each_segment():
    """Each segment's square block of the packed mask is plan_block_causal's mask on its own (Lq == Lk), and pairs
    across segments are never allowed."""
    cu, sink, C_, F, W = [0, 300, 301, 777, 1000], 5, 70, 20, 140
    m = vb.dense(cu, cu, sink, C_, F, W)
    for i in range(len(cu) - 1):
        a, b = cu[i], cu[i + 1]
        n = b - a
        alone = bm.block_causal_mask_fn(C_, F, W, sink)(torch.arange(n).view(-1, 1), torch.arange(n).view(1, -1))
        assert torch.equal(m[a:b, a:b], alone), f"segment {i}"
        m[a:b, a:b] = False
    assert not bool(m.any())


@pytest.mark.parametrize("case", CASES, ids=_id)
def test_block_one_is_the_causal_window(case):
    """block = 1 is plan_local_varlen(causal=True, window_size=(W - 1, 0)) on every pair of a query at a position
    >= 0.  A query ahead of every key of its segment (Lq_i > Lk_i, position < 0) lies in the first block, so it sees
    key 0 of its segment where the token rule gives it none."""
    cu_q, cu_k, sink, _, _, W = case
    W = _W((cu_q, cu_k, sink, 1, 1, W))
    blk, tok = vb.dense(cu_q, cu_k, sink, 1, 1, W), vm.dense(cu_q, cu_k, sink, W - 1, 0)
    for i in range(len(cu_q) - 1):
        a, b, c, d = cu_q[i], cu_q[i + 1], cu_k[i], cu_k[i + 1]
        ahead = max(0, min((b - a) - (d - c), b - a))  # rows at positions < 0
        assert torch.equal(blk[a + ahead:b], tok[a + ahead:b]), f"segment {i}"
        want = torch.zeros(2, ahead, cu_k[-1], dtype=torch.bool)
        want[0, :, c:min(d, c + max(1, sink))] = True
        want[1, :, c:min(d, c + sink)] = True
        assert torch.equal(blk[a:a + ahead], want[0]) and torch.equal(tok[a:a + ahead], want[1]), f"segment {i}: ahead"


@pytest.mark.parametrize("C_,F,W", [(1, 1, 1), (1, 1, 9), (7, 3, 7), (7, 7, 20), (128, 1, 128), (129, 40, 300),
                                    (300, 300, 1000)])
def test_reach_is_the_interval_of_positions(C_, F, W):
    """block_reach's interval against the brute-force set {p : k + 1 <= e(p) <= k + W}, negative positions included,
    and both bounds nondecreasing in k."""
    prev = None
    for k in range(0, 3 * C_ + 2 * W + 5):
        lo, hi = vb.reach(k, C_, F, W)
        ps = [p for p in range(-2 * C_ - 5, k + W + 2 * C_) if k + 1 <= bm.block_end(p, C_, F) <= k + W]
        assert ps == list(range(ps[0], ps[-1] + 1)) and ps[-1] == hi, (k, lo, hi)
        assert (lo == vb.NEG and ps[0] == -2 * C_ - 5) or ps[0] == lo, (k, lo, ps[0])
        if prev:
            assert lo >= prev[0] and hi >= prev[1]
        prev = (lo, hi)


def _random_case(rng):
    nseg = rng.randint(1, 6)
    lq = [rng.choice([0, 1, rng.randint(0, 600)]) for _ in range(nseg)]
    lk = [rng.choice([0, 1, rng.randint(0, 600)]) for _ in range(nseg)]
    if rng.random() < 0.4:
        lk = list(lq)
    C_ = rng.choice([1, 2, 50, 128, 129, 300])
    F = rng.randint(1, C_)
    W = rng.choice([-1, C_, C_ + rng.randint(0, 500)])
    return vm.sanitize(np.cumsum([0] + lq).tolist(), max(sum(lq), 1)), \
        vm.sanitize(np.cumsum([0] + lk).tolist(), max(sum(lk), 1)), rng.choice([0, 0, 3, 130, 700]), C_, F, W


def test_interval_mirror_equals_the_vote():
    """Both planners' interval forms give the brute-force vote's items, chunks and kinds, in launch order, on random
    packed batches (empty segments, Lq > Lk, Lq < Lk, F < C, sinks and windows)."""
    rng = random.Random(0)
    for _ in range(60):
        case = _random_case(rng)
        cu_q, cu_k, sink, C_, F, W = case
        for transposed in (False, True):
            want = vb.items(cu_q, cu_k, sink, C_, F, W, transposed)
            got = vb.items_interval(cu_q, cu_k, sink, C_, F, _W(case), transposed)
            assert got == want, f"{case} transposed={transposed}"


# --------------------------------------------------------------------------------------------
# C ABI
# --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("entry", ["svgb_attn_plan_block_varlen", "svgb_attn_plan_block_varlen_t"])
@pytest.mark.parametrize("args,needle", [
    ((0, 100, 0, 100), b"block C = 0 must lie in [1, 2^16)"),
    ((0, 70000, 70000, 70000), b"block C = 70000 must lie in [1, 2^16) (it is packed in 16 bits)"),
    ((0, 100, 100, 0), b"first_block F = 0 must lie in [1, C = 100]"),
    ((0, 100, 100, 101), b"first_block F = 101 must lie in [1, C = 100]"),
    ((0, 99, 100, 100), b"window W = 99 must be >= the block C = 100"),
    ((-3, 100, 100, 100), b"sink = -3 must be >= 0"),
])
def test_planner_refusals(lib, entry, args, needle):  # noqa: F811
    from svgb200._lib import Plan

    n = C.c_size_t()
    assert lib.svgb_attn_plan_local_varlen_bytes(3, 600, 700, C.byref(n)) == 0
    assert getattr(lib, entry)(PTR, PTR, 3, 600, 700, *args, PTR, n.value, C.byref(Plan()), None) < 0
    msg = lib.svgb_last_error()
    assert needle in msg and f"{entry}:".encode() in msg, msg


def test_planner_refuses_small_workspace(lib):  # noqa: F811
    from svgb200._lib import Plan

    n = C.c_size_t()
    assert lib.svgb_attn_plan_local_varlen_bytes(3, 600, 700, C.byref(n)) == 0
    assert lib.svgb_attn_plan_block_varlen(PTR, PTR, 3, 600, 700, 0, 200, 100, 50, PTR, n.value - 1, C.byref(Plan()),
                                           None) < 0
    assert b"workspace too small" in lib.svgb_last_error()


def _seg_plan(kind=5, Sq=600, Skv=600, m1=bm.m1_of(100, 50), layout=(256, 1024, 2048)):
    from svgb200._lib import Plan

    p = Plan()
    p.kind, p.S, p.BH = kind, Sq, Skv
    p.mask_mode, p.m0, p.m1, p.m2 = bm.MASK_BLOCK_CAUSAL, 3, m1, 300
    p.max_items, (p.items_off, p.chunks_off, p.bytes) = 8, layout
    return p


def test_forward_and_backward_refusals_stay(lib):  # noqa: F811
    """A block-causal segment plan is refused with e4m3 inputs, row vectors and in the wrong direction, as the local one
    is; the backward wants its key-major companion with the same parameters."""
    S = 600
    fwd = lambda plan, dtype=0, sc=(None, None, None), rows=(None, None, None): lib.svgb_attn_fwd(  # noqa: E731
        PTR, PTR, PTR, *sc, PTR, None, *rows, dtype, 2, S, 128, 128, S * 128, 128, S * 128, 0.1, C.byref(plan), PTR, None)
    assert fwd(_seg_plan(), dtype=2, sc=(PTR, PTR, PTR)) < 0
    assert b"not e4m3" in lib.svgb_last_error()
    assert fwd(_seg_plan(), rows=(None, None, PTR)) < 0
    assert b"row vectors" in lib.svgb_last_error()
    assert fwd(_seg_plan(kind=6)) < 0
    assert b"is for the backward" in lib.svgb_last_error()
    bwd = lambda plan, plan_t: lib.svgb_attn_bwd(  # noqa: E731
        PTR, PTR, PTR, PTR, PTR, PTR, PTR, PTR, PTR, 0, 2, S, 128, 128, S * 128, 0.1, C.byref(plan), PTR,
        C.byref(plan_t), PTR, PTR, 1 << 20, None)
    assert bwd(_seg_plan(), _seg_plan(kind=6, m1=bm.m1_of(100, 49))) < 0
    assert b"plan_t was built for another mask than plan" in lib.svgb_last_error()


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
    (dict(block=300), (0, 1000, 300, 300)),
    (dict(block=300, first_block=77, sink=5), (5, 1000, 300, 77)),
    (dict(block=300, window_size=(900, -1)), (0, 900, 300, 300)),
    (dict(block=1, window_size=(1, -1)), (0, 1, 1, 1)),
])
def test_plan_local_varlen_block_mapping(recorded, kw, expect):
    """block= goes to svgb_attn_plan_block_varlen as (sink, W, C, F); an unbounded window is the longer total + C."""
    from svgb200 import core

    cu_q = torch.tensor([0, 100, 500])
    cu_k = torch.tensor([0, 300, 700], dtype=torch.int32)
    assert core.plan_local_varlen(cu_q, cu_k, total_q=500, total_k=700, **kw) == "plan"
    (name, pq, pk, nseg, Sq, Skv, *params, dev), = recorded
    assert name == "svgb_attn_plan_block_varlen" and (nseg, Sq, Skv) == (2, 500, 700) and tuple(params) == expect
    assert pq != pk


@pytest.mark.parametrize("kw,needle", [
    (dict(block=300, causal=True), "plan_local_varlen: causal=True is redundant with block="),
    (dict(block=300, window_size=(600, 0)), r"plan_local_varlen: with block=, window_size\[1\] = 0 must be -1"),
    (dict(block=300, window_size=(-1, 5)), r"window_size\[1\] = 5 must be -1"),
    (dict(block=1 << 16), "plan_local_varlen: block=65536 must lie in"),
    (dict(block=-2), "plan_local_varlen: block=-2 must lie in"),
    (dict(block=300, first_block=0), "plan_local_varlen: first_block=0 must lie in"),
    (dict(block=300, first_block=301), "plan_local_varlen: first_block=301 must lie in"),
    (dict(block=300, window_size=(299, -1)), "plan_local_varlen: window=299 must be -1"),
    (dict(block=300, sink=-1), "plan_local_varlen: sink=-1 must be >= 0"),
])
def test_plan_local_varlen_block_refusals(recorded, kw, needle):
    """Refused by name before any launch (the bounds here are CPU tensors the planner never reaches)."""
    from svgb200 import core

    cu = torch.tensor([0, 100, 300], dtype=torch.int32)
    with pytest.raises(core.SvgbError, match=needle):
        core.plan_local_varlen(cu, total_q=300, **kw)
    assert recorded == []


def test_block_form_needs_device_bounds():
    """The block form plans on the device only: CPU bounds are refused naming the block-causal mask, and the token
    form keeps its own message."""
    from svgb200 import core

    cu = torch.tensor([0, 100, 300], dtype=torch.int32)
    with pytest.raises(core.SvgbError, match="block-causal masks inside packed segments are not supported on CPU "
                                             r"tensors: svgb200 operators need CUDA tensors \(no CPU fallback\)"):
        core.plan_local_varlen(cu, total_q=300, block=100, first_block=40, window_size=(300, -1))
    with pytest.raises(core.SvgbError, match=r"^svgb200 operators need CUDA tensors \(no CPU fallback\)$"):
        core.plan_local_varlen(cu, total_q=300, causal=True)


def test_block_zero_is_the_token_rule(recorded):
    from svgb200 import core

    cu = torch.tensor([0, 100, 300], dtype=torch.int32)
    core.plan_local_varlen(cu, total_q=300, causal=True, block=0)
    (name, *_, sink, left, right, _), = recorded
    assert name == "svgb_attn_plan_local_varlen" and (sink, left, right) == (0, 300, 0)


def test_key_major_companion(monkeypatch):
    """key_major() of a block-causal segment plan is svgb_attn_plan_block_varlen_t on the plan's own bounds copy with
    the same (sink, W, C, F)."""
    from svgb200 import core

    calls = []
    monkeypatch.setattr(core, "_plan_local_varlen", lambda *a: calls.append(a) or "plan_t")
    p = core.AttnPlan(_seg_plan(Sq=500, Skv=700, m1=bm.m1_of(100, 30)), torch.zeros(4096, dtype=torch.uint8), (3,))
    assert (p.S, p.S_kv) == (500, 700)
    assert p.key_major() == "plan_t"
    (name, pq, pk, nseg, Sq, Skv, *params, _), = calls
    base = p.ws.data_ptr() + 16 + 4
    assert name == "svgb_attn_plan_block_varlen_t" and (pq, pk) == (base, base + 4 * 4)
    assert (nseg, Sq, Skv, *params) == (3, 500, 700, 3, 300, 100, 30)
