"""The local mask inside packed variable-length segments (svgb_attn_plan_local_varlen) on the GPU: every segment of a
packed call bit for bit the same segment run alone, one segment bit for bit plan_local, the unbounded window against
the dense per-segment plan, the exact censuses (forward keys on every row, online softmax, backward keys, integer
gradients), fp64 autograd with an explicit boolean mask, GQA, views, B > 1, out=, determinism, launch counts, no host
synchronisation, and the plans read back against the host mirror.  Outputs go into NaN-filled buffers."""
import pytest
import torch

import local_mask as lm
import varlen_local_mask as vm
from oracle import bwd_census as bc
from oracle import census as oc
from test_attention_bwd_census_gpu import first_bad, run_bwd, run_key
from test_attention_census_gpu import bound_ok, check_census
from test_attention_gqa_gpu import check_exact, run_both

pytestmark = pytest.mark.gpu

DT = {"bf16": torch.bfloat16, "fp16": torch.float16}
BIG = 10 ** 6


def _plan(cuda, cu_q, cu_k, sink, left, right):
    from svgb200 import core

    t = lambda c: torch.tensor(c, dtype=torch.int32, device=cuda)  # noqa: E731
    return core.plan_local_varlen(t(cu_q), t(cu_k), total_q=cu_q[-1], total_k=cu_k[-1], sink=sink,
                                  window_size=(left, right))


def _fwd_bwd(plan, q, k, v, do, layout="bhsd"):
    """o, lse, dq, dk, dv, the outputs in NaN-filled buffers"""
    from svgb200 import core

    o = torch.full_like(q, float("nan"))
    o, lse = core.attn_fwd(q, k, v, plan, layout=layout, return_lse=True, out=o)
    grads = tuple(torch.full_like(t, float("nan")) for t in (q, k, v))
    core.attn_bwd(q, k, v, o, do, lse, plan, layout=layout, out=grads)
    return (o, lse) + grads


def _inputs(H, Sq, Skv, D, dtype, cuda, seed=0, B=1):
    g = torch.Generator().manual_seed(seed)
    q, do = (torch.randn(B, H, Sq, D, generator=g).to(dtype).to(cuda) for _ in range(2))
    k, v = (torch.randn(B, H, Skv, D, generator=g).to(dtype).to(cuda) for _ in range(2))
    return q, k, v, do


def _eq(name, a, b, what):
    bad = ~(a == b)  # NaN (an unwritten element) never matches
    assert not bool(bad.any()), f"{what}: {name} differs in {int(bad.sum())} of {a.numel()} elements"


# --------------------------------------------------------------------------------------------
# packed equals separate, bit for bit
# --------------------------------------------------------------------------------------------
# (lengths q, lengths k, sink, left, right): causal, windows (l, 0), (l, r), (0, r), sinks longer than a segment, empty
# and 1-token segments, bounds off 8 and 128, Lq > Lk (rows without keys) and Lq < Lk
PACKED = [
    ([300, 1, 777, 0, 130], None, 0, BIG, 0),
    ([513, 250, 1000], None, 0, 200, 0),
    ([513, 250, 1000], None, 0, 129, 40),
    ([700, 259, 3], None, 0, 0, 300),
    ([400, 90, 257], None, 500, 64, 0),
    ([300, 500, 0, 77], [100, 900, 60, 0], 0, BIG, 0),
    ([129, 1000, 5], [1000, 129, 5], 7, 255, 0),
    ([1, 640, 333], [300, 2000, 333], 33, 517, 13),
]


def _cu(lens):
    out = [0]
    for n in lens:
        out.append(out[-1] + n)
    return out


@pytest.mark.parametrize("D,dtype", [(128, "bf16"), (64, "fp16")])
@pytest.mark.parametrize("case", range(len(PACKED)))
def test_packed_equals_separate(cuda, case, D, dtype):
    """Every segment's o, lse, dq, dk, dv from one packed call equal the segment run alone: through plan_local when
    Lq == Lk, through a one-segment rectangular plan otherwise; a query segment with no keys gives o = 0, lse = -inf,
    dq = 0, a key segment no query reaches dk = dv = 0."""
    from svgb200 import core

    lq, lk, sink, left, right = PACKED[case]
    lk = lq if lk is None else lk
    cu_q, cu_k = _cu(lq), _cu(lk)
    H, dt = 3, DT[dtype]
    q, k, v, do = _inputs(H, cu_q[-1], cu_k[-1], D, dt, cuda, seed=case)
    packed = _fwd_bwd(_plan(cuda, cu_q, cu_k, sink, left, right), q, k, v, do)
    for i in range(len(lq)):
        a, b, c, d = cu_q[i], cu_q[i + 1], cu_k[i], cu_k[i + 1]
        what = f"segment {i} ({b - a} x {d - c})"
        got = [packed[0][:, :, a:b], packed[1].view(H, -1)[:, a:b], packed[2][:, :, a:b], packed[3][:, :, c:d],
               packed[4][:, :, c:d]]
        if b == a and d == c:
            continue
        if d == c or b == a:
            for name, x in zip(("o", "dq"), (got[0], got[2])):
                assert bool((x == 0).all()), f"{what}: {name} not zero"
            assert bool((got[1] == -float("inf")).all()), f"{what}: lse"
            for name, x in zip(("dk", "dv"), got[3:]):
                assert bool((x == 0).all()), f"{what}: {name} not zero"
            continue
        if b - a == d - c:
            alone_plan = core.plan_local(H, b - a, cuda, window_size=(min(left, b - a), right), sink=sink)
        else:
            alone_plan = _plan(cuda, [0, b - a], [0, d - c], sink, left, right)
        alone = _fwd_bwd(alone_plan, *(t[:, :, x:y].contiguous() for t, x, y in
                                       ((q, a, b), (k, c, d), (v, c, d), (do, a, b))))
        alone = [alone[0], alone[1].view(H, -1), *alone[2:]]
        for name, x, y in zip(("o", "lse", "dq", "dk", "dv"), got, alone):
            _eq(name, x, y, what)


@pytest.mark.parametrize("S,args", [(1100, (0, BIG, 0)), (3000, (37, 255, 0)), (2049, (0, 100, 300)),
                                    (119056, (0, BIG, 0))], ids=["causal", "sink-left", "two-sided", "hy720-causal"])
def test_one_segment_equals_plan_local(cuda, S, args):
    """nseg = 1, Sq == Skv: o, lse, dq, dk, dv of the segment plan are plan_local's bit for bit (HunyuanVideo 720p
    causal included)."""
    from svgb200 import core

    sink, left, right = args
    H = 2
    q, k, v, do = _inputs(H, S, S, 128, torch.bfloat16, cuda, seed=S)
    a = _fwd_bwd(_plan(cuda, [0, S], [0, S], sink, left, right), q, k, v, do)
    b = _fwd_bwd(core.plan_local(H, S, cuda, window_size=(min(left, S), min(right, S)), sink=sink), q, k, v, do)
    for name, x, y in zip(("o", "lse", "dq", "dk", "dv"), a, b):
        _eq(name, x, y, f"S={S} LOCAL{args}")


def test_unbounded_window_equals_dense_segments(cuda):
    """With the window unbounded and no sink every chunk is FULL, and each row sees the chunks that
    models.common.segment_attention's diagonal variable-block plan gives it, in the same order: o, lse, dq, dk, dv
    bit for bit."""
    from svgb200 import core
    from svgb200.models.common import segment_attention

    lq, lk = [300, 1, 777, 130, 1000], [500, 1, 777, 20, 60]
    cu_q, cu_k = _cu(lq), _cu(lk)
    H = 4
    q, k, v, do = _inputs(H, cu_q[-1], cu_k[-1], 128, torch.bfloat16, cuda, seed=5)
    plan = core.plan_local_varlen(*(torch.tensor(c, dtype=torch.int32, device=cuda) for c in (cu_q, cu_k)),
                                  total_q=cu_q[-1], total_k=cu_k[-1])
    got = []
    for f in (lambda x, y, z: core.attention(x, y, z, plan),
              lambda x, y, z: segment_attention("test", x, y, z, lq, lk)):
        xs = [t.clone().requires_grad_() for t in (q, k, v)]
        o = f(*xs)
        o.backward(do)
        got.append([o.detach()] + [t.grad for t in xs])
    for name, x, y in zip(("o", "dq", "dk", "dv"), *got):
        _eq(name, x, y, "unbounded window vs segment_attention")


# --------------------------------------------------------------------------------------------
# censuses
# --------------------------------------------------------------------------------------------
# square totals with unequal segments, so the census oracles (S x S) apply: rows without keys (Lq > Lk under causal),
# Lq < Lk, sinks, bounds off 8 and 128
CENSUS = [
    ([0, 300, 301, 1100], [0, 100, 700, 1100], 0, BIG, 0),
    ([0, 129, 700, 1100], [0, 129, 700, 1100], 37, 200, 0),
    ([0, 500, 500, 1100], [0, 260, 261, 1100], 3, 40, 129),
    ([0, 1, 1100], [0, 1000, 1100], 0, 0, 255),
]


def _cid(c):
    return f"n{len(c[0]) - 1}-s{c[2]}-l{min(c[3], 9999)}-r{c[4]}"


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("case", CENSUS, ids=_cid)
def test_census_varlen(cuda, case, D, dtype):
    """The forward key census on every row: which keys each row saw, how often, and its lse."""
    from svgb200 import core

    cu_q, cu_k, *args = case
    S, H, dt = cu_q[-1], 2, DT[dtype]
    plan = _plan(cuda, cu_q, cu_k, *args)
    cnt, n = oc.band_census(vm.mask_fn(cu_q, cu_k, *args), S, D, cuda)
    cnt, n = cnt.cpu(), n.cpu()
    bound_ok([cnt], dt)
    q = torch.zeros(1, H, S, D, dtype=dt, device=cuda)
    k = torch.randn(1, H, S, D, device=cuda).to(dt)
    for enc in oc.ENCODINGS:
        v = oc.identity_values(S, D, enc, H, dt, cuda)
        o, lse = core.attn_fwd(q, k, v, plan, return_lse=True, out=torch.full_like(q, float("nan")))
        check_census(o[0], lse, [cnt] * H, [n] * H, enc, f"varlen {case} D={D} {dtype}")


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("D", [64, 128])
def test_softmax_varlen(cuda, monkeypatch, D, dtype):
    """The softmax census's Wan case (S = 1260) in three causal segments: integer log2 scores that move the running
    max, every row bit for bit."""
    import test_softmax_census_gpu as tsc
    from oracle import softmax as sm

    cu_q, cu_k, args = [0, 400, 401, 1260], [0, 130, 700, 1260], (2, BIG, 0)
    case = sm.band_case("wan", D=D)
    case.band, case.mod = (lm.MASK_LOCAL, *args), vm.mask_fn(cu_q, cu_k, *args)
    monkeypatch.setattr(tsc, "_plan", lambda cuda_, case_: _plan(cuda_, cu_q, cu_k, *args))
    tsc.run(cuda, case, DT[dtype], f"varlen softmax D={D} {dtype}")


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("case", CENSUS, ids=_cid)
def test_key_census_varlen(cuda, case, D, dtype):
    cu_q, cu_k, *args = case
    S = cu_q[-1]
    plan = _plan(cuda, cu_q, cu_k, *args)
    tab = bc.band_tables(vm.mask_fn(cu_q, cu_k, *args), S, D, cuda)
    run_key(cuda, plan, [tab] * 2, S, D, DT[dtype], f"varlen {case} D={D} {dtype}")


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("case", CENSUS[:3], ids=_cid)
def test_grad_census_varlen(cuda, case, D, dtype):
    """Real scores and values with every intermediate exact, all eight backward instantiations."""
    cu_q, cu_k, *args = case
    S = cu_q[-1]
    mod = vm.mask_fn(cu_q, cu_k, *args)
    g = torch.Generator().manual_seed(S)
    gc = bc.GradCase(f"varlen{args}", S, D, 2, 1.0, *bc._grad_inputs(2, S, D, 1.0, g), band=(lm.MASK_LOCAL, *args),
                     mod=mod)
    dt = DT[dtype]
    got = run_bwd(cuda, _plan(cuda, cu_q, cu_k, *args), (gc.q, gc.k, gc.v, gc.o, gc.do), gc.lse(), dt, gc.sm_scale)
    for h in range(gc.H):
        _, budget, stats = bc.grad_exact(gc, h, cuda)
        assert max(budget) < bc.BUDGET and stats["ds_exact"] and stats["ds_max"] <= 8, f"head {h} not exact"
        for name, x, e in zip(("dq", "dk", "dv"), got, bc.grad_expected(gc, h, dt, cuda)):
            b = first_bad(x[h], e.cpu())
            assert b is None, f"{name} first differs at (head {h}, row {b[0]}, column {b[1]}) of {b[2]} rows"


# --------------------------------------------------------------------------------------------
# fp64 autograd with an explicit boolean mask
# --------------------------------------------------------------------------------------------
def _ref64(q, k, v, do, m, scale):
    x = [t.double().requires_grad_() for t in (q, k, v)]
    s = (x[0] @ x[1].transpose(-1, -2)) * scale
    s = s.masked_fill(~m, float("-inf"))
    p = torch.nan_to_num(torch.softmax(s, -1), nan=0.0)
    o = p @ x[2]
    o.backward(do.double())
    return [o.detach()] + [t.grad for t in x]


def _rel(a, b):
    d = float(b.double().norm())
    return float((a.double() - b.double()).norm()) / (d if d > 0 else 1.0)


@pytest.mark.parametrize("name", ["rows-without-keys", "kv-cache", "mixed"])
def test_matches_fp64_autograd(cuda, name):
    """Lq > Lk (rows without keys), a KV-cache chunk (4 680 queries against 32 760 keys, sink 1 560, window 14 040)
    and a mixed packed batch, against fp64 autograd under the explicit boolean mask: o, dq, dk, dv norm-wise."""
    from svgb200 import core

    if name == "rows-without-keys":
        cu_q, cu_k, args = [0, 900, 1000], [0, 300, 1500], (0, BIG, 0)
    elif name == "kv-cache":
        cu_q, cu_k, args = [0, 4680], [0, 32760], (1560, 14040, 0)
    else:
        cu_q, cu_k, args = [0, 1000, 1001, 2500, 2500, 3100], [0, 1000, 1300, 2000, 2128, 2728], (4, 600, 0)
    H, D = 2, 128
    q, k, v, do = _inputs(H, cu_q[-1], cu_k[-1], D, torch.bfloat16, cuda, seed=len(name))
    m = vm.mask_fn(cu_q, cu_k, *args)(torch.arange(cu_q[-1], device=cuda).view(-1, 1),
                                      torch.arange(cu_k[-1], device=cuda).view(1, -1))
    ref = _ref64(q, k, v, do, m.to(cuda), D ** -0.5)
    x = [t.clone().requires_grad_() for t in (q, k, v)]
    o = core.attention(*x, _plan(cuda, cu_q, cu_k, *args))
    o.backward(do)
    for nm, a, b in zip(("o", "dq", "dk", "dv"), [o.detach()] + [t.grad for t in x], ref):
        assert bool(torch.isfinite(a).all()), f"{name}: {nm} not finite"
        assert _rel(a, b) < 1e-2, f"{name}: {nm} relative difference {_rel(a, b):.2e}"
    if name == "rows-without-keys":
        assert bool((o[:, :, :600] == 0).all()) and bool((x[0].grad[:, :, :600] == 0).all())


# --------------------------------------------------------------------------------------------
# layouts, determinism, launch counts, synchronisation, plan read-back
# --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("Hkv", [16, 8, 1])
def test_gqa_varlen(cuda, Hkv):
    """GQA / MQA on a shared segment plan (Sq != Skv): o, lse, dq bit for bit the MHA call on repeated K / V, dk / dv
    its group sums."""
    cu_q, cu_k, args = [0, 1000, 1001, 2500], [0, 1200, 1300, 3100], (3, 700, 0)
    p = _plan(cuda, cu_q, cu_k, *args)
    check_exact(*run_both(cuda, p, p, 16, Hkv, cu_q[-1], cu_k[-1], 128, torch.bfloat16), 16 // Hkv, torch.bfloat16,
                "bhsd", f"Hkv={Hkv}")


@pytest.mark.parametrize("view", ["bshd-B2", "unbind", "shd"])
def test_views_varlen(cuda, view):
    """Transposed [B, S, H, D] views with B = 2 (every batch element segmented alike), one third of a packed QKV, and
    the packed [total, H, D] layout match the contiguous [B, H, S, D] call bit for bit, forward and backward."""
    B = 2 if view == "bshd-B2" else 1
    H, D = 4, 128
    cu = [0, 700, 701, 2000]
    plan = _plan(cuda, cu, cu, 0, BIG, 0)
    S = cu[-1]
    g = torch.Generator().manual_seed(B)
    if view == "unbind":
        qkv = torch.randn(B, S, 3, H, D, generator=g).to(torch.bfloat16).to(cuda)
        base = [t for t in qkv.unbind(2)] + [torch.randn(B, S, H, D, generator=g).to(torch.bfloat16).to(cuda)]
    else:
        base = [torch.randn(B, S, H, D, generator=g).to(torch.bfloat16).to(cuda) for _ in range(4)]
    ref = _fwd_bwd(plan, *(t.transpose(1, 2).contiguous() for t in base))
    if view == "shd":
        got = _fwd_bwd(plan, *(t[0].contiguous() for t in base), layout="shd")
        got = [got[0][None].transpose(1, 2), got[1]] + [t[None].transpose(1, 2) for t in got[2:]]
    else:
        got = _fwd_bwd(plan, *(t.transpose(1, 2) for t in base))
    for name, a, b in zip(("o", "lse", "dq", "dk", "dv"), got, ref):
        _eq(name, a, b, view)


def test_batch_elements_and_determinism(cuda):
    """B = 2 in 'bhsd': each batch element equals its own B = 1 call; two backward calls give the same bits."""
    from svgb200 import core

    cu_q, cu_k = [0, 333, 1000], [0, 500, 1200]
    plan = _plan(cuda, cu_q, cu_k, 0, 300, 0)
    q, k, v, do = _inputs(3, 1000, 1200, 64, torch.float16, cuda, seed=9, B=2)
    both = _fwd_bwd(plan, q, k, v, do)
    for b in range(2):
        one = _fwd_bwd(plan, q[b:b + 1], k[b:b + 1], v[b:b + 1], do[b:b + 1])
        for name, x, y in zip(("o", "lse", "dq", "dk", "dv"), both, one):
            x = x.view(2, -1, *x.shape[1:])[b] if name == "lse" else x[b:b + 1]
            _eq(name, x, y.view_as(x), f"batch {b}")
    dq, dk, dv = core.attn_bwd(q, k, v, both[0], do, both[1], plan)
    for name, x, y in zip(("dq", "dk", "dv"), (dq, dk, dv), both[2:]):
        _eq(name, x, y, "second backward")


def test_dropin_causal(cuda):
    """patch.flash_attn_varlen_func(causal=True, softmax_scale=s) is the segment plan's attention at scale s."""
    from svgb200 import core, patch

    cu_q, cu_k = [0, 300, 1000], [0, 300, 1400]
    g = torch.Generator().manual_seed(3)
    q = torch.randn(1000, 4, 128, generator=g).to(torch.bfloat16).to(cuda)
    k, v = (torch.randn(1400, 4, 128, generator=g).to(torch.bfloat16).to(cuda) for _ in range(2))
    t = lambda c: torch.tensor(c, dtype=torch.int32, device=cuda)  # noqa: E731
    o = patch.flash_attn_varlen_func(q, k, v, t(cu_q), t(cu_k), 700, 1100, causal=True, softmax_scale=0.05)
    ref = core.attn_fwd(q, k, v, _plan(cuda, cu_q, cu_k, 0, BIG, 0), layout="shd", sm_scale=0.05)
    _eq("o", o, ref, "drop-in")


def test_launch_counts_and_no_host_sync(cuda):
    """Two launches to plan, one forward, three backward (two more the first time, for the key-major plan), and
    none of it synchronises with the host."""
    from svgb200 import core

    cu = torch.tensor([0, 1000, 1001, 3000], dtype=torch.int32, device=cuda)
    q, k, v, do = _inputs(2, 3000, 3000, 128, torch.bfloat16, cuda)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        n0 = core.launch_count
        plan = core.plan_local_varlen(cu, total_q=3000, causal=True, sink=4)
        assert core.launch_count - n0 == 2
        n0 = core.launch_count
        o, lse = core.attn_fwd(q, k, v, plan, return_lse=True)
        assert core.launch_count - n0 == 1
        n0 = core.launch_count
        core.attn_bwd(q, k, v, o, do, lse, plan)
        assert core.launch_count - n0 == 5
        n0 = core.launch_count
        core.attn_bwd(q, k, v, o, do, lse, plan)
        assert core.launch_count - n0 == 3
    finally:
        torch.cuda.set_sync_debug_mode(0)


def _read(plan):
    """(bounds copy, items [(row0, nrows, [(col0, valid, elem)])] in launch order) of a segment plan"""
    d = plan.desc
    ws = plan.ws.cpu()
    i32 = lambda off, n: ws[off: off + 4 * n].clone().view(torch.int32)  # noqa: E731
    nseg = int(i32(16, 1)[0])  # SVGB_PLAN_SEG_BOUNDS_OFF: {nseg, cu_q, cu_k}
    assert (nseg,) == plan.source
    segs = i32(20, 2 * (nseg + 1)).tolist()
    n = int(i32(d.counts_off, 1)[0])
    assert 0 <= n <= d.max_items
    its = i32(d.items_off, 8 * n).view(n, 2, 4)
    chunks = i32(d.chunks_off, (ws.numel() - d.chunks_off) // 4).view(-1, 2)
    out = []
    for it in its:
        (r0, n0, off, ln), (r1, n1, off1, ln1) = it.tolist()
        assert (off1, ln1, r1) == (off, ln, r0 + 128) and n0 == min(128, n0 + n1)
        assert 0 <= off and off + ln <= chunks.shape[0]
        lst = [(int(c), (int(m) & 0xff) + 1, bool(int(m) & 256)) for c, m in chunks[off: off + ln]]
        out.append((r0, n0 + n1, lst))
    return segs, out


# (cu_q, cu_k, total_q, total_k, sink, left, right): the packed cases, and malformed bounds (out of order, negative,
# past the totals, a first bound other than 0) that are planned and never run
READ_BACK = [(_cu(lq), _cu(lq if lk is None else lk), sum(lq), sum(lq if lk is None else lk), *a)
             for lq, lk, *a in PACKED[:6]] + [([0, 5, 3, 9], [4, -7, 20, 6], 9, 12, 1, 3, 0)]


@pytest.mark.parametrize("case", READ_BACK, ids=lambda c: f"{c[2]}x{c[3]}-n{len(c[0]) - 1}")
def test_plan_read_back(cuda, case):
    """Both plans built on the GPU, read back: the bounds copy (malformed bounds clamped and made monotone), every
    item, chunk and kind, in launch order, equal the host mirror's; every row and chunk lies inside the totals."""
    raw_q, raw_k, Sq, Skv, sink, left, right = case
    from svgb200 import core

    t = lambda c: torch.tensor(c, dtype=torch.int32, device=cuda)  # noqa: E731
    plan = core.plan_local_varlen(t(raw_q), t(raw_k), total_q=Sq, total_k=Skv, sink=sink,
                                  window_size=(min(left, max(Sq, Skv)), right))
    cu_q, cu_k = vm.sanitize(raw_q, Sq), vm.sanitize(raw_k, Skv)
    for p, transposed in ((plan, False), (plan.key_major(), True)):
        segs, got = _read(p)
        assert segs == cu_q + cu_k
        want = vm.items(cu_q, cu_k, sink, min(left, max(Sq, Skv)), right, transposed)
        assert got == want, f"transposed={transposed}: first difference at item " \
                            f"{next(i for i, (a, b) in enumerate(zip(got + [None], want + [None])) if a != b)}"
        rows, cols = (Skv, Sq) if transposed else (Sq, Skv)
        for r0, nr, lst in got:
            assert 0 <= r0 and r0 + nr <= rows and all(0 <= c and c + v <= cols for c, v, _ in lst)
