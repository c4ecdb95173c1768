"""The block-causal mask inside packed variable-length segments (plan_local_varlen(block=)) on the GPU: the forward key
census, the backward key and integer-gradient censuses, fp64 autograd with B = 2 and GQA, determinism, the bit-for-bit
identities (one segment is plan_block_causal, every packed segment its own call, block = 1 the causal window, a
short-query segment the block-causal KV-cache plan), GQA, strided views, the plans read back against the host mirror,
and compiled flex_attention under a document-block-causal mask at the perf tool's shape.  Outputs and gradients go
into NaN-filled buffers."""
import pytest
import torch

import block_causal_mask as bm
import varlen_block_causal_mask as vb
from oracle import bwd_census as bc
from oracle import census as oc
from test_attention_bwd_census_gpu import first_bad, run_bwd, run_key
from test_attention_census_gpu import bound_ok, check_census
from test_attention_gqa_gpu import check_exact, run_both
from test_attention_varlen_local_gpu import _cu, _eq, _fwd_bwd, _inputs, _read, _ref64, _rel

pytestmark = pytest.mark.gpu

DT = {"bf16": torch.bfloat16, "fp16": torch.float16}


def _plan(cuda, cu_q, cu_k, sink, C_, F, W):
    from svgb200 import core

    t = lambda c: torch.tensor(c, dtype=torch.int32, device=cuda)  # noqa: E731
    return core.plan_local_varlen(t(cu_q), t(cu_k), total_q=cu_q[-1], total_k=cu_k[-1], block=C_, first_block=F,
                                  window_size=(W, -1), sink=sink)


# --------------------------------------------------------------------------------------------
# censuses (square totals with unequal segments, so the S x S census oracles apply)
# --------------------------------------------------------------------------------------------
# (cu_q, cu_k, sink, C, F, W): queries ahead of their keys (Lq > Lk), Lq < Lk, an empty segment, F < C, sinks, windows
CENSUS = [
    ([0, 300, 301, 1100], [0, 100, 700, 1100], 0, 128, 128, -1),
    ([0, 129, 700, 1100], [0, 129, 700, 1100], 37, 100, 30, 200),
    ([0, 500, 500, 1100], [0, 260, 261, 1100], 3, 129, 1, 258),
    ([0, 1, 1100], [0, 1000, 1100], 0, 300, 77, 300),
]


def _cid(c):
    return f"n{len(c[0]) - 1}-s{c[2]}-C{c[3]}-F{c[4]}-W{c[5]}"


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("case", CENSUS, ids=_cid)
def test_census(cuda, case, D, dtype):
    """Forward key census: every row keeps exactly its key set, how often it saw each key, and its lse."""
    from svgb200 import core

    cu_q, cu_k, *args = case
    S, H, dt = cu_q[-1], 2, DT[dtype]
    plan = _plan(cuda, cu_q, cu_k, *args)
    cnt, n = oc.band_census(vb.mask_fn(cu_q, cu_k, *args), S, D, cuda)
    cnt, n = cnt.cpu(), n.cpu()
    bound_ok([cnt], dt)
    q = torch.zeros(1, H, S, D, dtype=dt, device=cuda)
    k = torch.randn(1, H, S, D, device=cuda).to(dt)
    for enc in oc.ENCODINGS:
        v = oc.identity_values(S, D, enc, H, dt, cuda)
        o, lse = core.attn_fwd(q, k, v, plan, return_lse=True, out=torch.full_like(q, float("nan")))
        check_census(o[0], lse, [cnt] * H, [n] * H, enc, f"varlen block {case} D={D} {dtype}")


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("case", CENSUS, ids=_cid)
def test_key_census(cuda, case, D, dtype):
    """Backward key census: dq, dk, dv count exactly the allowed pairs of every row and key, both launches."""
    cu_q, cu_k, *args = case
    S = cu_q[-1]
    tab = bc.band_tables(vb.mask_fn(cu_q, cu_k, *args), S, D, cuda)
    run_key(cuda, _plan(cuda, cu_q, cu_k, *args), [tab] * 2, S, D, DT[dtype], f"varlen block {case} D={D} {dtype}")


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("case", CENSUS[:3], ids=_cid)
def test_grad_census(cuda, case, D, dtype):
    """Real scores and values with every intermediate exact, all eight backward instantiations, bit for bit."""
    cu_q, cu_k, sink, C_, F, W = case
    S = cu_q[-1]
    mod = vb.mask_fn(cu_q, cu_k, sink, C_, F, W)
    g = torch.Generator().manual_seed(S)
    gc = bc.GradCase(f"varlen block {case}", S, D, 2, 1.0, *bc._grad_inputs(2, S, D, 1.0, g),
                     band=(bm.MASK_BLOCK_CAUSAL, sink, bm.m1_of(C_, F), S + C_ if W == -1 else W), mod=mod)
    dt = DT[dtype]
    got = run_bwd(cuda, _plan(cuda, cu_q, cu_k, sink, C_, F, W), (gc.q, gc.k, gc.v, gc.o, gc.do), gc.lse(), dt,
                  gc.sm_scale)
    for h in range(gc.H):
        _, budget, stats = bc.grad_exact(gc, h, cuda)
        assert max(budget) < bc.BUDGET and stats["ds_exact"] and stats["ds_max"] <= 8, f"head {h} not exact"
        for name, x, e in zip(("dq", "dk", "dv"), got, bc.grad_expected(gc, h, dt, cuda)):
            b = first_bad(x[h], e.cpu())
            assert b is None, f"{name} first differs at (head {h}, row {b[0]}, column {b[1]}) of {b[2]} rows"


# --------------------------------------------------------------------------------------------
# fp64 autograd, B = 2, GQA, determinism
# --------------------------------------------------------------------------------------------
def test_fp64_autograd_batch_gqa_determinism(cuda):
    """B = 2, Hq = 4 over Hkv = 2, a packed batch with Lq > Lk, Lq < Lk, an empty and a 1-token segment, F < C, a
    window and a sink: o, dq, dk, dv against fp64 autograd under the explicit boolean mask, and a second call gives the
    same bits."""
    from svgb200 import core

    cu_q, cu_k = [0, 1000, 1001, 2500, 2500, 3100], [0, 700, 1300, 2000, 2128, 2728]
    args = (4, 300, 100, 600)
    B, Hq, Hkv, D = 2, 4, 2, 64
    g = torch.Generator().manual_seed(21)
    q, do = (torch.randn(B, Hq, cu_q[-1], D, generator=g).to(torch.bfloat16).to(cuda) for _ in range(2))
    k, v = (torch.randn(B, Hkv, cu_k[-1], D, generator=g).to(torch.bfloat16).to(cuda) for _ in range(2))
    m = vb.mask_fn(cu_q, cu_k, *args)(torch.arange(cu_q[-1], device=cuda).view(-1, 1),
                                      torch.arange(cu_k[-1], device=cuda).view(1, -1))
    ref = _ref64(q, k.repeat_interleave(Hq // Hkv, 1), v.repeat_interleave(Hq // Hkv, 1), do, m, D ** -0.5)
    ref[2:] = [t.view(B, Hkv, Hq // Hkv, *t.shape[2:]).sum(2) for t in ref[2:]]
    plan = _plan(cuda, cu_q, cu_k, *args)
    runs = []
    for _ in range(2):
        x = [t.clone().requires_grad_() for t in (q, k, v)]
        o = core.attention(*x, plan)
        o.backward(do)
        runs.append([o.detach()] + [t.grad for t in x])
    for name, a, a2, b in zip(("o", "dq", "dk", "dv"), *runs, ref):
        assert bool(torch.isfinite(a).all()), f"{name} not finite"
        assert torch.equal(a, a2), f"{name}: not deterministic"
        assert _rel(a, b) < 1e-2, f"{name}: relative difference {_rel(a, b):.2e}"


@pytest.mark.parametrize("Hkv", [8, 1])
def test_gqa(cuda, Hkv):
    """GQA / MQA on a shared block-causal segment plan (Sq != Skv): o, lse, dq bit for bit the MHA call on repeated
    K / V, dk / dv its group sums."""
    cu_q, cu_k = [0, 1000, 1001, 2500], [0, 1200, 1300, 3100]
    p = _plan(cuda, cu_q, cu_k, 3, 300, 100, 900)
    check_exact(*run_both(cuda, p, p, 16, Hkv, cu_q[-1], cu_k[-1], 128, torch.bfloat16), 16 // Hkv, torch.bfloat16,
                "bhsd", f"block Hkv={Hkv}")


# --------------------------------------------------------------------------------------------
# bit-for-bit identities
# --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S,args", [(1100, (0, 300, 300, -1)), (3000, (130, 700, 200, 1400)), (2049, (0, 1, 1, 255)),
                                    (4680 * 7, (1560, 4680, 1560, 14040))], ids=["chunks", "window-sink", "block1",
                                                                                 "wan-i2v"])
def test_one_segment_equals_plan_block_causal(cuda, S, args):
    """nseg = 1, Sq == Skv: o, lse, dq, dk, dv are plan_block_causal's bit for bit."""
    from svgb200 import core

    sink, C_, F, W = args
    H = 2
    q, k, v, do = _inputs(H, S, S, 128, torch.bfloat16, cuda, seed=S)
    a = _fwd_bwd(_plan(cuda, [0, S], [0, S], *args), q, k, v, do)
    b = _fwd_bwd(core.plan_block_causal(H, S, cuda, block=C_, first_block=F, window=W, sink=sink), q, k, v, do)
    for name, x, y in zip(("o", "lse", "dq", "dk", "dv"), a, b):
        _eq(name, x, y, f"S={S} BLOCK{args}")


# (lengths q, lengths k (None: the same), sink, C, F, W)
PACKED = [
    ([21 * 156, 13 * 156, 9 * 156, 5 * 156], None, 0, 3 * 156, 156, -1),
    ([21 * 156, 13 * 156, 9 * 156, 5 * 156], None, 156, 3 * 156, 156, 6 * 156),
    ([300, 1, 777, 0, 130], None, 0, 128, 50, -1),
    ([513, 250, 1000], None, 37, 129, 129, 258),
    ([300, 500, 0, 77], [100, 900, 60, 0], 0, 100, 40, -1),
    ([129, 1000, 5], [1000, 129, 5], 7, 64, 64, 256),
]


@pytest.mark.parametrize("D,dtype", [(128, "bf16"), (64, "fp16")])
@pytest.mark.parametrize("case", range(len(PACKED)))
def test_packed_equals_separate(cuda, case, D, dtype):
    """Every segment's o, lse, dq, dk, dv from one packed call equal the segment run alone: through plan_block_causal on
    its own slice when Lq == Lk, through a one-segment plan otherwise; a query segment with no keys gives o = 0,
    lse = -inf, dq = 0, a key segment no query reaches dk = dv = 0."""
    from svgb200 import core

    lq, lk, sink, C_, F, W = PACKED[case]
    lk = lq if lk is None else lk
    cu_q, cu_k = _cu(lq), _cu(lk)
    H, dt = 3, DT[dtype]
    q, k, v, do = _inputs(H, cu_q[-1], cu_k[-1], D, dt, cuda, seed=case)
    packed = _fwd_bwd(_plan(cuda, cu_q, cu_k, sink, C_, F, W), q, k, v, do)
    for i in range(len(lq)):
        a, b, c, d = cu_q[i], cu_q[i + 1], cu_k[i], cu_k[i + 1]
        what = f"segment {i} ({b - a} x {d - c})"
        got = [packed[0][:, :, a:b], packed[1].view(H, -1)[:, a:b], packed[2][:, :, a:b], packed[3][:, :, c:d],
               packed[4][:, :, c:d]]
        if b == a and d == c:
            continue
        if d == c or b == a:
            for name, x in zip(("o", "dq", "dk", "dv"), (got[0], got[2], got[3], got[4])):
                assert bool((x == 0).all()), f"{what}: {name} not zero"
            assert bool((got[1] == -float("inf")).all()), f"{what}: lse"
            continue
        if b - a == d - c:
            alone_plan = core.plan_block_causal(H, b - a, cuda, block=C_, first_block=F, window=W, sink=sink)
        else:
            alone_plan = _plan(cuda, [0, b - a], [0, d - c], sink, C_, F, W)
        alone = _fwd_bwd(alone_plan, *(t[:, :, x:y].contiguous() for t, x, y in
                                       ((q, a, b), (k, c, d), (v, c, d), (do, a, b))))
        alone = [alone[0], alone[1].view(H, -1), *alone[2:]]
        for name, x, y in zip(("o", "lse", "dq", "dk", "dv"), got, alone):
            _eq(name, x, y, what)


@pytest.mark.parametrize("W,sink", [(-1, 0), (300, 0), (1000, 130)])
def test_block_one_equals_the_causal_window(cuda, W, sink):
    """block = 1 is plan_local_varlen(causal=True, window_size=(W - 1, 0)) bit for bit when no query lies ahead of its
    keys (Lq_i <= Lk_i)."""
    from svgb200 import core

    cu_q, cu_k = [0, 700, 701, 2000, 2300], [0, 900, 901, 2500, 2800]
    q, k, v, do = _inputs(2, cu_q[-1], cu_k[-1], 128, torch.bfloat16, cuda, seed=W)
    a = _fwd_bwd(_plan(cuda, cu_q, cu_k, sink, 1, 1, W), q, k, v, do)
    t = lambda c: torch.tensor(c, dtype=torch.int32, device=cuda)  # noqa: E731
    p = core.plan_local_varlen(t(cu_q), t(cu_k), total_q=cu_q[-1], total_k=cu_k[-1], causal=True,
                               window_size=(W - 1 if W != -1 else -1, 0), sink=sink)
    b = _fwd_bwd(p, q, k, v, do)
    for name, x, y in zip(("o", "lse", "dq", "dk", "dv"), a, b):
        _eq(name, x, y, f"block=1 W={W} sink={sink}")


@pytest.mark.parametrize("args", [(0, 4680, 4680, -1), (1560, 4680, 1560, 14040), (0, 300, 77, 600)],
                         ids=["chunks", "window-sink", "first-block"])
def test_short_queries_equal_the_kvcache_plan(cuda, args):
    """One segment with Sq < Skv: the forward is plan_kvcache(block=)'s on a contiguous cache holding the same keys,
    bit for bit (the Self-Forcing step: a chunk of queries against the cache it was appended to)."""
    from svgb200 import core

    sink, C_, F, W = args
    Sq, Skv, H = 4680, 4 * 4680 - 1000, 4
    g = torch.Generator().manual_seed(C_)
    q = torch.randn(1, Sq, H, 128, generator=g).to(torch.bfloat16).to(cuda)
    kc, vc = (torch.randn(1, Skv, H, 128, generator=g).to(torch.bfloat16).to(cuda) for _ in range(2))
    kvp = core.plan_kvcache(torch.tensor([Skv], dtype=torch.int32, device=cuda), q_len=Sq, num_blocks=1, cache_len=Skv,
                            block=C_, first_block=F, window_size=(W, -1), sink=sink)
    o_kv = core.attn_fwd(q, kc, vc, kvp, out=torch.full_like(q, float("nan")))
    o = core.attn_fwd(q.transpose(1, 2), kc.transpose(1, 2), vc.transpose(1, 2), _plan(cuda, [0, Sq], [0, Skv], *args),
                      out=torch.full_like(q, float("nan")).transpose(1, 2))
    _eq("o", o.transpose(1, 2), o_kv, f"Sq={Sq} Skv={Skv} BLOCK{args}")


# --------------------------------------------------------------------------------------------
# layouts, plan read-back
# --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("view", ["bshd-B2", "unbind", "shd"])
def test_views(cuda, view):
    """Transposed [B, S, H, D] views with B = 2, one third of a packed QKV, and the packed [total, H, D] layout match
    the contiguous [B, H, S, D] call bit for bit, forward and backward, with out= buffers."""
    B = 2 if view == "bshd-B2" else 1
    H, D = 4, 128
    cu = [0, 700, 701, 2000]
    plan = _plan(cuda, cu, cu, 130, 300, 100, 900)
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


READ_BACK = [PACKED[0], PACKED[2], PACKED[4], PACKED[5], ([520], [1100], 260, 300, 100, 600),
             ([600, 300], [300, 900], 0, 1, 1, 5)]


@pytest.mark.parametrize("case", range(len(READ_BACK)))
def test_plan_read_back(cuda, case):
    """Both plans built on the GPU, read back: the parameters, and every item, chunk and kind in launch order, equal
    the host mirror's vote."""
    lq, lk, sink, C_, F, W = READ_BACK[case]
    lk = lq if lk is None else lk
    cu_q, cu_k = _cu(lq), _cu(lk)
    plan = _plan(cuda, cu_q, cu_k, sink, C_, F, W)
    Wp = max(cu_q[-1], cu_k[-1]) + C_ if W == -1 else W
    assert (plan.desc.mask_mode, plan.desc.m0, plan.desc.m1, plan.desc.m2) == (bm.MASK_BLOCK_CAUSAL, sink,
                                                                                bm.m1_of(C_, F), Wp)
    for p, transposed in ((plan, False), (plan.key_major(), True)):
        segs, got = _read(p)
        assert segs == cu_q + cu_k
        want = vb.items(cu_q, cu_k, sink, C_, F, W, transposed)
        assert got == want, f"transposed={transposed}: first difference at item " \
                            f"{next(i for i, (a, b) in enumerate(zip(got + [None], want + [None])) if a != b)}"


# --------------------------------------------------------------------------------------------
# compiled flex_attention under a document-block-causal mask
# --------------------------------------------------------------------------------------------
def test_against_compiled_flex_attention(cuda):
    """The perf tool's packed batch of Wan-480p clips (21 + 13 + 9 + 5 frames of 1 560 tokens, chunks of 3 frames, the
    first one frame, a 6-frame window and a one-frame sink) at 12 heads: forward within bf16 rounding of compiled
    flex_attention under the same mask."""
    try:
        from torch.nn.attention.flex_attention import create_block_mask, flex_attention

        flex = torch.compile(flex_attention)
    except Exception as e:  # pragma: no cover
        pytest.skip(f"flex_attention unavailable: {e}")
    from svgb200 import core

    frame = 1560
    cu = _cu([f * frame for f in (21, 13, 9, 5)])
    sink, C_, F, W = args = (frame, 3 * frame, frame, 6 * frame)
    H, S = 12, cu[-1]
    # per position: its clip and the clip's first token; per query: its block end, all in packed coordinates
    lens = torch.tensor([b - a for a, b in zip(cu, cu[1:])], device=cuda)
    clip = torch.repeat_interleave(torch.arange(len(lens), device=cuda), lens)
    start = torch.tensor(cu[:-1], device=cuda)[clip]
    ends = start + bm.block_end(torch.arange(S, device=cuda) - start, C_, F)

    def mask_mod(b, h, q_idx, kv_idx):
        e = ends[q_idx]
        near = (kv_idx < e) & (kv_idx >= e - W)
        return (clip[q_idx] == clip[kv_idx]) & ((kv_idx - start[kv_idx] < sink) | near)

    g = torch.Generator().manual_seed(1)
    q, k, v = (torch.randn(1, H, S, 128, generator=g).to(torch.bfloat16).to(cuda) for _ in range(3))
    try:
        bmask = create_block_mask(mask_mod, 1, 1, S, S, device=cuda)
        ref = flex(q, k, v, block_mask=bmask)
    except Exception as e:  # pragma: no cover
        pytest.skip(f"flex_attention compilation unavailable: {e}")
    o = core.attn_fwd(q, k, v, _plan(cuda, cu, cu, *args))
    assert _rel(o, ref) < 1e-2, f"relative difference {_rel(o, ref):.2e}"
