"""GPU tests of attention between a query sequence of length Sq and a key/value sequence of length Skv (svgb_attn_fwd_kv,
svgb_attn_bwd_kv, the rectangular variable-block planner, and the Python entries that route to them).

  key census   : the forward census (q = 0, one-hot key-identity V: o = round16(cnt / n), lse = ln n) and the backward
                 key census (oracle.bwd_census: every dQ / dK / dV value is a count of allowed pairs times a power of
                 two) on rectangular maps, into NaN-filled outputs, compared bit for bit
  equality     : with Sq == Skv the new entries give the square entries' o, lse, dQ, dK, dV bit for bit
  gradients    : fp64 autograd through oracle.attention.masked_attention_bhsd (its mask callback returns each query row's
                 full key mask, so it takes k / v of another length), at the tolerances of test_attention_bwd_gpu
"""
import ctypes as C
import itertools

import pytest
import torch

from oracle import bwd_census as obc
from oracle import census as oc
from oracle.census import rect_census

pytestmark = pytest.mark.gpu

TOL = {torch.bfloat16: 4e-2, torch.float16: 1e-2}


def sizes(total, n, gen, zeros=()):
    """n block sizes summing to total (>= 0), the blocks in `zeros` empty"""
    live = [i for i in range(n) if i not in zeros]
    cuts = torch.sort(torch.randint(0, total + 1, (len(live) - 1,), generator=gen))[0]
    part = torch.diff(torch.cat([torch.tensor([0]), cuts, torch.tensor([total])]))
    out = torch.zeros(n, dtype=torch.int32)
    out[live] = part.to(torch.int32)
    return out


def rect_map(H, Sq, Skv, gen, QC=5, KC=4):
    """per-head maps with an empty q-block row (dq = 0), an unselected k-block column (dk = dv = 0) and an empty k-block
    -> (map [H, QC, KC] bool, row sizes [H, QC], col sizes [H, KC])"""
    bm = torch.rand(H, QC, KC, generator=gen) < 0.6
    bm[:, 1, :] = False
    bm[:, :, 2] = False
    bm[:, 3, :] = True
    row = torch.stack([sizes(Sq, QC, gen) for _ in range(H)])
    col = torch.stack([sizes(Skv, KC, gen, zeros=(0,) if Skv > 1 else (0, 1, 2)) for _ in range(H)])
    return bm, row, col


def plan_kv(bm, row, col, Sq, Skv, dev):
    """svgb_attn_plan_varblock_kv called directly (core.plan_varblock takes the square planner when Sq == Skv)"""
    from svgb200 import core
    from svgb200._lib import Plan, check, lib

    H, QC, KC = bm.shape
    m, r, c = bm.to(dev).to(torch.uint8), row.to(dev).int(), col.to(dev).int()
    n = C.c_size_t()
    check(lib().svgb_attn_plan_varblock_kv_bytes(H, Sq, Skv, QC, KC, C.byref(n)), "bytes")
    ws = torch.empty(n.value, dtype=torch.uint8, device=dev)
    d = Plan()
    check(lib().svgb_attn_plan_varblock_kv(m.data_ptr(), r.data_ptr(), c.data_ptr(), H, Sq, Skv, QC, KC, ws.data_ptr(),
                                           ws.numel(), C.byref(d), torch.cuda.current_stream().cuda_stream), "plan")
    return core.AttnPlan(d, ws, (m, r, c, (m._version, r._version, c._version)))


def kv_entries(q, k, v, do, plan, layout):
    """(o, lse, dq, dk, dv) of svgb_attn_fwd_kv and svgb_attn_bwd_kv called directly with the arguments core passes
    them when Sq != Skv (core.attn_fwd / attn_bwd take the square entries when Sq == Skv)"""
    from svgb200 import core
    from svgb200._lib import check, lib

    BH, Sq, Skv, D, qs, kvs = core._kv_geometry(q, k, layout)
    scale, dt, stream = float(D) ** -0.5, core._dt(q), torch.cuda.current_stream().cuda_stream
    o, dq, dk, dv = (torch.empty_like(t) for t in (q, q, k, v))
    lse = torch.empty(BH, Sq, dtype=torch.float32, device=q.device)
    check(lib().svgb_attn_fwd_kv(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), lse.data_ptr(), dt, BH, Sq,
                                 Skv, D, *qs, *kvs, *qs, scale, C.byref(plan.desc), plan.ws.data_ptr(), stream),
          "fwd_kv")
    plan_t = plan.key_major()
    n = C.c_size_t()
    check(lib().svgb_attn_bwd_kv_bytes(BH, Sq, Skv, C.byref(n)), "bwd_kv_bytes")
    ws = torch.empty(n.value, dtype=torch.uint8, device=q.device)
    check(lib().svgb_attn_bwd_kv(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), do.data_ptr(), lse.data_ptr(),
                                 dq.data_ptr(), dk.data_ptr(), dv.data_ptr(), dt, BH, Sq, Skv, D, *qs, *kvs, scale,
                                 C.byref(plan.desc), plan.ws.data_ptr(), C.byref(plan_t.desc), plan_t.ws.data_ptr(),
                                 ws.data_ptr(), ws.numel(), stream), "bwd_kv")
    return o, lse, dq, dk, dv


# ------------------------------------------------------------------------------------------------------------------
# key census
# ------------------------------------------------------------------------------------------------------------------
SKV = [1, 127, 128, 129, 512]
SQ = [200, 1000]  # not multiples of 128; 200 < Skv = 512 and 1000 > every Skv


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("Sq", SQ)
@pytest.mark.parametrize("Skv", SKV)
def test_key_census(cuda, Skv, Sq, D, dtype):
    """o, lse, dQ, dK, dV of rectangular maps written into NaN-filled buffers equal the census closed forms bit for
    bit on every row, for both key encodings."""
    from svgb200 import core

    H = 2
    gen = torch.Generator().manual_seed(Skv * 7 + Sq + D)
    bm, row, col = rect_map(H, Sq, Skv, gen)
    plan = core.plan_varblock(bm.to(cuda), row.to(cuda), col.to(cuda), Sq, S_kv=Skv)
    assert plan.S_kv == Skv
    for enc in oc.ENCODINGS:
        tabs = [rect_census(bm[h], row[h], col[h], D) for h in range(H)]
        tabs_t = [rect_census(bm[h].T, col[h], row[h], D // 2) for h in range(H)]
        tabs_h = [rect_census(bm[h], row[h], col[h], D // 2) for h in range(H)]
        # forward: q = 0, V one-hot by the key's code over D
        q = torch.zeros(1, H, Sq, D, dtype=dtype, device=cuda)
        k = torch.randn(1, H, Skv, D, generator=gen).to(dtype).to(cuda)
        v = oc.identity_values(Skv, D, enc, H, dtype, cuda)
        o = torch.full_like(q, float("nan"))
        _, lse = core.attn_fwd(q, k, v, plan, return_lse=True, out=o)
        for h in range(H):
            cnt, n = tabs[h]
            assert torch.equal(o[0, h].cpu(), oc.expected_output(cnt[enc], n, dtype)), f"o, head {h}, enc {enc}"
            ln = torch.where(n > 0, torch.log(n.double()), torch.tensor(-float("inf"), dtype=torch.float64))
            assert torch.allclose(lse[h].cpu().double(), ln, atol=1e-5, rtol=0), f"lse, head {h}"
        # backward key census
        n_rows = torch.stack([tabs_h[h][1] for h in range(H)])
        qc, _, _, oc_, doc, lsec = obc.key_inputs(Sq, D, enc, n_rows)
        _, kc, vc, _, _, _ = obc.key_inputs(Skv, D, enc, torch.ones(H, Skv, dtype=torch.long))
        qb, ob, dob = (t.to(dtype).reshape(1, H, Sq, D).contiguous().to(cuda) for t in (qc, oc_, doc))
        kb, vb = (t.to(dtype).reshape(1, H, Skv, D).contiguous().to(cuda) for t in (kc, vc))
        out = (torch.full_like(qb, float("nan")), torch.full_like(kb, float("nan")), torch.full_like(vb, float("nan")))
        dq, dk, dv = core.attn_bwd(qb, kb, vb, ob, dob, lsec.to(cuda), plan, sm_scale=obc.KEY_SCALE, out=out)
        for h in range(H):
            cnt, cnt_t = tabs_h[h][0][enc], tabs_t[h][0][enc]
            assert int(cnt.max()) <= obc.MAX_COUNT[dtype] and int(cnt_t.max()) <= obc.MAX_COUNT[dtype]
            eq = obc.key_expected(cnt, torch.zeros_like(cnt), Sq, D, enc)[0]
            _, ek, ev = obc.key_expected(torch.zeros_like(cnt_t), cnt_t, Skv, D, enc)
            for name, got, exp in (("dq", dq, eq), ("dk", dk, ek), ("dv", dv, ev)):
                assert torch.equal(got[0, h].cpu(), exp.to(dtype)), f"{name}, head {h}, enc {enc}"


# ------------------------------------------------------------------------------------------------------------------
# Sq == Skv through the new entries
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layout", ["bhsd", "shd"])
@pytest.mark.parametrize("kind", ["varblock", "dense"])
@pytest.mark.parametrize("rect_plan", [False, True])
def test_kv_abi_entries_match_square_entries_at_equal_lengths(cuda, kind, layout, rect_plan):
    """svgb_attn_fwd_kv / svgb_attn_bwd_kv at Sq == Skv give svgb_attn_fwd / svgb_attn_bwd's o, lse, dq, dk, dv bit for
    bit, under the square planner's plan and under svgb_attn_plan_varblock_kv's plan of the same map."""
    from svgb200 import core

    H, S, D, dtype = 4, 1000, 128, torch.bfloat16
    gen = torch.Generator().manual_seed(21)
    if kind == "dense":
        bm, row = torch.ones(H, 1, 1, dtype=torch.bool), torch.full((H, 1), S, dtype=torch.int32)
        col = row
    else:
        bm, row, col = rect_map(H, S, S, gen, QC=9, KC=33)
    sq = core.plan_varblock(bm.to(cuda), row.to(cuda), col.to(cuda), S)
    plan = plan_kv(bm, row, col, S, S, cuda) if rect_plan else sq
    shape = (1, H, S, D) if layout == "bhsd" else (S, H, D)
    q, k, v, do = (torch.randn(*shape, generator=gen).to(dtype).to(cuda) for _ in range(4))
    o, lse = core.attn_fwd(q, k, v, sq, layout=layout, return_lse=True)
    g = core.attn_bwd(q, k, v, o, do, lse, sq, layout=layout)
    o2, lse2, *g2 = kv_entries(q, k, v, do, plan, layout)
    assert torch.equal(o, o2) and torch.equal(lse, lse2)
    for a, b in zip(g, g2):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------------------------
# gradients against the fp64 oracle
# ------------------------------------------------------------------------------------------------------------------
def oracle_grads(q, k, v, do, masks, sm_scale=None, dev=None):
    """fp64 autograd through masked_attention_bhsd; q, do [H, Sq, D], k, v [H, Skv, D]; masks: bool [Sq, Skv] per head
    (None: dense).  Returns (o, dq, dk, dv) in fp64 on the CPU."""
    from oracle.attention import masked_attention_bhsd

    res = []
    for h in range(q.shape[0]):
        x = [t[h:h + 1].to(dev).double().requires_grad_() for t in (q, k, v)]
        m = None if masks is None else masks[h].to(dev)
        fn = None if m is None else (lambda qi, ki, m=m: m[qi[:, 0].to(m.device)])
        o = masked_attention_bhsd(*x, fn, row_chunk=8192, sm_scale=sm_scale, dtype=torch.float64)
        o.backward(do[h:h + 1].double().cpu())
        res.append([o.detach()[0]] + [t.grad[0].cpu() for t in x])
    return [torch.stack([r[i] for r in res]) for i in range(4)]


def check(got, ref, dtype, names=("o", "dq", "dk", "dv")):
    for name, g, r in zip(names, got, ref):
        g = g.double().cpu()
        assert torch.isfinite(g).all(), f"{name}: non-finite values"
        err = float((g - r).abs().max())
        assert err <= TOL[dtype] * float(r.abs().max()) + 1e-6, f"{name}: max error {err} vs max |ref| {float(r.abs().max())}"


def element_masks(bm, row, col):
    from oracle.attention import block_mask_to_element_mask

    return [block_mask_to_element_mask(bm[h], row[h], col[h]) for h in range(bm.shape[0])]


def lay(t, layout, B):
    """[H, S, D] -> [B, H / B, S, D] or [S, H, D], contiguous"""
    H, S, D = t.shape
    return t.view(B, H // B, S, D).contiguous() if layout == "bhsd" else t.transpose(0, 1).contiguous()


def unlay(t, layout):
    return t.reshape(-1, *t.shape[-2:]) if layout == "bhsd" else t.transpose(0, 1)


# (Sq, Skv, map): "dense" one block per side; "vb" a rectangular variable-block map with empty blocks
CASES = {"short_kv": (1000, 77, "dense"), "long_kv": (300, 1500, "dense"), "vb_q_longer": (1000, 600, "vb"),
         "vb_kv_longer": (333, 1200, "vb"), "vb/scale": (700, 300, "vb")}


@pytest.mark.parametrize("layout", ["bhsd", "shd"])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("case", list(CASES))
def test_gradients_vs_oracle(cuda, case, dtype, D, layout):
    """o, dQ, dK, dV of core.attention with k, v of another length (batch 2, two heads each, each head its own map)
    vs fp64 autograd."""
    from svgb200 import core

    Sq, Skv, kind = CASES[case]
    sm_scale = 0.3 if case.endswith("/scale") else None
    B, H = 2, 4
    gen = torch.Generator().manual_seed(list(CASES).index(case) * 11 + D)
    if kind == "dense":
        bm = torch.ones(H, 1, 1, dtype=torch.bool)
        row, col = torch.full((H, 1), Sq, dtype=torch.int32), torch.full((H, 1), Skv, dtype=torch.int32)
        masks = None
    else:
        bm, row, col = rect_map(H, Sq, Skv, gen, QC=7, KC=11)
        masks = element_masks(bm, row, col)
    plan = core.plan_varblock(bm.to(cuda), row.to(cuda), col.to(cuda), Sq, S_kv=Skv)
    q, do = (torch.randn(H, Sq, D, generator=gen).to(dtype) for _ in range(2))
    k, v = (torch.randn(H, Skv, D, generator=gen).to(dtype) for _ in range(2))
    x = [lay(t, layout, B).to(cuda).requires_grad_() for t in (q, k, v)]
    o = core.attention(*x, plan, layout=layout, sm_scale=sm_scale)
    o.backward(lay(do, layout, B).to(cuda))
    got = [unlay(o.detach(), layout)] + [unlay(t.grad, layout) for t in x]
    check(got, oracle_grads(q, k, v, do, masks, sm_scale=sm_scale, dev=cuda), dtype)


@pytest.mark.parametrize("Skv", [512, 257], ids=["wan_text", "wan_i2v"])
def test_wan_720p_cross_attention(cuda, Skv):
    """Full size: Wan 720p text cross-attention (75 600 queries x 512 keys) and the I2V image branch (x 257), 40 heads,
    D = 128, bf16, dense; forward and gradients vs fp64 autograd on the GPU."""
    from svgb200 import core

    H, Sq, D, dtype = 40, 75600, 128, torch.bfloat16
    gen = torch.Generator(device=cuda).manual_seed(Skv)
    q, do = (torch.randn(H, Sq, D, device=cuda, generator=gen).to(dtype) for _ in range(2))
    k, v = (torch.randn(H, Skv, D, device=cuda, generator=gen).to(dtype) for _ in range(2))
    one = torch.ones(H, 1, 1, dtype=torch.bool, device=cuda)
    plan = core.plan_varblock(one, torch.full((H, 1), Sq, device=cuda), torch.full((H, 1), Skv, device=cuda), Sq,
                              S_kv=Skv)
    x = [t[None].clone().requires_grad_() for t in (q, k, v)]
    o = core.attention(*x, plan)
    o.backward(do[None])
    got = [o.detach()[0]] + [t.grad[0] for t in x]
    for h0 in range(0, H, 8):  # the fp64 reference in groups of heads (bounded memory)
        ref = oracle_grads(q[h0:h0 + 8], k[h0:h0 + 8], v[h0:h0 + 8], do[h0:h0 + 8], None, dev=cuda)
        check([g[h0:h0 + 8] for g in got], ref, dtype)


def test_chunk_of_frames_against_context(cuda):
    """A chunk of 3 frames attending to 21 frames (the chunk is frames 18..20 of the key sequence) under a rectangular
    varblock map: each query frame sees the first frame and the frames up to its own within a window of 6."""
    from svgb200 import core

    P, Fq, Fk, H, D, dtype = 400, 3, 21, 2, 128, torch.bfloat16
    Sq, Skv = Fq * P, Fk * P
    bm = torch.zeros(H, Fq, Fk, dtype=torch.bool)
    for i in range(Fq):
        f = Fk - Fq + i
        bm[:, i, 0] = True
        bm[:, i, max(0, f - 5):f + 1] = True
    row, col = torch.full((H, Fq), P, dtype=torch.int32), torch.full((H, Fk), P, dtype=torch.int32)
    plan = core.plan_varblock(bm.to(cuda), row.to(cuda), col.to(cuda), Sq, S_kv=Skv)
    gen = torch.Generator().manual_seed(4)
    q, do = (torch.randn(H, Sq, D, generator=gen).to(dtype) for _ in range(2))
    k, v = (torch.randn(H, Skv, D, generator=gen).to(dtype) for _ in range(2))
    x = [t[None].to(cuda).requires_grad_() for t in (q, k, v)]
    o = core.attention(*x, plan)
    o.backward(do[None].to(cuda))
    got = [o.detach()[0]] + [t.grad[0] for t in x]
    check(got, oracle_grads(q, k, v, do, element_masks(bm, row, col), dev=cuda), dtype)


# ------------------------------------------------------------------------------------------------------------------
# determinism, model-level entries, launch counts
# ------------------------------------------------------------------------------------------------------------------
def test_deterministic(cuda):
    """Two backward runs on a rectangular plan give bit-identical gradients (no atomics)."""
    from svgb200 import core

    H, Sq, Skv, D, dtype = 4, 5000, 1300, 128, torch.bfloat16
    gen = torch.Generator().manual_seed(8)
    bm, row, col = rect_map(H, Sq, Skv, gen, QC=17, KC=9)
    plan = core.plan_varblock(bm.to(cuda), row.to(cuda), col.to(cuda), Sq, S_kv=Skv)
    q, do = (torch.randn(1, H, Sq, D, generator=gen).to(dtype).to(cuda) for _ in range(2))
    k, v = (torch.randn(1, H, Skv, D, generator=gen).to(dtype).to(cuda) for _ in range(2))
    o, lse = core.attn_fwd(q, k, v, plan, return_lse=True)
    a = core.attn_bwd(q, k, v, o, do, lse, plan)
    b = core.attn_bwd(q, k, v, o, do, lse, plan)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


def seg_masks(segs, kv_segs, H):
    m = torch.zeros(sum(segs), sum(kv_segs), dtype=torch.bool)
    r = c = 0
    for a, b in zip(segs, kv_segs):
        m[r:r + a, c:c + b] = True
        r, c = r + a, c + b
    return [m] * H


def test_dense_attention_kv_segments(cuda):
    """dense_attention with kv_seg_lens (query segment i attends key segment i, an empty key segment included) and
    with a whole shorter key sequence, under grad, vs the oracle."""
    from svgb200.models import common

    H, D, dtype = 2, 128, torch.bfloat16
    gen = torch.Generator().manual_seed(9)
    for segs, kv_segs in (([700, 300, 24], [100, 0, 412]), ([1024], [257])):
        Sq, Skv = sum(segs), sum(kv_segs)
        q, do = (torch.randn(H, Sq, D, generator=gen).to(dtype) for _ in range(2))
        k, v = (torch.randn(H, Skv, D, generator=gen).to(dtype) for _ in range(2))
        x = [t[None].to(cuda).requires_grad_() for t in (q, k, v)]
        o = common.dense_attention(*x, segs, kv_segs) if len(segs) > 1 else common.dense_attention(*x)
        o.backward(do[None].to(cuda))
        got = [o.detach()[0]] + [t.grad[0] for t in x]
        check(got, oracle_grads(q, k, v, do, seg_masks(segs, kv_segs, H), dev=cuda), dtype)


@pytest.mark.parametrize("fn", ["flash_attn_varlen_func", "flashinfer_varlen_func"])
def test_varlen_mirrors_use_key_segments(cuda, fn):
    """The varlen mirrors attend the cu_seqlens_kv segments when they differ from cu_seqlens_q (forward and gradients
    vs the oracle); with equal boundaries they give today's result bit for bit."""
    from svgb200 import core, patch

    H, D, dtype = 2, 128, torch.bfloat16
    segs, kv_segs = [600, 424], [256, 300]
    Sq, Skv = sum(segs), sum(kv_segs)
    gen = torch.Generator().manual_seed(10)
    q, do = (torch.randn(H, Sq, D, generator=gen).to(dtype) for _ in range(2))
    k, v = (torch.randn(H, Skv, D, generator=gen).to(dtype) for _ in range(2))
    cu = lambda s: torch.tensor([0, *itertools.accumulate(s)], dtype=torch.int32, device=cuda)  # noqa: E731
    f = getattr(patch, fn)
    to = (lambda t: t.transpose(0, 1).contiguous()) if fn == "flash_attn_varlen_func" else (lambda t: t[None])
    back = (lambda t: t.transpose(0, 1)) if fn == "flash_attn_varlen_func" else (lambda t: t[0])
    x = [to(t.to(cuda)).requires_grad_() for t in (q, k, v)]
    o = f(*x, cu(segs), cu(kv_segs), max(segs), max(kv_segs))
    o.backward(to(do.to(cuda)))
    got = [back(o.detach())] + [back(t.grad) for t in x]
    check(got, oracle_grads(q, k, v, do, seg_masks(segs, kv_segs, H), dev=cuda), dtype)
    # equal boundaries: today's plan and launch (the query segments for both sides)
    kk, vv = (to(torch.randn(H, Sq, D, generator=gen).to(dtype).to(cuda)) for _ in range(2))
    qq = x[0].detach()
    n0 = core.launch_count
    y = f(qq, kk, vv, cu(segs), cu(segs), max(segs), max(segs))
    assert core.launch_count - n0 == 2
    # the call both mirrors made before key segments were read: the query segments' square plan on both sides
    n = len(segs)
    sz = torch.tensor(segs, dtype=torch.int32, device=cuda).expand(H, n).contiguous()
    eye = torch.eye(n, dtype=torch.bool, device=cuda).expand(H, n, n).contiguous()
    ref = core.attn_fwd(qq, kk, vv, core.plan_varblock(eye, sz, sz, Sq),
                        layout="shd" if fn == "flash_attn_varlen_func" else "bhsd")
    assert torch.equal(y, ref)


def test_equal_length_calls_keep_their_launches(cuda):
    """Equal-length calls through attn_fwd / attn_bwd / attention / dense_attention issue the square entries' launches
    (plan 1, forward 1, backward 3, key-major plan 1)."""
    from svgb200 import core
    from svgb200.models import common

    H, S, D, dtype = 2, 640, 128, torch.bfloat16
    q, k, v, do = (torch.randn(1, H, S, D, device=cuda).to(dtype) for _ in range(4))
    one = torch.ones(H, 1, 1, dtype=torch.bool, device=cuda)
    sz = torch.full((H, 1), S, device=cuda)
    n0 = core.launch_count
    plan = core.plan_varblock(one, sz, sz, S, S_kv=S)
    assert plan.desc.m0 == 0 and core.launch_count - n0 == 1
    n0 = core.launch_count
    o, lse = core.attn_fwd(q, k, v, plan, return_lse=True)
    core.attn_bwd(q, k, v, o, do, lse, plan)
    assert core.launch_count - n0 == 1 + 1 + 3
    n0 = core.launch_count
    common.dense_attention(q, k, v)
    assert core.launch_count - n0 == 2
    x = [t.clone().requires_grad_() for t in (q, k, v)]
    n0 = core.launch_count
    core.attention(*x, plan).backward(do)
    assert core.launch_count - n0 == 1 + 3


def test_rectangular_python_errors(cuda):
    """Gather plans and row vectors need Sq == Skv; k must match q outside the sequence length; a square plan does not
    run k, v of another length."""
    from svgb200 import core

    H = 2
    one = torch.ones(H, 1, 1, dtype=torch.bool, device=cuda)
    sq, skv = torch.full((H, 1), 300, device=cuda), torch.full((H, 1), 100, device=cuda)
    with pytest.raises(core.SvgbError, match="gather"):
        core.plan_varblock(one, sq, skv, 300, gather=True, S_kv=100)
    plan = core.plan_varblock(one, sq, skv, 300, S_kv=100)
    q = torch.zeros(1, H, 300, 64, dtype=torch.bfloat16, device=cuda)
    k = torch.zeros(1, H, 100, 64, dtype=torch.bfloat16, device=cuda)
    with pytest.raises(core.SvgbError, match="row vectors"):
        core.attn_fwd(q, k, k, plan, o_rows=torch.zeros(H, 300, dtype=torch.int32, device=cuda))
    with pytest.raises(core.SvgbError, match="sequence length only"):
        core.attn_fwd(q, k[:, :, :, :32].contiguous(), k[:, :, :, :32].contiguous(), plan)
    with pytest.raises(core.SvgbError, match="plan was built"):
        core.attn_fwd(q, k, k, core.plan_varblock(one, sq, sq, 300))
    with pytest.raises(core.SvgbError, match="plan was built"):
        core.attn_fwd(q, q, q, plan)
