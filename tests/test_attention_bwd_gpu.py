"""GPU tests of the attention backward (svgb_attn_bwd, core.attn_bwd, core.attention) against the fp64 oracle.

Gradients are compared with torch autograd through oracle.attention.masked_attention_bhsd in float64 on the same
(exactly representable) 16-bit inputs.  Tolerance: the kernels round P and dS to the input type before the tensor-core
products (as the forward rounds P before P V) and round each gradient once more at the store; each rounding is 2^-9
(bf16) / 2^-12 (fp16) relative, and sums of such terms over a row stay within a small multiple of that relative to the
largest gradient entry.  So max |g - ref| <= TOL * max |ref| per gradient, TOL = 4e-2 (bf16) / 1e-2 (fp16): a wrong key
set, a missing scale or a wrong delta moves the error to O(1) of that bound.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

TOL = {torch.bfloat16: 4e-2, torch.float16: 1e-2}
MASK_NONE, MASK_HY, MASK_WAN, MASK_COG = 0, 1, 2, 3
# small band shapes (S not a multiple of 128): (mode, m0, m1, m2, S)
#   HY : 3 frames x 100 tokens + 20 prompt + 24 padding rows; WAN: 3 x 100, sink = first frame; COG: 20 text rows first
BANDS = {
    "hy": (MASK_HY, 300, 320, 150, 344),
    "wan": (MASK_WAN, 100, 0, 130, 300),
    "cog": (MASK_COG, 20, 20, 140, 320),
    "none": (MASK_NONE, 0, 0, 0, 200),
}


def random_partition(seq_len, num_blocks, gen):
    cuts = torch.randperm(seq_len - 1, generator=gen)[: num_blocks - 1] + 1
    cuts, _ = torch.sort(cuts)
    return torch.diff(torch.cat([torch.tensor([0]), cuts, torch.tensor([seq_len])])).to(torch.int32)


def with_empty_blocks(sz):
    """merge block 2 into block 1 and block 5 into block 4: two empty clusters per head"""
    sz = sz.clone()
    for a, b in ((1, 2), (4, 5)):
        sz[:, a] += sz[:, b]
        sz[:, b] = 0
    return sz


def to_layout(x, layout):
    """[H, S, D] -> the kernel's layout ([1, H, S, D] or [S, H, D]), contiguous"""
    return x[None].contiguous() if layout == "bhsd" else x.transpose(0, 1).contiguous()


def from_layout(x, layout):
    return x[0] if layout == "bhsd" else x.transpose(0, 1)


def oracle_grads(q, k, v, do, masks, sm_scale=None):
    """fp64 autograd through masked_attention_bhsd; q,k,v,do [H,S,D]; masks: list of bool [S,S] per head"""
    from oracle.attention import masked_attention_bhsd

    out = []
    for h, m in enumerate(masks):
        x = [t[h:h + 1].double().requires_grad_() for t in (q, k, v)]
        o = masked_attention_bhsd(*x, lambda qi, ki: m[qi[:, 0]][:, ki[0]], sm_scale=sm_scale, dtype=torch.float64)
        o.backward(do[h:h + 1].double())
        out.append([t.grad[0] for t in x])
    return [torch.stack([g[i] for g in out]) for i in range(3)]


def band_mask(mode, m0, m1, m2, S):
    from oracle.attention import generic_mask_fn

    return generic_mask_fn(mode, m0, m1, m2)(torch.arange(S).view(-1, 1), torch.arange(S).view(1, -1))


def varblock_case(kind, H, S, gen):
    """-> (map [H,QC,KC], row sizes, col sizes, element masks) for the variable-block cases"""
    from oracle.attention import block_mask_to_element_mask

    if kind == "dense":
        bm, row = torch.ones(H, 1, 1, dtype=torch.bool), torch.full((H, 1), S, dtype=torch.int32)
        col = row
    elif kind == "varlen":  # HunyuanVideo's padded-prompt split: two segments that attend inside themselves
        seg = torch.tensor([S - 77, 77], dtype=torch.int32)
        bm, row = torch.eye(2, dtype=torch.bool).expand(H, 2, 2).contiguous(), seg.expand(H, 2).contiguous()
        col = row
    else:
        density = float(kind[2:])
        row = with_empty_blocks(torch.stack([random_partition(S, 9, gen) for _ in range(H)]))
        col = with_empty_blocks(torch.stack([random_partition(S, 33, gen) for _ in range(H)]))
        bm = torch.rand(H, 9, 33, generator=gen) > density
    masks = [block_mask_to_element_mask(bm[h], row[h], col[h]) for h in range(H)]
    return bm, row, col, masks


def make_plan(kind, H, S, cuda, gen):
    from svgb200 import core

    if kind in BANDS:
        mode, m0, m1, m2, _ = BANDS[kind]
        return core.plan_band(mode, m0, m1, m2, H, S, cuda), [band_mask(mode, m0, m1, m2, S)] * H
    bm, row, col, masks = varblock_case(kind, H, S, gen)
    return core.plan_varblock(bm.to(cuda), row.to(cuda), col.to(cuda), S), masks


def inputs(H, S, D, dtype, gen):
    return [torch.randn(H, S, D, generator=gen).to(dtype) for _ in range(4)]


def check_grads(got, ref, dtype):
    for name, g, r in zip(("dq", "dk", "dv"), got, ref):
        g = g.double().cpu()
        assert torch.isfinite(g).all(), f"{name}: non-finite values"
        err = float((g - r).abs().max())
        assert err <= TOL[dtype] * float(r.abs().max()) + 1e-6, f"{name}: max error {err} vs max |ref| {float(r.abs().max())}"


# "<kind>/B2": batch 2 (four heads, each with its own variable-block map; 'shd' holds them as four heads);
# "<kind>/scale": an explicit sm_scale through core.attention, which the backward must take from the forward
CASES = ["hy", "wan", "cog", "vb0.2", "vb0.7", "vb0.9", "dense", "varlen", "wan/B2", "vb0.5/B2", "cog/scale",
         "vb0.7/scale"]
SCALE = 0.3


@pytest.mark.parametrize("layout", ["bhsd", "shd"])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("kind", CASES)
def test_gradients_vs_oracle(cuda, kind, dtype, D, layout):
    """dQ, dK, dV of core.attention under band and variable-block plans vs fp64 autograd of the masked softmax."""
    from svgb200 import core

    base, _, extra = kind.partition("/")
    B = 2 if extra == "B2" else 1
    sm_scale = SCALE if extra == "scale" else None
    H = 2 * B
    gen = torch.Generator().manual_seed(CASES.index(kind) * 7 + D)
    S = BANDS[base][4] if base in BANDS else 1000
    plan, masks = make_plan(base, H, S, cuda, gen)
    q, k, v, do = inputs(H, S, D, dtype, gen)

    def lay(t):
        return to_layout(t, layout) if layout == "shd" else t.view(B, H // B, S, D).contiguous()

    x = [lay(t).to(cuda).requires_grad_() for t in (q, k, v)]
    o = core.attention(*x, plan, layout=layout, sm_scale=sm_scale)
    o.backward(lay(do).to(cuda))
    got = [from_layout(t.grad, layout) if layout == "shd" else t.grad.reshape(H, S, D) for t in x]
    check_grads(got, oracle_grads(q, k, v, do, masks, sm_scale=sm_scale), dtype)


def test_edge_rows_and_keys(cuda):
    """A q-block that selects nothing gets dQ == 0 exactly; a k-block that no q-block selects gets dK == dV == 0;
    no NaN or Inf anywhere."""
    from svgb200 import core

    H, S, D, dtype = 2, 1000, 128, torch.bfloat16
    gen = torch.Generator().manual_seed(3)
    row = torch.stack([random_partition(S, 9, gen) for _ in range(H)])
    col = torch.stack([random_partition(S, 33, gen) for _ in range(H)])
    bm = torch.rand(H, 9, 33, generator=gen) > 0.5
    bm[:, 0, :] = False   # q-block 0 sees no key
    bm[:, :, 5] = False   # k-block 5 is seen by no query
    plan = core.plan_varblock(bm.to(cuda), row.to(cuda), col.to(cuda), S)
    q, k, v, do = (t[None].to(cuda) for t in inputs(H, S, D, dtype, gen))
    o, lse = core.attn_fwd(q, k, v, plan, return_lse=True)
    dq, dk, dv = (t[0].cpu() for t in core.attn_bwd(q, k, v, o, do, lse, plan))
    for h in range(H):
        r0 = int(row[h, 0])
        c0, c1 = int(col[h, :5].sum()), int(col[h, :6].sum())
        assert torch.equal(dq[h, :r0], torch.zeros_like(dq[h, :r0]))
        assert torch.equal(dk[h, c0:c1], torch.zeros_like(dk[h, c0:c1]))
        assert torch.equal(dv[h, c0:c1], torch.zeros_like(dv[h, c0:c1]))
    for t in (dq, dk, dv):
        assert torch.isfinite(t.float()).all()


def test_deterministic(cuda):
    """Two backward runs give bit-identical gradients (no atomics)."""
    from svgb200 import core

    H, S, D, dtype = 4, 4096 + 200, 128, torch.bfloat16
    gen = torch.Generator().manual_seed(5)
    plan = core.plan_band(MASK_HY, 3600, 3700, 1024, H, S, cuda)
    q, k, v, do = (t[None].to(cuda) for t in inputs(H, S, D, dtype, gen))
    o, lse = core.attn_fwd(q, k, v, plan, return_lse=True)
    a = core.attn_bwd(q, k, v, o, do, lse, plan)
    b = core.attn_bwd(q, k, v, o, do, lse, plan)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


def test_autograd_wiring(cuda):
    """Through the patched flex_attention and dense_attention, gradients reach Q, K and V and match the oracle; the
    same calls without requires_grad equal core.attn_fwd bit for bit."""
    from svgb200 import core, patch
    from svgb200.models import common
    from svgb200.models import hyvideo as hy

    H, F, P, ctx, D, dtype = 2, 3, 128, 64, 128, torch.bfloat16
    S = ctx + F * P
    gen = torch.Generator().manual_seed(11)
    q, k, v, do = inputs(H, S, D, dtype, gen)
    bmask = hy.prepare_flexattention(1, H, D, dtype, cuda, ctx, 20, F, P, diag_width=1.3, multiplier=1.3)
    m = band_mask(bmask.mode, bmask.m0, bmask.m1, bmask.m2, S)
    for fn, masks, plan in (
            (lambda a, b, c: patch.flex_attention(a, b, c, block_mask=bmask), [m] * H, bmask.plan),
            (lambda a, b, c: common.dense_attention(a, b, c, [S - 40, 40]), None, None)):
        x = [t[None].to(cuda).requires_grad_() for t in (q, k, v)]
        o = fn(*x)
        assert o.grad_fn is not None
        o.backward(do[None].to(cuda))
        if masks is None:
            seg = torch.zeros(S, S, dtype=torch.bool)
            seg[: S - 40, : S - 40] = True
            seg[S - 40:, S - 40:] = True
            masks = [seg] * H
        check_grads([t.grad[0] for t in x], oracle_grads(q, k, v, do, masks), dtype)
        with torch.no_grad():
            y = fn(*[t.detach() for t in x])
        if plan is not None:
            assert torch.equal(y, core.attn_fwd(*[t.detach() for t in x], plan))
    # dense_attention without grad: the plain forward
    qd, kd, vd = (t[None].to(cuda) for t in (q, k, v))
    y = common.dense_attention(qd, kd, vd)
    sz = torch.full((H, 1), S, dtype=torch.int32, device=cuda)
    ref = core.attn_fwd(qd, kd, vd, core.plan_varblock(torch.ones(H, 1, 1, dtype=torch.bool, device=cuda), sz, sz, S))
    assert torch.equal(y, ref)


@pytest.mark.parametrize("entry", ["sparse_flex_attention", "dense_attention", "dynamic_block_sparse_fwd_flashinfer",
                                   "flash_attn_varlen_func", "sparse_attn_forward", "wan_sparse_attn_forward",
                                   "flashinfer_sparse_attn_forward"])
def test_entries_without_grad_make_one_forward_launch(cuda, entry):
    """The 16-bit attention entries run core.attention; on inputs that do not require grad that is core.attn_fwd:
    the entry's own planner launch (none for a prebuilt BandMask plan) and one attention launch, with attn_fwd's bits
    under the same plan."""
    from svgb200 import core, kmeans_utils, ops, patch
    from svgb200.models import common
    from svgb200.models import hyvideo as hy

    H, D, dtype = 2, 128, torch.bfloat16
    gen = torch.Generator().manual_seed(17)
    S, layout, planned = 600, "bhsd", 1
    if entry == "sparse_flex_attention":
        ctx, F, P = 64, 3, 128
        S, planned = ctx + F * P, 0
        bmask = hy.prepare_flexattention(1, H, D, dtype, cuda, ctx, 20, F, P, diag_width=1.3, multiplier=1.3)
        call = lambda a, b, c: common.sparse_flex_attention(a, b, c, bmask)  # noqa: E731
        plan = lambda: bmask.plan  # noqa: E731
    elif entry in ("dense_attention", "flash_attn_varlen_func"):
        segs = [S - 77, 77]
        cu = torch.tensor([0, S - 77, S], dtype=torch.int32, device=cuda)
        if entry == "dense_attention":
            call = lambda a, b, c: common.dense_attention(a, b, c, segs)  # noqa: E731
        else:
            layout = "shd"
            call = lambda a, b, c: patch.flash_attn_varlen_func(a, b, c, cu, cu, S - 77, S - 77)  # noqa: E731

        def plan():
            bm, row, _, _ = varblock_case("varlen", H, S, gen)
            return core.plan_varblock(bm.to(cuda), row.to(cuda), row.to(cuda), S)
    elif entry == "dynamic_block_sparse_fwd_flashinfer":
        maps = [t[None] for t in varblock_case("vb0.5", H, S, gen)[:3]]  # [B, H, ...] on the host, as the reference
        call = lambda a, b, c: kmeans_utils.dynamic_block_sparse_fwd_flashinfer(a, b, c, *maps)  # noqa: E731
        plan = lambda: kmeans_utils._flashinfer_plan(q, *maps)  # noqa: E731
    elif entry == "sparse_attn_forward":  # text first, [S, H, D]; each mask object plans once (ops.bsr_to_plan cache)
        F, P, T = 6, 160, 16
        S, layout = F * P + T, "shd"
        meta = ops.FAMetadata(T, F, P, ops._gen_temporal_mask(F, P, 1.8, device=cuda), None)
        call = lambda a, b, c: ops.sparse_attn_forward(a, b, c, meta, "temporal")  # noqa: E731
        plan = lambda: ops.bsr_to_plan(*meta.temporal_mask_metadata, F * P, T, cuda)  # noqa: E731
    else:
        F, P = 5, 240
        S = F * P
        md = ops.gen_temporal_mask(F, P, 1.3, device=cuda)
        if entry == "wan_sparse_attn_forward":  # [S, H, D]
            layout = "shd"
            call = lambda a, b, c: ops.wan_sparse_attn_forward(a, b, c, ops.WanFAMetadata(F, P, md))  # noqa: E731
        else:
            call = lambda a, b, c: ops.flashinfer_sparse_attn_forward(a, b, c, md)  # noqa: E731
        plan = lambda: ops.bsr_to_plan(*md, S, 0, cuda)  # noqa: E731
    q, k, v = (to_layout(t, layout).to(cuda) for t in inputs(H, S, D, dtype, gen)[:3])
    n0 = core.launch_count
    y = call(q, k, v)
    assert core.launch_count - n0 == planned + 1
    assert torch.equal(y, core.attn_fwd(q, k, v, plan(), layout=layout))


def test_no_backward_paths_raise(cuda):
    """FP8 attention and gather plans have no backward: under grad they raise SvgbError instead of returning a result
    detached from the graph."""
    from svgb200 import core
    from svgb200.models import common

    H, S, D = 2, 512, 128
    x = [torch.randn(1, H, S, D, device=cuda).to(torch.bfloat16).requires_grad_() for _ in range(3)]
    bmask = common.BandMask(core.plan_band(MASK_HY, 400, 450, 128, H, S, cuda), MASK_HY, 400, 450, 128, S)
    with pytest.raises(core.SvgbError, match="fp8"):
        common.sparse_flex_attention_fp8(*x, bmask)
    with pytest.raises(core.SvgbError, match="fp8"):
        common.fp8_attention(*x, bmask.plan)
    sz = torch.full((H, 2), S // 2, dtype=torch.int32, device=cuda)
    gplan = core.plan_varblock(torch.ones(H, 2, 2, dtype=torch.bool, device=cuda), sz, sz, S, gather=True)
    with pytest.raises(core.SvgbError, match="gather"):
        core.attention(*x, gplan)
    prof = core.plan_band(core.MASK_PROF_HY_S, 3, 128, 2, H, S, cuda)
    with pytest.raises(core.SvgbError, match="profiling"):
        core.attention(*x, prof)


def test_hunyuan_720p_band_sampled_rows(cuda):
    """HunyuanVideo 720p band plan (S = 119056, W = 19072), one head, bf16, D = 128: dQ on a seeded sample of query
    rows and dK, dV on a seeded sample of keys vs the fp64 oracle restricted to those rows (the full-size softmax
    statistics computed in fp64 on the GPU in row chunks)."""
    from oracle.attention import generic_mask_fn
    from svgb200 import core

    ctx, F, P, plen, W = 256, 33, 3600, 71, 19072
    V = F * P
    S, D, dtype = ctx + V, 128, torch.bfloat16
    mode, m0, m1, m2 = MASK_HY, V, V + plen, W
    gen = torch.Generator(device=cuda).manual_seed(0)
    q, k, v, do = (torch.randn(1, 1, S, D, device=cuda, generator=gen).to(dtype) for _ in range(4))
    plan = core.plan_band(mode, m0, m1, m2, 1, S, cuda)
    o, lse = core.attn_fwd(q, k, v, plan, return_lse=True)
    dq, dk, dv = (t[0, 0] for t in core.attn_bwd(q, k, v, o, do, lse, plan))
    g = torch.Generator().manual_seed(1)
    rows = torch.cat([torch.randint(0, S, (48,), generator=g), torch.tensor([0, V - 1, V, V + plen, S - 1])]).to(cuda)
    keys = torch.cat([torch.randint(0, S, (48,), generator=g), torch.tensor([0, V - 1, V, V + plen, S - 1])]).to(cuda)
    mod = generic_mask_fn(mode, m0, m1, m2)
    scale = D ** -0.5
    qf, kf, vf, dof = (t[0, 0].double() for t in (q, k, v, do))
    kidx = torch.arange(S, device=cuda).view(1, -1)
    lse_ref = torch.empty(S, dtype=torch.float64, device=cuda)
    delta = torch.empty(S, dtype=torch.float64, device=cuda)
    for r0 in range(0, S, 2048):
        r1 = min(S, r0 + 2048)
        s = (qf[r0:r1] @ kf.T) * scale
        s.masked_fill_(~mod(torch.arange(r0, r1, device=cuda).view(-1, 1), kidx), float("-inf"))
        lse_ref[r0:r1] = torch.logsumexp(s, -1)
        p = torch.exp(s - lse_ref[r0:r1, None])
        delta[r0:r1] = ((p @ vf) * dof[r0:r1]).sum(-1)
        del s, p
    # dQ rows
    s = (qf[rows] @ kf.T) * scale
    allowed = mod(rows.view(-1, 1), kidx)
    p = torch.exp(s - lse_ref[rows, None]).masked_fill(~allowed, 0)
    dq_ref = ((p * (dof[rows] @ vf.T - delta[rows, None])) @ kf) * scale
    # dK, dV keys
    st = (qf @ kf[keys].T) * scale
    allowed = mod(torch.arange(S, device=cuda).view(-1, 1), keys.view(1, -1))
    pt = torch.exp(st - lse_ref[:, None]).masked_fill(~allowed, 0)
    dv_ref = pt.T @ dof
    dk_ref = ((pt * (dof @ vf[keys].T - delta[:, None])).T @ qf) * scale
    check_grads([dq[rows], dk[keys], dv[keys]], [t.cpu() for t in (dq_ref, dk_ref, dv_ref)], dtype)


@pytest.mark.parametrize("op", ["sparse_attn_forward", "wan_sparse_attn_forward", "flashinfer_sparse_attn_forward"])
def test_bsr_ops_gradients(cuda, op):
    """The BSR ops API runs one plan shared by every head (items_stride = 0); its key-major plan is shared the same way,
    and the gradients through each op match the oracle under the block -> element mask."""
    from oracle import attention as oa
    from svgb200 import ops

    H, D, dtype = 2, 128, torch.bfloat16
    gen = torch.Generator().manual_seed(13)
    if op == "sparse_attn_forward":  # text first, [S, H, D]
        F, P, T = 6, 160, 16
        md = ops._gen_temporal_mask(F, P, 1.8, device=cuda)
        ref_bm, bs = oa.ref_gen_temporal_mask(F, P, 1.8)
        mask, S, layout = oa.gen_mask_block2element(ref_bm, bs, T), F * P + T, "shd"
        meta = ops.FAMetadata(T, F, P, md, None)
        fn = lambda a, b, c: ops.sparse_attn_forward(a, b, c, meta, "temporal")  # noqa: E731
    else:
        F, P = 5, 240
        md = ops.gen_temporal_mask(F, P, 1.3, device=cuda)
        ref_bm, bs = oa.ref_gen_temporal_mask_wan(F, P, 1.3, first_frame=False)
        mask, S = oa.gen_mask_block2element(ref_bm, bs, 0), F * P
        if op == "wan_sparse_attn_forward":  # [S, H, D]
            layout = "shd"
            fn = lambda a, b, c: ops.wan_sparse_attn_forward(a, b, c, ops.WanFAMetadata(F, P, md))  # noqa: E731
        else:  # [cfg, H, S, D]
            layout = "bhsd"
            fn = lambda a, b, c: ops.flashinfer_sparse_attn_forward(a, b, c, md)  # noqa: E731
    q, k, v, do = inputs(H, S, D, dtype, gen)
    x = [to_layout(t, layout).to(cuda).requires_grad_() for t in (q, k, v)]
    o = fn(*x)
    assert o.grad_fn is not None
    o.backward(to_layout(do, layout).to(cuda))
    check_grads([from_layout(t.grad, layout) for t in x], oracle_grads(q, k, v, do, [mask] * H), dtype)
