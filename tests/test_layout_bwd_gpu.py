"""GPU tests of the layout operators under autograd (core._HeadPlacement, core._Permute) and of what they make
differentiable: the SVG1 cores and the reference's SVG1 / SVG2 call sequences.

A placement or a permutation only moves rows, so its gradient is exact: the tests compare it bit for bit with
oracle.layout applied in the opposite direction to the upstream gradient.  Through the attention, dQ, dK and dV are
compared bit for bit with the same computation composed from the no-grad API, and within the attention backward's
tolerance (test_attention_bwd_gpu.check_grads) with fp64 autograd through oracle.layout and the oracle attention.
"""
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE / "golden"))
import ref_import as R  # noqa: E402
from test_attention_bwd_gpu import check_grads, oracle_grads  # noqa: E402

pytestmark = pytest.mark.gpu

DTYPES = [torch.bfloat16, torch.float16]
# (ctx, F, P, D, text_first): HunyuanVideo 720p (text last), Wan 720p (no text), CogVideoX 720x480 (text first)
SHAPES = {
    "hy720p": (256, 33, 3600, 128, False),
    "wan720p": (0, 21, 3600, 128, False),
    "cog": (226, 13, 1350, 64, True),
}
# cfg 2 x 2 heads: one spatial (0) and one temporal (1) head in each cfg half
BEST = [[0, 1], [1, 0]]


def _mirrors(text_first):
    from svgb200 import placement as pl

    if text_first:
        return pl.cog_sparse_head_placement, pl.cog_hidden_states_placement
    return pl.hunyuan_sparse_head_placement, pl.hunyuan_hidden_states_placement


def _oracle_place(g, best, ctx, F, P, text_first, inverse):
    from oracle import layout as ol

    cfg, H, S, D = g.shape
    return ol.head_placement(g.cpu().view(cfg * H, S, D), np.asarray(best).reshape(-1), ctx, F, P,
                             text_first=text_first, inverse=inverse)


def _randn(shape, dtype, cuda, gen):
    return torch.randn(shape, device=cuda, generator=gen).to(dtype)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("shape", list(SHAPES))
def test_placement_gradients_exact(cuda, shape, dtype):
    """The placement mirror's dQ / dK / dV are its incoming gradients placed back (inverse placement), the inverse
    mirror's gradient is its incoming gradient placed forward: bit for bit, outputs passed as zeros_like buffers as the
    reference does, the three gradients in one launch."""
    from svgb200 import core

    ctx, F, P, D, tf = SHAPES[shape]
    S = ctx + F * P
    fwd, inv = _mirrors(tf)
    gen = torch.Generator(device=cuda).manual_seed(len(shape) * 10 + D)
    best = torch.tensor(BEST, device=cuda)
    q, k, v, gq, gk, gv, gh = (_randn((2, 2, S, D), dtype, cuda, gen) for _ in range(7))
    x = [t.clone().requires_grad_() for t in (q, k, v)]
    outs = [torch.zeros_like(t) for t in x]
    fwd(*x, *outs, best, ctx, F, P)
    assert all(o.grad_fn is not None for o in outs)
    ref = [torch.zeros_like(t) for t in (q, k, v)]
    fwd(q, k, v, *ref, best, ctx, F, P)
    for o, r in zip(outs, ref):
        assert torch.equal(o.detach(), r)
    n0 = core.launch_count
    torch.autograd.backward(outs, [gq, gk, gv])
    assert core.launch_count - n0 == 1
    for t, g in zip(x, (gq, gk, gv)):
        assert torch.equal(t.grad.cpu().view(4, S, D), _oracle_place(g, BEST, ctx, F, P, tf, inverse=True))
    del x, outs, ref
    h = q.clone().requires_grad_()
    o = torch.zeros_like(h)
    assert inv(h, o, best, ctx, F, P) is o and o.grad_fn is not None
    o.backward(gh)
    assert torch.equal(h.grad.cpu().view(4, S, D), _oracle_place(gh, BEST, ctx, F, P, tf, inverse=False))


@pytest.mark.parametrize("text_first", [False, True])
def test_placement_partial_requires_grad(cuda, text_first):
    """Only q requires grad: k and v get no gradient, dQ is exact.  An output buffer that had a history of its own
    gets no gradient for its old contents (every row is overwritten)."""
    from svgb200 import core

    ctx, F, P, D = (34, 5, 200, 64) if text_first else (64, 4, 256, 128)
    S = ctx + F * P
    fwd, _ = _mirrors(text_first)
    gen = torch.Generator(device=cuda).manual_seed(7)
    best = torch.tensor(BEST, device=cuda)
    q, k, v, g = (_randn((2, 2, S, D), torch.bfloat16, cuda, gen) for _ in range(4))
    qg = q.clone().requires_grad_()
    w = torch.ones((), device=cuda, dtype=torch.bfloat16, requires_grad=True)
    qo = torch.zeros_like(q) * w  # a buffer with history
    ko, vo = torch.zeros_like(k), torch.zeros_like(v)
    fwd(qg, k, v, qo, ko, vo, best, ctx, F, P)
    n0 = core.launch_count
    (qo.float() * g.float()).sum().backward()
    assert core.launch_count - n0 == 1
    assert k.grad is None and v.grad is None
    assert w.grad is None or float(w.grad) == 0.0
    assert torch.equal(qg.grad.cpu().view(4, S, D), _oracle_place(g, BEST, ctx, F, P, text_first, inverse=True))


@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("dtype", DTYPES)
def test_permutation_gradients_exact(cuda, dtype, D):
    """permute_tensor_by_labels_triton / permute_by_sorted_indices back-propagate by scattering, and
    apply_inverse_permutation_triton by gathering, under the same sorted indices: bit for bit against
    oracle.layout, on labels with empty clusters (only even ids are used) and many ties."""
    from oracle import layout as ol
    from svgb200 import permute as pm

    B, H, S, K = 1, 3, 9283, 200
    g = torch.Generator().manual_seed(D)
    labels = torch.randint(0, K // 2, (B * H, S), generator=g) * 2
    x, gy, gx = (torch.randn(B, H, S, D, generator=g).to(dtype) for _ in range(3))
    xg = x.to(cuda).requires_grad_()
    y, idx = pm.permute_tensor_by_labels_triton(xg, labels.to(cuda), 2, num_clusters=K)
    assert y.grad_fn is not None
    perm = idx.cpu().numpy()
    assert np.array_equal(perm, ol.stable_argsort_labels(labels.numpy()))
    y.backward(gy.to(cuda))
    ref_scatter = ol.permute_scatter(gy.view(B * H, S, D), perm)
    assert torch.equal(xg.grad.cpu().view(B * H, S, D), ref_scatter)
    xg2 = x.to(cuda).requires_grad_()
    pm.permute_by_sorted_indices(xg2, idx).backward(gy.to(cuda))
    assert torch.equal(xg2.grad.cpu().view(B * H, S, D), ref_scatter)
    z = y.detach().clone().requires_grad_()
    out = pm.apply_inverse_permutation_triton(z, idx, 2)
    assert out.grad_fn is not None and torch.equal(out.detach().cpu(), x)
    out.backward(gx.to(cuda))
    assert torch.equal(z.grad.cpu().view(B * H, S, D), ol.permute_gather(gx.view(B * H, S, D), perm))


# ---- SVG1 cores --------------------------------------------------------------------------------------------------
def _make_core(model, cfg, H, dtype, cuda):
    """-> (core, ctx, F, P, D)"""
    from svgb200.models import cog, hyvideo, wan

    if model == "hy":
        return hyvideo.HunyuanSVG1Core(64, 20, 4, 256, H, 128, 0.4, cuda, cfg_size=cfg, dtype=dtype), 64, 4, 256, 128
    if model == "wan":
        return wan.WanSVG1Core(4, 256, H, 128, 0.4, cuda, cfg_size=cfg, dtype=dtype), 0, 4, 256, 128
    return cog.CogSVG1Core(34, 5, 200, H, 64, 0.45, cuda, cfg_size=cfg, dtype=dtype), 34, 5, 200, 64


def _fix_head_choice(c, best):
    """Make sample_mse return MSEs whose argmin is `best` ([cfg, H]), so the test picks the mixed head choice."""
    def sample_mse(query, key, value, sampled_rows=None):
        return torch.stack([best, 1 - best]).to(query.device, query.dtype)
    c.sample_mse = sample_mse


def _oracle_core_grads(q, k, v, do, best, bm, ctx, F, P, text_first):
    """fp64 autograd through oracle.layout.head_placement -> oracle band attention -> inverse placement."""
    from oracle import layout as ol
    from oracle.attention import generic_mask_fn, masked_attention_bhsd

    cfg, H, S, D = q.shape
    b = best.reshape(-1).cpu().numpy()
    xs = [t.reshape(cfg * H, S, D).cpu().double().requires_grad_() for t in (q, k, v)]
    placed = [ol.head_placement(t, b, ctx, F, P, text_first=text_first) for t in xs]
    o = masked_attention_bhsd(*placed, generic_mask_fn(bm.mode, bm.m0, bm.m1, bm.m2), dtype=torch.float64)
    ol.head_placement(o, b, ctx, F, P, text_first=text_first, inverse=True).backward(
        do.reshape(cfg * H, S, D).cpu().double())
    return [t.grad for t in xs]


def _composed_grads(q, k, v, do, best, bm, ctx, F, P, text_first):
    """The same gradients from the no-grad API: placement -> attn_fwd(return_lse) -> attn_bwd on the placed dO ->
    inverse placement."""
    from svgb200 import core

    kw = dict(text_first=text_first)
    with torch.no_grad():
        placed = [torch.empty_like(t) for t in (q, k, v)]
        core.head_placement([q, k, v], placed, best, ctx, F, P, **kw)
        o, lse = core.attn_fwd(*placed, bm.plan, return_lse=True)
        dop = [torch.empty_like(do)]
        core.head_placement([do], dop, best, ctx, F, P, **kw)
        dplaced = core.attn_bwd(*placed, o, dop[0], lse, bm.plan)
        grads = [torch.empty_like(t) for t in (q, k, v)]
        core.head_placement(list(dplaced), grads, best, ctx, F, P, inverse=True, **kw)
    return grads


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("model", ["hy", "wan", "cog"])
def test_svg1_core_gradients(cuda, model, dtype):
    """SVG1Core.sparse_core under grad: the forward equals the no-grad output bit for bit; dQ, dK, dV equal the
    no-grad composition bit for bit, are within the attention backward's tolerance of fp64 autograd through the
    oracle, and two backward runs give the same bits."""
    from svgb200 import core

    cfg, H = 2, 2
    c, ctx, F, P, D = _make_core(model, cfg, H, dtype, cuda)
    S = ctx + F * P
    best = torch.tensor(BEST, device=cuda)
    _fix_head_choice(c, best)
    gen = torch.Generator(device=cuda).manual_seed(3 + D)
    q, k, v, do = (_randn((cfg, H, S, D), dtype, cuda, gen) for _ in range(4))
    with torch.no_grad():
        y0 = c.sparse_core(q, k, v)
    x = [t.clone().requires_grad_() for t in (q, k, v)]
    y = c.sparse_core(*x)
    assert y.grad_fn is not None
    assert torch.equal(y.detach(), y0)
    y.backward(do)
    got = [t.grad.clone() for t in x]
    for g, r in zip(got, _composed_grads(q, k, v, do, best, c.block_mask, ctx, F, P, c.text_first)):
        assert torch.equal(g, r)
    for t in x:
        t.grad = None
    n0 = core.launch_count
    c.sparse_core(*x).backward(do)
    # forward: placement, attention, inverse placement; backward: dO placement, attn_bwd (3), one inverse placement
    # for dQ, dK and dV together
    assert core.launch_count - n0 == 3 + 5
    for g, t in zip(got, x):
        assert torch.equal(g, t.grad)
    ref = _oracle_core_grads(q, k, v, do, best, c.block_mask, ctx, F, P, c.text_first)
    check_grads([g.reshape(cfg * H, S, D) for g in got], ref, dtype)


def test_svg1_core_launches_without_grad(cuda):
    """Without grad one sparse_core call makes the launches it always made: sample_mse (7), placement, band
    attention, inverse placement."""
    from gen_inputs import structured_qkv
    from svgb200 import core

    c, ctx, F, P, D = _make_core("hy", 1, 2, torch.bfloat16, cuda)
    q, k, v = (t.to(cuda) for t in structured_qkv(0, 2, F, P, ctx, D))
    rows = torch.randint(0, 500, (24,), generator=torch.Generator().manual_seed(0))
    n0 = core.launch_count
    y = c.sparse_core(q, k, v, sampled_rows=rows)
    assert core.launch_count - n0 == 10 and y.grad_fn is None


# ---- the reference's call sequences, replayed ---------------------------------------------------------------------
def test_svg1_reference_sequence(cuda):
    """hyvideo/attention.py:473-524 step by step: sample_mse -> argmin -> zeros_like x3 -> placement mirror ->
    patched flex_attention -> inverse placement into zeros_like; gradients vs the fp64 oracle."""
    from gen_inputs import structured_qkv
    from svgb200 import patch
    from svgb200 import placement as pl

    c, ctx, F, P, D = _make_core("hy", 1, 4, torch.bfloat16, cuda)
    S = ctx + F * P
    q, k, v = structured_qkv(4, 4, F, P, ctx, D)
    do = torch.randn(1, 4, S, D, generator=torch.Generator().manual_seed(4)).bfloat16()
    x = [t.to(cuda).requires_grad_() for t in (q, k, v)]
    rows = torch.randint(0, 500, (24,), generator=torch.Generator().manual_seed(1))
    best = torch.argmin(c.sample_mse(*x, sampled_rows=rows), dim=0)
    outs = [torch.zeros_like(t) for t in x]
    pl.hunyuan_sparse_head_placement(*x, *outs, best, ctx, F, P)
    hidden = patch.flex_attention(*outs, block_mask=c.block_mask)
    o = pl.hunyuan_hidden_states_placement(hidden, torch.zeros_like(hidden), best, ctx, F, P)
    assert o.grad_fn is not None
    o.backward(do.to(cuda))
    ref = _oracle_core_grads(q, k, v, do, best, c.block_mask, ctx, F, P, False)
    check_grads([t.grad[0] for t in x], ref, torch.bfloat16)


def test_wan_svg2_reference_sequence(cuda):
    """wan/attention.py:499-559 step by step: batch_kmeans_Euclid -> identify_dynamic_map ->
    permute_tensor_by_labels_triton x3 -> dynamic_block_sparse_fwd_flashinfer -> apply_inverse_permutation_triton.
    The oracle mask is the block map seen through both permutations: (i, j) allowed iff map[label_q(i), label_k(j)]."""
    from svgb200 import kmeans_utils as ku
    from svgb200 import permute as pm

    H, F, P, D, QC, KC = 2, 4, 300, 128, 6, 20
    S = F * P
    g = torch.Generator().manual_seed(2)
    q, k, v, do = (torch.randn(1, H, S, D, generator=g).bfloat16() for _ in range(4))
    x = [t.to(cuda).requires_grad_() for t in (q, k, v)]
    torch.manual_seed(0)
    ql, qc, qs, _ = ku.batch_kmeans_Euclid(x[0].view(H, S, D), QC, max_iters=4)
    kl, kc, ks, _ = ku.batch_kmeans_Euclid(x[1].view(H, S, D), KC, max_iters=4)
    for lab, sz, n in ((ql, qs, QC), (kl, ks, KC)):  # block sizes are the label counts
        assert torch.equal(torch.stack([torch.bincount(r, minlength=n) for r in lab]).cpu(), sz.long().cpu())
    dyn = ku.identify_dynamic_map(qc.view(1, H, QC, D), kc.view(1, H, KC, D), qs.view(1, H, QC), ks.view(1, H, KC),
                                  0.8, 0.1)
    qp, qidx = pm.permute_tensor_by_labels_triton(x[0], ql, dim=2)
    kp, kidx = pm.permute_tensor_by_labels_triton(x[1], kl, dim=2)
    vp, _ = pm.permute_tensor_by_labels_triton(x[2], kl, dim=2, sorted_indices=kidx)
    op = ku.dynamic_block_sparse_fwd_flashinfer(qp, kp, vp, dyn, qs.view(1, H, QC), ks.view(1, H, KC), is_cpu=False)
    o = pm.apply_inverse_permutation_triton(op, qidx, dim=2)
    assert o.grad_fn is not None
    o.backward(do.to(cuda))
    dyn, ql, kl = dyn[0].cpu(), ql.cpu(), kl.cpu()
    masks = [dyn[h][ql[h]][:, kl[h]] for h in range(H)]
    check_grads([t.grad[0] for t in x], oracle_grads(q[0], k[0], v[0], do[0], masks), torch.bfloat16)


# ---- the reference's own processors (skipped when the reference is not importable) --------------------------------
needs_ref = pytest.mark.skipif(not R.reference_available(), reason="needs the unmodified Sparse-VideoGen reference importable (tools/install_reference.py); its own processor code runs here")


@needs_ref
@pytest.mark.parametrize("case", ["hyvideo-svg", "wan-svg", "cog-svg", "wan-sap"])
def test_reference_processor_under_grad(cuda, case):
    """The reference's own attention_core_logic with svgb200 installed, on inputs that require grad: the output has a
    grad_fn and equals the no-grad output bit for bit (same sampled rows), and the gradients are finite and nonzero."""
    from gen_inputs import structured_qkv
    from svgb200 import patch

    model, kind = case.split("-")
    A = R.import_model_module(model, "attention")
    U = R.import_model_module(model, "utils")
    patch.install(A)
    H, F, P, sparsity = 2, 4, 256, 0.4
    ctx, plen, D = {"hyvideo": (48, 20, 128), "wan": (0, 0, 128), "cog": (34, 0, 64)}[model]
    S = ctx + F * P
    if kind == "sap":
        cls = A.WanAttn_SAPAttn_Processor
        cls.context_length, cls.num_frame, cls.frame_size = 0, F, P
        cls.num_q_centroids, cls.num_k_centroids, cls.top_p_kmeans, cls.min_kc_ratio = 6, 20, 0.8, 0.1
        cls.kmeans_iter_init, cls.kmeans_iter_step = 4, 1
        cls.first_layers_fp, cls.first_times_fp = 0, 900
        args = (torch.tensor([100.0]),)
    else:
        cls = getattr(A, {"hyvideo": "Hunyuan_SVGAttn_Processor2_0", "wan": "WanAttn_SVGAttn_Processor2_0",
                          "cog": "CogVideoX_SparseAttn_Processor2_0"}[model])
        cls.context_length, cls.num_frame, cls.frame_size = ctx, F, P
        cls.num_sampled_rows = 24
        cls.first_layers_fp, cls.first_times_fp = 0, (0.0 if model == "cog" else 900)
        if model == "hyvideo":
            cls.prompt_length, cls.sample_mse_max_row = plen, 500
        elif model == "wan":
            cls.sample_mse_max_row = 600
        w = U.sparsity_to_width(sparsity, ctx, F, P)
        if model == "cog":
            cls.block_mask = A.prepare_flexattention(1, H, D, torch.bfloat16, cuda, ctx, F, P, diag_width=w,
                                                     multiplier=w)
        else:
            cls.block_mask = A.prepare_flexattention(1, H, D, torch.bfloat16, cuda, ctx, plen, F, P, diag_width=w,
                                                     multiplier=w)
        if model == "hyvideo":
            cu = torch.tensor([0, F * P + plen, S], dtype=torch.int32, device=cuda)
            args = (torch.tensor([100.0]), 0, (cu, cu, S, S))
        else:
            args = (torch.tensor([500.0 if model == "cog" else 100.0]),)
    q, k, v = (t.to(cuda) for t in structured_qkv(5, H, F, P, ctx, D, text_first=model == "cog"))
    torch.manual_seed(9)
    with torch.no_grad():
        y0 = cls(layer_idx=0).attention_core_logic(q, k, v, *args)
    x = [t.clone().requires_grad_() for t in (q, k, v)]
    torch.manual_seed(9)
    y = cls(layer_idx=0).attention_core_logic(*x, *args)
    assert y.grad_fn is not None
    if kind == "svg":
        assert torch.equal(y.detach(), y0)
    y.float().square().sum().backward()
    for t in x:
        assert torch.isfinite(t.grad.float()).all() and t.grad.abs().sum() > 0
