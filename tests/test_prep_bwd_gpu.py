"""Backward of the pre-attention chain on the GPU: the fused qkv_prep backward, the in-place norm and RoPE backwards
and their autograd wiring (core._QkvPrep / _RowNorm / _QkRope).

Exact tests (layout, RoPE census, fused == stepwise) compare bits.  Tests against float64 autograd (through
tests/prep_fp64.py, oracle.prep's chain restated in float64, on float64 copies of the 16-bit inputs) use a norm-wise
relative error
    |got - ref|_2 / |ref|_2 <= REL[dtype]
with REL = 1.5e-2 (bf16) and 4e-3 (fp16): the backward rounds the RoPE transpose and dx to the 16-bit dtype
(relative 2^-9 / 2^-12 each), so the norm-wise error is a few of those units; the parameter gradients are fp32 sums
rounded once to the weight dtype."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

REL = {torch.bfloat16: 1.5e-2, torch.float16: 4e-3}
DTYPES = [torch.bfloat16, torch.float16]


def rel_close(got, ref, dtype, what="", tol=None):
    got = got.double().cpu()
    ref = ref.double().cpu()
    tol = REL[dtype] if tol is None else tol
    assert torch.isfinite(got).all(), f"{what}: non-finite values"
    err = float((got - ref).norm() / ref.norm().clamp_min(1e-30))
    assert err <= tol, f"{what}: norm-wise relative error {err:.3e} > {tol}"


def poison(cuda, nbytes=64 << 20):
    """Fill the caching allocator's free blocks with NaN so outputs the kernels never write show up as NaN."""
    t = torch.full((nbytes // 2,), float("nan"), dtype=torch.float16, device=cuda)
    del t


def packed_inputs(B, S, H, D, dtype, gen, cuda, requires_grad=True):
    """q_in, k_in, v_in as strided views of one packed [B, S, 3*H*D] projection output."""
    packed = torch.randn(B, S, 3 * H * D, generator=gen).to(dtype).to(cuda).requires_grad_(requires_grad)
    return packed, (packed[..., :H * D], packed[..., H * D:2 * H * D], packed[..., 2 * H * D:])


def small_ints(shape, gen, lo=-8, hi=9):
    return torch.randint(lo, hi, shape, generator=gen).float()


def census_tables(n, width, gen):
    """cos / sin drawn per element from {-1, -1/2, 0, 1/2, 1}: c[2i] != c[2i+1] occurs, every product is exact."""
    vals = torch.tensor([-1.0, -0.5, 0.0, 0.5, 1.0])
    return vals[torch.randint(0, 5, (n, width), generator=gen)], vals[torch.randint(0, 5, (n, width), generator=gen)]


def rope_t_ref(dy, c, s, complex_):
    """Closed-form transpose of the interleaved / complex rotation on [..., n, D] (float64)."""
    dy, c, s = dy.double(), c.double(), s.double()
    a, b = dy[..., 0::2], dy[..., 1::2]
    if complex_:
        return torch.stack([a * c + b * s, b * c - a * s], -1).flatten(-2)
    ce, co, se, so = c[..., 0::2], c[..., 1::2], s[..., 0::2], s[..., 1::2]
    return torch.stack([a * ce + b * so, b * co - a * se], -1).flatten(-2)


# ---- 1. layout census ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("D", [64, 128, 256])
def test_layout_census_exact(cuda, dtype, D):
    """Norm NONE, no RoPE: dq_in / dk_in / dv_in are the transpose of rows [out_row0, out_row0 + S_in) of the incoming
    gradients, bit for bit; the rows outside that range are NaN and must never be read."""
    from svgb200 import core

    B, S, H, r0, tail = 2, 301, 3, 37, 11
    g = torch.Generator().manual_seed(D)
    packed, (qi, ki, vi) = packed_inputs(B, S, H, D, dtype, g, cuda)
    outs = core.qkv_prep(qi, ki, vi, H, out_row0=r0, out_rows=r0 + S + tail)
    grads = []
    for _ in range(3):
        gr = torch.full((B, H, r0 + S + tail, D), float("nan"), dtype=dtype)
        gr[:, :, r0:r0 + S] = torch.randn(B, H, S, D, generator=g).to(dtype)
        grads.append(gr.to(cuda))
    poison(cuda)
    torch.autograd.backward(outs, grads)
    want = torch.cat([gr[:, :, r0:r0 + S].transpose(1, 2).reshape(B, S, H * D) for gr in grads], -1)
    assert not torch.isnan(packed.grad).any()
    assert torch.equal(packed.grad, want)
    # the direct entry point, with the forward's strides
    dqi, dki, dvi, *rest = core.qkv_prep_bwd(*grads, H, S, out_row0=r0)
    assert rest == [None] * 4
    assert torch.equal(torch.cat([dqi, dki, dvi], -1), want)


# ---- 2. RoPE census -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("D", [64, 128, 256])
def test_rope_census_inplace_exact(cuda, dtype, mode, D):
    """The in-place RoPE under autograd (Hq != Hk): integer gradients, tables from {-1,-1/2,0,1/2,1}; the rotated
    rows get the closed-form transpose bit for bit, the text rows pass through."""
    from svgb200 import _kernels

    B, Hq, Hk, S, txt = 2, 4, 2, 203, 29
    g = torch.Generator().manual_seed(mode * 1000 + D)
    width = D // 2 if mode == 2 else D
    cos, sin = census_tables(S - txt, width, g)
    q0 = torch.randn(B, Hq, S, D, generator=g).to(dtype).to(cuda).requires_grad_()
    k0 = torch.randn(B, Hk, S, D, generator=g).to(dtype).to(cuda).requires_grad_()
    q, k = q0 * 1, k0 * 1
    fn = [_kernels.apply_qk_rope_inplace_cossin, _kernels.apply_qk_rope_inplace_cossin_txtlast,
          _kernels.apply_qk_rope_inplace_cossin_complex][mode]
    fn(q, k, cos.to(cuda), sin.to(cuda), txt)
    dq, dk = small_ints(q.shape, g).to(dtype), small_ints(k.shape, g).to(dtype)
    poison(cuda)
    torch.autograd.backward((q, k), (dq.to(cuda), dk.to(cuda)))
    lo, hi = (0, S - txt) if mode == 1 else (txt, S)
    for got, d in ((q0.grad, dq), (k0.grad, dk)):
        want = d.double().clone()
        want[:, :, lo:hi] = rope_t_ref(d[:, :, lo:hi], cos, sin, mode == 2)
        assert torch.equal(got.double().cpu(), want)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("rope, text_first", [(1, False), (1, True), (2, True)])
@pytest.mark.parametrize("D", [64, 128, 256])
def test_rope_census_fused_exact(cuda, dtype, rope, text_first, D):
    from svgb200 import core

    B, S, H, txt = 2, 157, 3, 21
    g = torch.Generator().manual_seed(rope * 100 + D + text_first)
    width = D // 2 if rope == 2 else D
    cos, sin = census_tables(S - txt, width, g)
    lo = txt if text_first else 0
    packed, (qi, ki, vi) = packed_inputs(B, S, H, D, dtype, g, cuda)
    outs = core.qkv_prep(qi, ki, vi, H, rope=rope, cos=cos.to(cuda), sin=sin.to(cuda), rope_lo=lo, rope_n=S - txt)
    grads = [small_ints((B, H, S, D), g).to(dtype) for _ in range(3)]
    poison(cuda)
    torch.autograd.backward(outs, [t.to(cuda) for t in grads])
    want = []
    for i, d in enumerate(grads):
        w = d.double().clone()
        if i < 2:
            w[:, :, lo:lo + S - txt] = rope_t_ref(d[:, :, lo:lo + S - txt], cos, sin, rope == 2)
        want.append(w.transpose(1, 2).reshape(B, S, H * D))
    assert torch.equal(packed.grad.double().cpu(), torch.cat(want, -1))


# ---- 3. fused == stepwise -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("norm", [0, 1, 2])
@pytest.mark.parametrize("rope", [0, 1, 2])
def test_fused_backward_equals_stepwise(cuda, dtype, norm, rope):
    """The fused backward against the reference's in-place sequence under autograd (transpose -> _kernels norm on a
    .view(-1, D) -> _kernels RoPE): input gradients bit for bit, norm weight gradients within tolerance (the two
    reductions sum in different orders)."""
    from svgb200 import _kernels, core

    B, S, H, D, txt = 2, 333, 5, 128, 40
    g = torch.Generator().manual_seed(norm * 10 + rope)
    base = torch.randn(B, S, 3 * H * D, generator=g).to(dtype)
    w = [torch.randn(D, generator=g).to(dtype).to(cuda) for _ in range(4)]
    width = D // 2 if rope == 2 else D
    cos, sin = (torch.randn(S - txt, width, generator=g).to(cuda) for _ in range(2))
    lo = txt if rope == 2 else 0
    grads = [torch.randn(B, H, S, D, generator=g).to(dtype).to(cuda) for _ in range(3)]

    def params():
        p = base.to(cuda).requires_grad_()
        ws = [t.clone().requires_grad_() for t in w]
        return p, ws

    p1, w1 = params()
    qi, ki, vi = p1[..., :H * D], p1[..., H * D:2 * H * D], p1[..., 2 * H * D:]
    outs = core.qkv_prep(qi, ki, vi, H, norm=norm, gamma_q=w1[0] if norm else None, gamma_k=w1[1] if norm else None,
                         beta_q=w1[2] if norm == 2 else None, beta_k=w1[3] if norm == 2 else None, eps=1e-6,
                         rope=rope, cos=cos if rope else None, sin=sin if rope else None, rope_lo=lo,
                         rope_n=S - txt if rope else None)
    torch.autograd.backward(outs, grads)

    p2, w2 = params()
    sq, sk, sv = (p2[..., i * H * D:(i + 1) * H * D].unflatten(2, (H, -1)).transpose(1, 2).contiguous()
                  for i in range(3))
    if norm == 1:
        _kernels.rms_norm_forward(sq.view(-1, D), w2[0], 1e-6), _kernels.rms_norm_forward(sk.view(-1, D), w2[1], 1e-6)
    elif norm == 2:
        _kernels.layer_norm_forward(sq.view(-1, D), w2[0], w2[2])
        _kernels.layer_norm_forward(sk.view(-1, D), w2[1], w2[3])
    if rope == 1:
        _kernels.apply_qk_rope_inplace_cossin_txtlast(sq, sk, cos, sin, txt)
    elif rope == 2:
        _kernels.apply_qk_rope_inplace_cossin_complex(sq, sk, cos, sin, txt)
    assert torch.equal(outs[0], sq) and torch.equal(outs[1], sk) and torch.equal(outs[2], sv)
    torch.autograd.backward((sq, sk, sv), grads)

    assert torch.equal(p1.grad, p2.grad)
    for i in range(4 if norm == 2 else 2 if norm else 0):
        rel_close(w1[i].grad, w2[i].grad, dtype, f"weight {i}")


# ---- 4. against float64 autograd through the reference chain --------------------------------------------------------------
def ref_grads(qi, ki, vi, H, norm, ws, eps, rope, cos, sin, lo, n, grads):
    """float64 autograd through prep_fp64.qkv_chain on float64 copies of the 16-bit inputs."""
    import prep_fp64 as op

    leaves = [t.detach().double().cpu().requires_grad_() for t in (qi, ki, vi)]
    wl = [None if t is None else t.detach().double().cpu().requires_grad_() for t in ws]
    c, s = (None, None) if not rope else (cos.cpu().double(), sin.cpu().double())
    outs = op.qkv_chain(*leaves, H, norm, *wl, eps, rope, c, s, lo, n)
    torch.autograd.backward(outs, [gr.double().cpu() for gr in grads])
    return [t.grad for t in leaves], [None if t is None or t.grad is None else t.grad for t in wl]


ORACLE_CASES = [  # (norm, rope, text_first, H, D, S)
    (0, 0, False, 3, 128, 97), (0, 1, False, 3, 128, 97), (0, 2, True, 3, 64, 97),
    (1, 0, False, 3, 128, 131), (1, 1, False, 3, 128, 131), (1, 1, True, 2, 256, 131), (1, 2, True, 3, 64, 131),
    (2, 0, False, 3, 64, 77), (2, 1, True, 3, 64, 77), (2, 2, True, 2, 128, 77),
    (3, 0, False, 3, 128, 59), (3, 2, True, 3, 64, 59), (3, 1, False, 2, 256, 59),
]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("norm, rope, text_first, H, D, S", ORACLE_CASES)
def test_against_fp64_autograd(cuda, dtype, norm, rope, text_first, H, D, S):
    from svgb200 import core

    B, txt = 2, 13
    g = torch.Generator().manual_seed(norm * 97 + rope * 7 + D + S)
    packed, (qi, ki, vi) = packed_inputs(B, S, H, D, dtype, g, cuda)
    gw = H * D if norm == 3 else D
    ws = [(1 + 0.3 * torch.randn(gw, generator=g)).to(dtype).to(cuda).requires_grad_() if norm else None
          for _ in range(2)]
    ws += [(0.3 * torch.randn(gw, generator=g)).to(dtype).to(cuda).requires_grad_() if norm == 2 else None
           for _ in range(2)]
    width = D // 2 if rope == 2 else D
    n = S - txt if rope else 0
    lo = txt if text_first else 0
    cos = torch.randn(n, width, generator=g).to(cuda) if rope else None
    sin = torch.randn(n, width, generator=g).to(cuda) if rope else None
    outs = core.qkv_prep(qi, ki, vi, H, norm=norm, gamma_q=ws[0], gamma_k=ws[1], beta_q=ws[2], beta_k=ws[3],
                         eps=1e-6, rope=rope, cos=cos, sin=sin, rope_lo=lo, rope_n=n if rope else None)
    grads = [torch.randn(B, H, S, D, generator=g).to(dtype).to(cuda) for _ in range(3)]
    torch.autograd.backward(outs, grads)
    dx_ref, dw_ref = ref_grads(qi, ki, vi, H, norm, ws, 1e-6, rope, cos, sin, lo, n, grads)
    for i, name in enumerate(("dq_in", "dk_in", "dv_in")):
        rel_close(packed.grad[..., i * H * D:(i + 1) * H * D], dx_ref[i], dtype, name)
    for i, w in enumerate(ws):
        if w is not None:
            assert w.grad.dtype == dtype
            rel_close(w.grad, dw_ref[i], dtype, f"weight {i}")


@pytest.mark.parametrize("dtype", DTYPES)
def test_wan_hidden_rms_5120_against_fp64(cuda, dtype):
    """Wan: RMS over the full hidden row H*D = 40*128 = 5120, complex RoPE on every row, odd S."""
    from svgb200 import prep

    B, S, H, D = 1, 67, 40, 128
    g = torch.Generator().manual_seed(5120)
    packed, (qi, ki, vi) = packed_inputs(B, S, H, D, dtype, g, cuda)
    wq, wk = ((1 + 0.3 * torch.randn(H * D, generator=g)).to(dtype).to(cuda).requires_grad_() for _ in range(2))
    fr, fi = (torch.randn(S, D // 2, generator=g).to(cuda) for _ in range(2))
    outs = prep.wan_qkv(qi, ki, vi, H, wq, wk, 1e-6, fr, fi)
    grads = [torch.randn(B, H, S, D, generator=g).to(dtype).to(cuda) for _ in range(3)]
    torch.autograd.backward(outs, grads)
    dx_ref, dw_ref = ref_grads(qi, ki, vi, H, 3, [wq, wk, None, None], 1e-6, 2, fr, fi, 0, S, grads)
    for i in range(3):
        rel_close(packed.grad[..., i * H * D:(i + 1) * H * D], dx_ref[i], dtype, f"dx {i}")
    rel_close(wq.grad, dw_ref[0], dtype, "dgamma_q")
    rel_close(wk.grad, dw_ref[1], dtype, "dgamma_k")


@pytest.mark.parametrize("dtype", DTYPES)
def test_cog_layernorm_d64_text_first_against_fp64(cuda, dtype):
    from svgb200 import prep

    B, S, H, D, txt = 2, 91, 4, 64, 17
    g = torch.Generator().manual_seed(64)
    packed, (qi, ki, vi) = packed_inputs(B, S, H, D, dtype, g, cuda)
    w = [(1 + 0.3 * torch.randn(D, generator=g)).to(dtype).to(cuda).requires_grad_() for _ in range(4)]
    cos, sin = (torch.randn(S - txt, D, generator=g).to(cuda) for _ in range(2))
    outs = prep.cog_qkv(qi, ki, vi, H, w[0], w[1], w[2], w[3], cos, sin, txt)
    grads = [torch.randn(B, H, S, D, generator=g).to(dtype).to(cuda) for _ in range(3)]
    torch.autograd.backward(outs, grads)
    dx_ref, dw_ref = ref_grads(qi, ki, vi, H, 2, [w[0], w[2], w[1], w[3]], 1e-6, 1, cos, sin, txt, S - txt, grads)
    for i in range(3):
        rel_close(packed.grad[..., i * H * D:(i + 1) * H * D], dx_ref[i], dtype, f"dx {i}")
    for got, ref in zip((w[0], w[2], w[1], w[3]), dw_ref):
        rel_close(got.grad, ref, dtype, "norm weights")


# ---- 5. end to end ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
def test_hunyuan_single_block_against_fp64(cuda, dtype):
    from svgb200 import prep

    B, S, H, D, txt = 1, 203, 3, 128, 31
    g = torch.Generator().manual_seed(11)
    packed, (qi, ki, vi) = packed_inputs(B, S, H, D, dtype, g, cuda)
    wq, wk = ((1 + 0.3 * torch.randn(D, generator=g)).to(dtype).to(cuda).requires_grad_() for _ in range(2))
    cos, sin = (torch.randn(S - txt, D, generator=g).to(cuda) for _ in range(2))
    outs = prep.hunyuan_single_block_qkv(qi, ki, vi, H, wq, wk, 1e-6, cos, sin, txt)
    grads = [torch.randn(B, H, S, D, generator=g).to(dtype).to(cuda) for _ in range(3)]
    torch.autograd.backward(outs, grads)
    dx_ref, dw_ref = ref_grads(qi, ki, vi, H, 1, [wq, wk, None, None], 1e-6, 1, cos, sin, 0, S - txt, grads)
    for i in range(3):
        rel_close(packed.grad[..., i * H * D:(i + 1) * H * D], dx_ref[i], dtype, f"dx {i}")
    rel_close(wq.grad, dw_ref[0], dtype, "dgamma_q")
    rel_close(wk.grad, dw_ref[1], dtype, "dgamma_k")


@pytest.mark.parametrize("prompt_norm", [True, False])
def test_hunyuan_double_block_both_streams(cuda, prompt_norm):
    """Both streams in one node: the video stream (RMS + RoPE) reads rows [0, Sv) of the gradient, the prompt stream
    (its own RMS weights, no RoPE) rows [Sv, Sv + St); all six inputs and all four weight sets get their gradients."""
    from svgb200 import prep

    dtype = torch.bfloat16
    B, Sv, St, H, D = 2, 150, 37, 3, 128
    g = torch.Generator().manual_seed(12 + prompt_norm)
    vid = [torch.randn(B, Sv, H * D, generator=g).to(dtype).to(cuda).requires_grad_() for _ in range(3)]
    txt = [torch.randn(B, St, H * D, generator=g).to(dtype).to(cuda).requires_grad_() for _ in range(3)]
    w = [(1 + 0.3 * torch.randn(D, generator=g)).to(dtype).to(cuda).requires_grad_() for _ in range(4)]
    if not prompt_norm:
        w[2] = w[3] = None
    cos, sin = (torch.randn(Sv, D, generator=g).to(cuda) for _ in range(2))
    outs = prep.hunyuan_double_block_qkv(*vid, *txt, H, w[0], w[1], w[2], w[3], 1e-6, cos, sin)
    assert "_QkvPrep" in outs[0].grad_fn.name()  # one node records both streams
    grads = [torch.randn(B, H, Sv + St, D, generator=g).to(dtype).to(cuda) for _ in range(3)]
    torch.autograd.backward(outs, grads)
    rv, rwv = ref_grads(*vid, H, 1, [w[0], w[1], None, None], 1e-6, 1, cos, sin, 0, Sv,
                           [gr[:, :, :Sv] for gr in grads])
    rt, rwt = ref_grads(*txt, H, 1 if prompt_norm else 0, [w[2], w[3], None, None], 1e-6, 0, None, None, 0, 0,
                           [gr[:, :, Sv:] for gr in grads])
    for t, r in zip(vid + txt, rv + rt):
        rel_close(t.grad, r, dtype, "stream input")
    rel_close(w[0].grad, rwv[0], dtype, "norm_q_weight")
    rel_close(w[1].grad, rwv[1], dtype, "norm_k_weight")
    if prompt_norm:
        rel_close(w[2].grad, rwt[0], dtype, "norm_added_q_weight")
        rel_close(w[3].grad, rwt[1], dtype, "norm_added_k_weight")


def test_prep_attention_loss_reaches_projections_and_norm_weights(cuda):
    """prep -> core.attention -> loss: the projection outputs and the QK norm weights get finite, non-zero
    gradients, and the chain matches float64 autograd through the reference prep chain and torch attention."""
    from svgb200 import core, prep

    dtype = torch.bfloat16
    B, S, H, D, txt = 1, 256, 2, 128, 32
    g = torch.Generator().manual_seed(21)
    packed, (qi, ki, vi) = packed_inputs(B, S, H, D, dtype, g, cuda)
    wq, wk = ((1 + 0.3 * torch.randn(D, generator=g)).to(dtype).to(cuda).requires_grad_() for _ in range(2))
    cos, sin = (torch.randn(S - txt, D, generator=g).to(cuda) for _ in range(2))
    q, k, v = prep.hunyuan_single_block_qkv(qi, ki, vi, H, wq, wk, 1e-6, cos, sin, txt)
    plan = core.plan_band(core.MASK_NONE, 0, 0, 0, B * H, S, cuda)
    o = core.attention(q, k, v, plan)
    wo = torch.randn(o.shape, generator=g).to(dtype).to(cuda)
    (o.float() * wo.float()).sum().backward()
    for t in (packed.grad, wq.grad, wk.grad):
        assert t is not None and torch.isfinite(t.float()).all() and t.float().abs().sum() > 0

    import prep_fp64 as op

    leaves = [t.detach().double().cpu().requires_grad_() for t in (qi, ki, vi)]
    wl = [t.detach().double().cpu().requires_grad_() for t in (wq, wk)]
    rq, rk, rv = op.qkv_chain(*leaves, H, 1, wl[0], wl[1], None, None, 1e-6, 1, cos.cpu().double(),
                              sin.cpu().double(), 0, S - txt)
    p = torch.softmax(rq @ rk.transpose(-1, -2) / math.sqrt(D), -1)
    ((p @ rv) * wo.double().cpu()).sum().backward()
    # the bf16 attention backward adds its own rounding (P and dS in bf16) on top of the prep backward's
    for i in range(3):
        rel_close(packed.grad[..., i * H * D:(i + 1) * H * D], leaves[i].grad, dtype, f"projection {i}", 4e-2)
    rel_close(wq.grad, wl[0].grad, dtype, "norm_q_weight", 4e-2)
    rel_close(wk.grad, wl[1].grad, dtype, "norm_k_weight", 4e-2)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("layer", [False, True])
@pytest.mark.parametrize("n", [32, 64, 128, 256])
def test_inplace_norm_on_view_against_fp64(cuda, dtype, layer, n):
    """The _kernels drop-ins applied in place on a .view(-1, n) of a non-leaf: x and the weights get the gradient of
    the norm (not of the identity)."""
    import prep_fp64 as op
    from svgb200 import _kernels

    g = torch.Generator().manual_seed(n + layer)
    x0 = torch.randn(3, 5, 41, n, generator=g).to(dtype).to(cuda).requires_grad_()
    w = (1 + 0.3 * torch.randn(n, generator=g)).to(dtype).to(cuda).requires_grad_()
    b = (0.3 * torch.randn(n, generator=g)).to(dtype).to(cuda).requires_grad_()
    x = x0.transpose(1, 2).contiguous()
    if layer:
        _kernels.layer_norm_forward(x.view(-1, n), w, b)
    else:
        _kernels.rms_norm_forward(x.view(-1, n), w, 1e-5)
    gy = torch.randn(x.shape, generator=g).to(dtype).to(cuda)
    x.backward(gy)
    xl, wl, bl = (t.detach().double().cpu().requires_grad_() for t in (x0, w, b))
    y = op.layer_norm(xl.transpose(1, 2), wl, bl) if layer else op.rms_norm(xl.transpose(1, 2), wl, 1e-5)
    y.backward(gy.double().cpu())
    rel_close(x0.grad, xl.grad, dtype, "dx")
    rel_close(w.grad, wl.grad, dtype, "dgamma")
    if layer:
        rel_close(b.grad, bl.grad, dtype, "dbeta")


# ---- 6. determinism and full size ---------------------------------------------------------------------------------
def test_fullsize_hunyuan_deterministic_and_sampled_fp64(cuda):
    """HunyuanVideo 720p single block (S = 119056, H = 24, D = 128, RMS per head, RoPE text last): two backward runs
    give the same bits (dx and dgamma), and sampled token rows match float64."""
    import prep_fp64 as op
    from svgb200 import core

    dtype = torch.bfloat16
    B, S, H, D, txt = 1, 119056, 24, 128, 256
    g = torch.Generator(device=cuda).manual_seed(4)
    qi, ki = (torch.randn(B, S, H * D, device=cuda, generator=g).to(dtype) for _ in range(2))
    wq, wk = ((1 + 0.3 * torch.randn(D, device=cuda, generator=g)).to(dtype) for _ in range(2))
    cos, sin = (torch.randn(S - txt, D, device=cuda, generator=g) for _ in range(2))
    grads = [torch.randn(B, H, S, D, device=cuda, generator=g).to(dtype) for _ in range(3)]
    kw = dict(q_in=qi, k_in=ki, norm=core.NORM_RMS_HEAD, gamma_q=wq, gamma_k=wk, eps=1e-6, rope=1, cos=cos, sin=sin,
              rope_lo=0, rope_n=S - txt)
    first = core.qkv_prep_bwd(*grads, H, S, **kw)
    second = core.qkv_prep_bwd(*grads, H, S, **kw)
    assert first[5] is None and first[6] is None  # RMS: no dbeta
    for a, b in zip(first[:5], second[:5]):
        assert torch.equal(a, b)
    rows = torch.cat([torch.randint(0, S - txt, (40,), generator=torch.Generator().manual_seed(0)),
                      torch.arange(S - txt - 2, S - txt + 2), torch.tensor([S - 1])]).to(cuda)
    for i, (x, w) in enumerate(((qi, wq), (ki, wk))):
        xs = x[0, rows].detach().double().cpu().view(-1, H, D).requires_grad_()
        rot = (rows < S - txt).cpu()
        y = op.rms_norm(xs, w.double().cpu(), 1e-6)
        c, s = cos[rows.clamp(max=S - txt - 1)].double().cpu(), sin[rows.clamp(max=S - txt - 1)].double().cpu()
        yr = torch.where(rot[:, None, None], op.rope_interleave(y.transpose(0, 1), c, s).transpose(0, 1), y)
        yr.backward(grads[i][0, :, rows].transpose(0, 1).double().cpu())
        rel_close(first[i][0, rows].view(-1, H, D), xs.grad, dtype, "sampled dx")
    assert torch.equal(first[2], grads[2].transpose(1, 2).reshape(B, S, H * D))
    assert torch.isfinite(first[3].float()).all() and torch.isfinite(first[4].float()).all()


# ---- 7. no grad: unchanged ----------------------------------------------------------------------------------------
def test_no_grad_paths_unchanged(cuda):
    """Without grad every entry makes exactly the launches it made before (one per call, two for the double block)
    and the forward bits equal those of the recording path."""
    from svgb200 import _kernels, core, prep

    dtype = torch.bfloat16
    B, S, H, D, txt = 1, 160, 2, 128, 16
    g = torch.Generator().manual_seed(31)
    qi, ki, vi = (torch.randn(B, S, H * D, generator=g).to(dtype).to(cuda) for _ in range(3))
    wq, wk = (torch.randn(D, generator=g).to(dtype).to(cuda) for _ in range(2))
    cos, sin = (torch.randn(S - txt, D, generator=g).to(cuda) for _ in range(2))
    cf, sf = (torch.randn(S, D, generator=g).to(cuda) for _ in range(2))  # the double block rotates every video row

    def launches(fn):
        n0 = core.launch_count
        r = fn()
        return core.launch_count - n0, r

    n, plain = launches(lambda: prep.hunyuan_single_block_qkv(qi, ki, vi, H, wq, wk, 1e-6, cos, sin, txt))
    assert n == 1
    n, dbl = launches(lambda: prep.hunyuan_double_block_qkv(qi, ki, vi, qi, ki, vi, H, wq, wk, wq, wk, 1e-6, cf, sf))
    assert n == 2
    x = plain[0].clone()
    n, _ = launches(lambda: _kernels.rms_norm_forward(x.view(-1, D), wq, 1e-6))
    assert n == 1
    n, _ = launches(lambda: _kernels.apply_qk_rope_inplace_cossin_txtlast(x, x.clone(), cos, sin, txt))
    assert n == 1
    with torch.no_grad():
        wg = wq.clone().requires_grad_()
        n, r = launches(lambda: prep.hunyuan_single_block_qkv(qi, ki, vi, H, wg, wk, 1e-6, cos, sin, txt))
        assert n == 1 and r[0].grad_fn is None
    qg = qi.clone().requires_grad_()
    rec = prep.hunyuan_single_block_qkv(qg, ki, vi, H, wq, wk, 1e-6, cos, sin, txt)
    assert rec[0].grad_fn is not None
    for a, b in zip(plain, rec):
        assert torch.equal(a, b.detach())
    rec2 = prep.hunyuan_double_block_qkv(qg, ki, vi, qi, ki, vi, H, wq, wk, wq, wk, 1e-6, cf, sf)
    for a, b in zip(dbl, rec2):
        assert torch.equal(a, b.detach())


def test_raises_under_grad(cuda):
    from svgb200 import core, triton_glue as tg

    dtype = torch.bfloat16
    B, S, H, D = 1, 64, 2, 64
    qi, ki, vi = (torch.randn(B, S, H * D, device=cuda).to(dtype).requires_grad_() for _ in range(3))
    out = tuple(torch.empty(B, H, S, D, device=cuda, dtype=dtype) for _ in range(3))
    with pytest.raises(core.SvgbError, match="out=.*no backward"):
        core.qkv_prep(qi, ki, vi, H, out=out)
    cos = torch.randn(S, D, device=cuda, requires_grad=True)
    with pytest.raises(core.SvgbError, match="cos / sin"):
        core.qkv_prep(qi, ki, vi, H, rope=1, cos=cos, sin=cos.detach())
    q = torch.randn(B, H, S, D, device=cuda).to(dtype)
    with pytest.raises(core.SvgbError, match="cos / sin"):
        core.qk_rope_(q, q.clone(), cos, cos.detach(), 0, core.ROPE_TXT_FIRST)
    x = torch.randn(2, 7, 256, device=cuda, requires_grad=True)
    w = torch.randn(256, device=cuda)
    scale, shift = torch.randn(2, 1, 256, device=cuda), torch.randn(2, 1, 256, device=cuda)
    for fn in (lambda: tg.triton_layernorm_forward(x, w, w, 1e-6, True),
               lambda: tg.layernorm_modulate_forward(x, None, None, 1e-6, scale, shift),
               lambda: tg.triton_rmsnorm_forward(x, w, 1e-6),
               lambda: tg.triton_modulate_shift_forward(x, scale, shift),
               lambda: tg.triton_modulate_gate_residual_forward(x.detach(), x, scale)):
        with pytest.raises(core.SvgbError, match="has no backward"):
            fn()
    with torch.no_grad():
        tg.triton_rmsnorm_forward(x, w, 1e-6)
    leaf = torch.randn(4, 64, device=cuda).to(dtype).requires_grad_()
    with pytest.raises(RuntimeError, match="leaf"):
        core.rms_norm_(leaf, torch.ones(64, device=cuda, dtype=dtype))
