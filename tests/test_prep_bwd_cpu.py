"""Host side of the pre-attention chain's backward, without a GPU: the C ABI's argument checks, the raises under grad,
and the autograd wiring (core._RowNorm / _QkRope / _QkvPrep) with the kernel calls replaced by float64
stand-ins (tests/prep_fp64.py), so that what is checked here is the routing: mark_dirty on a view, which gradient goes where, and the
row ranges of the double block's two streams."""
import ctypes as C
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent


@pytest.fixture(scope="module")
def lib():
    import importlib.util

    spec = importlib.util.spec_from_file_location("svgb200_build", ROOT / "sparse-videogen_b200" / "build.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.build_lib()
    from svgb200 import _lib

    return _lib.lib()


def test_abi_argument_errors(lib):
    n = C.c_size_t()
    A = 256  # a 16-byte aligned stand-in address: every call below fails its checks before touching memory
    assert lib.svgb_qkv_prep_bwd_bytes(1, 100, 4, 96, 1, C.byref(n)) < 0
    assert b"Unsupported head_dim" in lib.svgb_last_error()
    assert lib.svgb_qkv_prep_bwd_bytes(1, 100, 4, 128, 4, C.byref(n)) < 0
    assert lib.svgb_qkv_prep_bwd_bytes(1, 100, 4, 128, 0, C.byref(n)) == 0 and n.value == 0
    assert lib.svgb_qkv_prep_bwd_bytes(1, 100, 4, 128, 1, C.byref(n)) == 0 and n.value > 0
    assert lib.svgb_qkv_prep_bwd_bytes(1, 75600, 40, 128, 3, C.byref(n)) == 0 and n.value < 64 << 20
    assert lib.svgb_row_norm_bwd_bytes(10, 48, C.byref(n)) < 0
    assert lib.svgb_row_norm_bwd_bytes(10, 128, C.byref(n)) == 0 and n.value > 0
    # workspace too small
    assert lib.svgb_rms_norm_bwd(A, A, A, A, A, 10, 128, C.c_float(1e-6), 0, A, 0, None) < 0
    assert b"workspace too small" in lib.svgb_last_error()
    assert lib.svgb_layer_norm_bwd(A, A, A, A, A, None, 10, 128, 0, A, 1 << 20, None) < 0
    assert b"null pointer" in lib.svgb_last_error()
    assert lib.svgb_rms_norm_bwd(A + 8, A, A, A, A, 10, 128, C.c_float(1e-6), 0, A, 1 << 20, None) < 0
    assert b"16-byte aligned" in lib.svgb_last_error()
    # RoPE: the forward's checks
    assert lib.svgb_qk_rope_bwd(A, A, A, A, A, A, 1, 2, 2, 100, 96, 0, 0, 0, None) < 0
    assert b"Unsupported head_dim" in lib.svgb_last_error()
    assert lib.svgb_qk_rope_bwd(A, A, A, A, A, A, 1, 2, 2, 100, 128, 100, 0, 0, None) < 0
    assert b"len_text" in lib.svgb_last_error()
    assert lib.svgb_qk_rope_bwd(A, A, None, A, A, A, 1, 2, 2, 100, 128, 0, 0, 0, None) < 0
    assert lib.svgb_qk_rope_bwd(A, A, A, A, A, A, 1, 2, 2, 100, 128, 0, 3, 0, None) < 0
    assert b"mode" in lib.svgb_last_error()

    def prep_bwd(D=128, norm=1, rope=1, rope_lo=0, rope_n=90, dbeta=A, ws_bytes=1 << 24, ts=384, g=A, x=A):
        return lib.svgb_qkv_prep_bwd(A, A, A, 100 * D, 3 * 100 * D, x, x, ts, 100 * ts, A, A, A, 1, 100, 3, D, 0,
                                     norm, g, g, C.c_float(1e-6), rope, A, A, rope_lo, rope_n, A, A, dbeta, dbeta, 0,
                                     A, ws_bytes, None)

    assert prep_bwd(D=96) < 0 and b"Unsupported head_dim" in lib.svgb_last_error()
    assert prep_bwd(rope_lo=20, rope_n=90) < 0 and b"token range" in lib.svgb_last_error()
    assert prep_bwd(rope=3) < 0 and b"rope 3 unknown" in lib.svgb_last_error()
    assert prep_bwd(norm=2, dbeta=None) < 0 and b"dbeta" in lib.svgb_last_error()
    assert prep_bwd(g=None) < 0 and b"gamma" in lib.svgb_last_error()
    assert prep_bwd(x=None) < 0 and b"q_in" in lib.svgb_last_error()
    assert prep_bwd(ts=380) < 0 and b"multiples of 8" in lib.svgb_last_error()
    assert prep_bwd(ws_bytes=16) < 0 and b"workspace too small" in lib.svgb_last_error()


# ---- raises under grad, before any device work (CPU tensors would fail the CUDA check otherwise) -----------------
def test_glue_raises_under_grad():
    from svgb200 import core

    x = torch.zeros(2, 3, 64, requires_grad=True)
    w, v = torch.ones(64), torch.zeros(2, 1, 64)
    calls = {
        "layernorm_modulate": lambda: core.layernorm_modulate(x, w, w, 1e-6, v, v),
        "rmsnorm_hidden": lambda: core.rmsnorm_hidden(x, w, 1e-6),
        "modulate_shift": lambda: core.modulate_shift(x, v, v),
        "gate_residual": lambda: core.gate_residual(x.detach(), x, v),
    }
    for name, fn in calls.items():
        with pytest.raises(core.SvgbError, match=f"{name} has no backward"):
            fn()
        with torch.no_grad(), pytest.raises(core.SvgbError, match="CUDA"):  # without grad: the call proceeds
            fn()


def test_prep_entry_raises_under_grad():
    from svgb200 import core

    qi = torch.zeros(1, 8, 128, dtype=torch.bfloat16, requires_grad=True)
    out = tuple(torch.zeros(1, 2, 8, 64, dtype=torch.bfloat16) for _ in range(3))
    with pytest.raises(core.SvgbError, match=r"out=\.\.\.\) has no backward"):
        core.qkv_prep(qi, qi, qi, 2, out=out)
    cos = torch.zeros(8, 64, requires_grad=True)
    with pytest.raises(core.SvgbError, match="cos / sin get no gradient"):
        core.qkv_prep(qi.detach(), qi.detach(), qi.detach(), 2, rope=1, cos=cos, sin=cos.detach())
    q = torch.zeros(1, 2, 8, 64, dtype=torch.bfloat16)
    with pytest.raises(core.SvgbError, match="cos / sin get no gradient"):
        core.qk_rope_(q, q, cos, cos.detach(), 0, core.ROPE_TXT_FIRST)
    with torch.no_grad(), pytest.raises(core.SvgbError, match="CUDA"):
        core.qkv_prep(qi, qi, qi, 2, out=out)


# ---- autograd wiring with float64 stand-ins ------------------------------------------------------------------------
@pytest.fixture
def stand_ins(monkeypatch):
    """Replace every kernel call of the prep chain by the float64 reference (forward) and its autograd (backward)."""
    import prep_fp64 as op
    from svgb200 import core

    calls = []

    def row_norm(x, gamma, beta, eps):
        x.copy_(op.rms_norm(x, gamma, eps) if beta is None else op.layer_norm(x, gamma, beta))

    @torch.enable_grad()  # a backward runs with grad mode off; the stand-in builds its own graph
    def row_norm_bwd(x, dy, gamma, eps, layer):
        x, gamma = x.detach().requires_grad_(), gamma.detach().requires_grad_()
        beta = torch.zeros_like(gamma, requires_grad=True)
        y = op.layer_norm(x, gamma, beta) if layer else op.rms_norm(x, gamma, eps)
        gs = torch.autograd.grad(y, (x, gamma, beta) if layer else (x, gamma), dy)
        return gs[0], gs[1], gs[2] if layer else None

    def rope(q, k, cos, sin, len_text, mode):
        for t, r in zip((q, k), op.qk_rope_inplace(q, k, cos, sin, len_text, mode)):
            t.copy_(r)

    @torch.enable_grad()
    def rope_bwd(dq, dk, cos, sin, len_text, mode):
        q, k = (torch.zeros_like(t, requires_grad=True) for t in (dq, dk))
        return torch.autograd.grad(op.qk_rope_inplace(q, k, cos, sin, len_text, mode), (q, k), (dq, dk))

    def qkv_prep(q_in, k_in, v_in, heads, *, out, out_row0=0, norm=0, gamma_q=None, gamma_k=None, beta_q=None,
                 beta_k=None, eps=1e-6, rope=0, cos=None, sin=None, rope_lo=0, rope_n=None):
        S = q_in.shape[1]
        n = cos.shape[0] if rope and rope_n is None else rope_n
        for o, r in zip(out, op.qkv_chain(q_in, k_in, v_in, heads, norm, gamma_q, gamma_k, beta_q, beta_k, eps, rope,
                                          cos, sin, rope_lo, n)):
            o[:, :, out_row0:out_row0 + S] = r
        return out

    @torch.enable_grad()
    def qkv_prep_bwd(dq, dk, dv, heads, S_in, *, q_in=None, k_in=None, out_row0=0, norm=0, gamma_q=None,
                     gamma_k=None, eps=1e-6, rope=0, cos=None, sin=None, rope_lo=0, rope_n=None):
        calls.append((out_row0, S_in, norm, rope))
        B, H, _, D = dq.shape
        shape = (B, S_in, H * D)
        xs = [(torch.zeros(shape, dtype=dq.dtype) if t is None else t.detach()).requires_grad_()
              for t in (q_in, k_in, None)]
        ws = [None if t is None else t.detach().requires_grad_() for t in (gamma_q, gamma_k)]
        n = cos.shape[0] if rope and rope_n is None else rope_n
        outs = op.qkv_chain(*xs, heads, norm, *ws, None, None, eps, rope, cos, sin, rope_lo, n)
        rows = slice(out_row0, out_row0 + S_in)
        leaves = xs + [w for w in ws if w is not None]
        gs = torch.autograd.grad(outs, leaves, (dq[:, :, rows], dk[:, :, rows], dv[:, :, rows]), allow_unused=True)
        return (*gs[:3], *(gs[3:5] if norm else (None, None)), None, None)

    monkeypatch.setattr(core, "_need_cuda", lambda *ts: None)
    monkeypatch.setattr(core, "_row_norm", row_norm)
    monkeypatch.setattr(core, "_row_norm_bwd", row_norm_bwd)
    monkeypatch.setattr(core, "_rope", rope)
    monkeypatch.setattr(core, "qk_rope_bwd", rope_bwd)
    monkeypatch.setattr(core, "_qkv_prep", qkv_prep)
    monkeypatch.setattr(core, "qkv_prep_bwd", qkv_prep_bwd)
    return calls


@pytest.mark.parametrize("layer", [False, True])
def test_row_norm_on_a_view_carries_the_history(stand_ins, layer):
    """The norm applied in place on .view(-1, D) of a non-leaf (the reference's call): the base tensor carries the
    norm's history (CopySlices), so the projection and the weights get the gradient of the norm, not of the
    identity."""
    import prep_fp64 as op
    from svgb200 import _kernels

    g = torch.Generator().manual_seed(1)
    w = torch.randn(2, 5, 3, 64, generator=g, dtype=torch.float64, requires_grad=True)
    gm = torch.randn(64, generator=g, dtype=torch.float64, requires_grad=True)
    bt = torch.randn(64, generator=g, dtype=torch.float64, requires_grad=True)
    gy = torch.randn(2, 3, 5, 64, generator=g, dtype=torch.float64)
    x = (w * 1).transpose(1, 2).contiguous()
    if layer:
        _kernels.layer_norm_forward(x.view(-1, 64), gm, bt)
    else:
        _kernels.rms_norm_forward(x.view(-1, 64), gm, 1e-5)
    x.backward(gy)
    leaves = [t.detach().requires_grad_() for t in (w, gm, bt)]
    xt = leaves[0].transpose(1, 2)
    ref = op.layer_norm(xt, leaves[1], leaves[2]) if layer else op.rms_norm(xt, leaves[1], 1e-5)
    ref.backward(gy)
    assert torch.allclose(w.grad, leaves[0].grad) and torch.allclose(gm.grad, leaves[1].grad)
    if layer:
        assert torch.allclose(bt.grad, leaves[2].grad)
    else:
        assert bt.grad is None


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_rope_in_place_marks_q_and_k_dirty(stand_ins, mode):
    import prep_fp64 as op
    from svgb200 import core

    g = torch.Generator().manual_seed(mode)
    q0 = torch.randn(1, 4, 20, 64, generator=g, dtype=torch.float64, requires_grad=True)
    k0 = torch.randn(1, 2, 20, 64, generator=g, dtype=torch.float64, requires_grad=True)
    width = 32 if mode == 2 else 64
    cos, sin = torch.randn(15, width, generator=g), torch.randn(15, width, generator=g)
    q, k = q0 * 1, k0 * 1
    rq, rk = core.qk_rope_(q, k, cos, sin, 5, mode)
    assert rq is q and rk is k and q.grad_fn is not None
    gq, gk = torch.randn_like(q), torch.randn_like(k)
    torch.autograd.backward((q, k), (gq, gk))
    lq, lk = (t.detach().requires_grad_() for t in (q0, k0))
    torch.autograd.backward(op.qk_rope_inplace(lq, lk, cos, sin, 5, mode), (gq, gk))
    assert torch.allclose(q0.grad, lq.grad) and torch.allclose(k0.grad, lk.grad)


def test_leaf_requiring_grad_gets_the_in_place_error(stand_ins):
    from svgb200 import core

    x = torch.randn(4, 64, dtype=torch.float64, requires_grad=True)
    with pytest.raises(RuntimeError, match="leaf"):
        core.rms_norm_(x, torch.ones(64, dtype=torch.float64))


@pytest.mark.parametrize("prompt_norm", [True, False])
def test_double_block_reads_each_streams_rows(stand_ins, prompt_norm):
    """hunyuan_double_block_qkv under grad: one node, whose backward makes one call per stream -- the video stream on
    rows [0, Sv), the prompt stream on rows [Sv, Sv + St) -- and the gradients equal float64 autograd through
    torch.cat of the two float64 reference chains."""
    import prep_fp64 as op
    from svgb200 import prep

    B, Sv, St, H, D = 2, 9, 4, 2, 64
    g = torch.Generator().manual_seed(7)
    f64 = dict(generator=g, dtype=torch.float64)
    vid = [torch.randn(B, Sv, H * D, **f64, requires_grad=True) for _ in range(3)]
    txt = [torch.randn(B, St, H * D, **f64, requires_grad=True) for _ in range(3)]
    w = [torch.randn(D, **f64, requires_grad=True) for _ in range(4)]
    if not prompt_norm:
        w[2] = w[3] = None
    cos, sin = torch.randn(Sv, D, generator=g), torch.randn(Sv, D, generator=g)
    outs = prep.hunyuan_double_block_qkv(*vid, *txt, H, w[0], w[1], w[2], w[3], 1e-6, cos, sin)
    grads = [torch.randn(B, H, Sv + St, D, **f64) for _ in range(3)]
    torch.autograd.backward(outs, grads)
    assert stand_ins == [(0, Sv, 1, 1), (Sv, St, 1 if prompt_norm else 0, 0)]

    leaves = [t.detach().requires_grad_() for t in vid + txt]
    wl = [None if t is None else t.detach().requires_grad_() for t in w]
    a = op.qkv_chain(*leaves[:3], H, 1, wl[0], wl[1], None, None, 1e-6, 1, cos, sin, 0, Sv)
    b = op.qkv_chain(*leaves[3:], H, 1 if prompt_norm else 0, wl[2], wl[3], None, None, 1e-6, 0, None, None, 0, 0)
    torch.autograd.backward([torch.cat([x, y], 2) for x, y in zip(a, b)], grads)
    for t, r in zip(vid + txt, leaves):
        assert torch.allclose(t.grad, r.grad)
    for t, r in zip(w, wl):
        if t is not None:
            assert torch.allclose(t.grad, r.grad)


@pytest.mark.parametrize("norm, rope", [(0, 0), (1, 1), (2, 1), (3, 2), (1, 2), (2, 0)])
def test_fp64_reference_restates_the_oracle(norm, rope):
    """prep_fp64 (the gradient reference) is oracle.prep's chain without the roundings: on bf16 inputs the oracle
    (fp32, rounded like the kernels) and prep_fp64 rounded once to bf16 differ by at most a few bf16 units."""
    import prep_fp64
    from oracle import prep as op

    B, S, H, D, txt = 2, 37, 3, 64, 5
    g = torch.Generator().manual_seed(norm * 10 + rope)
    qi, ki, vi = (torch.randn(B, S, H * D, generator=g).bfloat16() for _ in range(3))
    gw = H * D if norm == 3 else D
    gq, gk, bq, bk = ((1 + 0.3 * torch.randn(gw, generator=g)).bfloat16() for _ in range(4))
    width = D // 2 if rope == 2 else D
    cos, sin = torch.randn(S - txt, width, generator=g), torch.randn(S - txt, width, generator=g)
    args = (H, norm, gq, gk, bq, bk, 1e-6, rope, cos, sin, txt, S - txt)
    for a, b in zip(op.qkv_chain(qi, ki, vi, *args), prep_fp64.qkv_chain(qi, ki, vi, *args)):
        assert b.dtype == torch.float64
        torch.testing.assert_close(a.float(), b.bfloat16().float(), rtol=3e-2, atol=3e-2)
