"""Float64 restatement of oracle.prep's pre-attention chain, the reference for the chain's gradients (test helper).

Same functions and arguments as oracle.prep (rms_norm, layer_norm, rope_interleave, rope_complex, qk_rope_inplace,
qkv_chain), computed in float64 with no intermediate rounding and returned in float64, so float64 autograd through
them gives the exact-math gradient.  oracle.prep computes in fp32 and rounds to the input dtype like the kernels;
tests/test_prep_bwd_cpu.py checks that the two agree on 16-bit inputs.
"""
from __future__ import annotations

import torch


def rms_norm(x, gamma, eps):
    x = x.double()
    return x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps) * gamma.double()


def layer_norm(x, gamma, beta, eps=1e-5):
    x = x.double()
    mean = x.mean(-1, keepdim=True)
    var = (x - mean).pow(2).mean(-1, keepdim=True)
    return (x - mean) * torch.rsqrt(var + eps) * gamma.double() + beta.double()


def rope_interleave(x, cos, sin):
    """out[e] = x[e]*cos[e] + (e even ? -x[e+1] : x[e-1])*sin[e] on [..., S, D], cos/sin [S, D]."""
    x = x.double()
    rot = torch.stack([-x[..., 1::2], x[..., 0::2]], dim=-1).flatten(-2)
    return x * cos.double() + rot * sin.double()


def rope_complex(x, real, imag):
    """complex pairs (a, b) -> (a c - b s, b c + a s) on [..., S, D], real/imag [S, D/2]."""
    x = x.double()
    a, b = x[..., 0::2], x[..., 1::2]
    c, s = real.double(), imag.double()
    return torch.stack([a * c - b * s, b * c + a * s], dim=-1).flatten(-2)


def qk_rope_inplace(q, k, cos, sin, len_text, mode):
    """mode 0: skip the first len_text rows; 1: skip the last; 2: complex, skip the first.  Returns new tensors."""
    S = q.shape[2]
    lo, hi = (0, S - len_text) if mode == 1 else (len_text, S)
    fn = rope_complex if mode == 2 else rope_interleave
    return [torch.cat([t[:, :, :lo].double(), fn(t[:, :, lo:hi], cos, sin), t[:, :, hi:].double()], 2) for t in (q, k)]


def qkv_chain(q_in, k_in, v_in, heads, norm, gamma_q, gamma_k, beta_q, beta_k, eps, rope, cos, sin, rope_lo, rope_n):
    """[B,S,H*D] x3 -> (q, k, v) [B,H,S,D]: optional full-hidden RMS (norm 3), head split, per-head RMS (1) or
    LayerNorm (2, eps 1e-5), RoPE (1 interleaved, 2 complex) on rows [rope_lo, rope_lo + rope_n)."""
    B, S, HD = q_in.shape
    D = HD // heads

    def split(t):
        return t.double().reshape(B, S, heads, D).transpose(1, 2)

    q, k = q_in, k_in
    if norm == 3:
        q, k = rms_norm(q, gamma_q, eps), rms_norm(k, gamma_k, eps)
    q, k, v = split(q), split(k), split(v_in)
    if norm == 1:
        q, k = rms_norm(q, gamma_q, eps), rms_norm(k, gamma_k, eps)
    elif norm == 2:
        q, k = layer_norm(q, gamma_q, beta_q), layer_norm(k, gamma_k, beta_k)
    if rope:
        fn = rope_complex if rope == 2 else rope_interleave
        lo, hi = rope_lo, rope_lo + rope_n
        q, k = (torch.cat([t[:, :, :lo], fn(t[:, :, lo:hi], cos, sin), t[:, :, hi:]], 2) for t in (q, k))
    return q, k, v
