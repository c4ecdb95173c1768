"""Fused pre-attention chain: the reference's per-layer sequence
    get_transpose_qkv -> get_qk_norm -> get_rotary_emb (-> get_encoder_condition_and_concat)
(svg/models/hyvideo/attention.py:253-301, svg/models/wan/attention.py:100-135, svg/models/cog/attention.py:20-35)
as single passes over the projection outputs.  Each helper returns (q, k, v) in the [B, H, S, D] layout the
attention core consumes.  Under grad each helper is differentiable in its projection outputs and norm weights
(core._QkvPrep; the double block records both streams in one node).
"""
from __future__ import annotations

from . import core


def hunyuan_single_block_qkv(query, key, value, heads, norm_q_weight, norm_k_weight, eps, cos, sin, txt_len):
    """Single-stream block: hidden = cat(video, text) was projected as one sequence; QK RMSNorm on every row,
    RoPE on all but the last `txt_len` rows (apply_qk_rope_single, hyvideo/attention.py:170-178)."""
    S = query.shape[1]
    return core.qkv_prep(query, key, value, heads, norm=core.NORM_RMS_HEAD, gamma_q=norm_q_weight,
                         gamma_k=norm_k_weight, eps=eps, rope=1, cos=cos, sin=sin, rope_lo=0, rope_n=S - txt_len)


def hunyuan_double_block_qkv(query, key, value, enc_query, enc_key, enc_value, heads, norm_q_weight, norm_k_weight,
                             norm_added_q_weight, norm_added_k_weight, eps, cos, sin):
    """Dual-stream block: the video stream is normed + rotated, the prompt stream has its own norms and no RoPE,
    then torch.cat([video, prompt], dim=2) (hyvideo/attention.py:283-301) — here both streams are written
    straight into one [B, H, S_video + S_text, D] tensor."""
    Sv, St = query.shape[1], enc_query.shape[1]
    video = dict(out_row0=0, norm=core.NORM_RMS_HEAD, gamma_q=norm_q_weight, gamma_k=norm_k_weight, eps=eps, rope=1,
                 cos=cos, sin=sin, rope_lo=0, rope_n=Sv)
    prompt = dict(out_row0=Sv, norm=core.NORM_RMS_HEAD if norm_added_q_weight is not None else core.NORM_NONE,
                  gamma_q=norm_added_q_weight, gamma_k=norm_added_k_weight, eps=eps)
    return core.qkv_prep_streams([((query, key, value), video), ((enc_query, enc_key, enc_value), prompt)], heads,
                                 Sv + St)


def wan_qkv(query, key, value, heads, norm_q_weight, norm_k_weight, eps, freqs_real, freqs_imag):
    """Wan self-attention: RMSNorm over the full hidden row (triton_rmsnorm_forward, wan/attention.py:107-120),
    head split, complex RoPE on every row (wan/attention.py:44-48)."""
    return core.qkv_prep(query, key, value, heads, norm=core.NORM_RMS_HIDDEN, gamma_q=norm_q_weight,
                         gamma_k=norm_k_weight, eps=eps, rope=2, cos=freqs_real, sin=freqs_imag, rope_lo=0,
                         rope_n=query.shape[1])


def cog_qkv(query, key, value, heads, norm_q_weight, norm_q_bias, norm_k_weight, norm_k_bias, cos, sin,
            text_seq_length: int):
    """CogVideoX: per-head LayerNorm on Q/K (cog/attention.py:24-29), RoPE on all but the FIRST
    `text_seq_length` rows (cog/attention.py:31-34)."""
    S = query.shape[1]
    norm = core.NORM_LAYER if norm_q_weight is not None else core.NORM_NONE
    return core.qkv_prep(query, key, value, heads, norm=norm, gamma_q=norm_q_weight, gamma_k=norm_k_weight,
                         beta_q=norm_q_bias, beta_k=norm_k_bias, rope=1, cos=cos, sin=sin, rope_lo=text_seq_length,
                         rope_n=S - text_seq_length)
