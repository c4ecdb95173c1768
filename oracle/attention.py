"""Oracle: masked / block-sparse attention and the mask generators.  TEST INFRASTRUCTURE ONLY.

Restates (reference paths relative to /root/reference):
  ref_torch_attn_impl            svg/kernels/test/test_sparse_attn.py:109-157
  gen_mask_block2element         svg/kernels/test/test_sparse_attn.py:66-87
  _block_mask_to_element_mask    svg/kernels/test/test_sparse_attn_dyn_blk_wan.py:47-57
  dynamic_block_sparse_fwd_torch svg/kmeans_utils.py:902-995
  temporal_mask_mod (HY/WAN/COG) svg/models/{hyvideo,wan,cog}/utils.py:20-44 / 25-41 / 30-46
  sparsity_to_width              svg/models/hyvideo/utils.py:142-151
  get_attention_mask             svg/models/hyvideo/utils.py:47-93, wan/utils.py:63-110
  sample_mse                     svg/models/hyvideo/attention.py:375-399
  ref_gen_spatial/temporal_mask  svg/kernels/test/test_sparse_attn.py:20-63,
                                 svg/kernels/ops/attention_ops_wan.py:96-129
"""
from __future__ import annotations

import math
from math import ceil, floor

import numpy as np
import torch


# --------------------------------------------------------------------------------------------
# naive attention (the "naive torch-matmul attention" of BASELINE config 1)
# --------------------------------------------------------------------------------------------
def ref_torch_attn_impl(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, mask: torch.Tensor | None):
    """q,k,v: [S, H, D]; mask: [S, S] (nonzero = attend) or None.  fp32 math on CPU.

    Follows test_sparse_attn.py:109-157: per head  QK^T / sqrt(d) -> masked_fill(-inf) -> softmax
    -> @V.  A fully masked row yields NaN there; we return 0 for such rows (reference engine
    behaviour, SURVEY Appendix B #4)."""
    S, H, D = q.shape
    out = torch.empty(S, H, D, dtype=torch.float32)
    scale = D ** 0.5
    for h in range(H):
        qh = q[:, h, :].float()
        kh = k[:, h, :].float()
        vh = v[:, h, :].float()
        s = qh @ kh.T / scale
        if mask is not None:
            s = s.masked_fill(mask == 0, float("-inf"))
        w = torch.softmax(s, dim=-1)
        w = torch.nan_to_num(w, nan=0.0)
        out[:, h, :] = w @ vh
    return out


def masked_attention_bhsd(q, k, v, mask_fn, row_chunk: int = 1024, sm_scale=None, return_lse: bool = False,
                          dtype=torch.float32):
    """q,k,v: [BH, S, D]; mask_fn(q_idx[Sq,1], kv_idx[1,S]) -> bool[Sq,S] or None.
    Row-chunked so it scales to long S without materialising S x S.  sm_scale defaults to D^-1/2; `dtype` is the
    compute precision (torch.float64 for LSE checks).  return_lse: also the natural-log log-sum-exp of the scaled,
    masked scores [BH, S] (-inf for rows without a key)."""
    BH, S, D = q.shape
    out = torch.empty(BH, S, D, dtype=dtype)
    lse = torch.empty(BH, S, dtype=dtype)
    scale = D ** -0.5 if sm_scale is None else sm_scale
    kv_idx = torch.arange(S).view(1, S)
    for h in range(BH):
        kh = k[h].to(dtype)
        vh = v[h].to(dtype)
        for r0 in range(0, S, row_chunk):
            r1 = min(S, r0 + row_chunk)
            s = (q[h, r0:r1].to(dtype) @ kh.T) * scale
            if mask_fn is not None:
                m = mask_fn(torch.arange(r0, r1).view(-1, 1), kv_idx)
                s = s.masked_fill(~m, float("-inf"))
            w = torch.nan_to_num(torch.softmax(s, dim=-1), nan=0.0)
            out[h, r0:r1] = w @ vh
            lse[h, r0:r1] = torch.logsumexp(s, dim=-1)
    return (out, lse) if return_lse else out


def gen_mask_block2element(block_mask: np.ndarray, block_size, len_text_prompt: int) -> torch.Tensor:
    """test_sparse_attn.py:66-87 (text FIRST: prepend all-ones text rows / columns)."""
    bm = (block_mask >= 0).astype(np.int32)
    bm = np.repeat(bm, block_size[1], axis=1)
    bm = np.repeat(bm, block_size[0], axis=0)
    bm = np.concatenate([np.ones((bm.shape[0], len_text_prompt), dtype=np.int32), bm], axis=1)
    bm = np.concatenate([np.ones((len_text_prompt, bm.shape[1]), dtype=np.int32), bm], axis=0)
    return torch.from_numpy(bm.astype(np.bool_))


def block_mask_to_element_mask(block_mask_map: torch.Tensor, block_row_sz, block_col_sz) -> torch.Tensor:
    """test_sparse_attn_dyn_blk_wan.py:47-57."""
    r = torch.as_tensor(block_row_sz, dtype=torch.long)
    c = torch.as_tensor(block_col_sz, dtype=torch.long)
    rows = torch.repeat_interleave(block_mask_map.bool(), r, dim=0)
    return torch.repeat_interleave(rows, c, dim=1)


def dynamic_block_sparse_fwd(q, k, v, dynamic_map, qc_size, kc_size, sm_scale=None, return_lse: bool = False,
                             dtype=torch.float32):
    """Variable-block sparse attention, [B,H,S,D].  Same result as kmeans_utils.py:902-995 (online
    softmax over selected blocks == masked softmax over the expanded element mask; rows with no
    reachable key -> 0, :993).  Computed as masked softmax in fp32 (or `dtype`).  return_lse: also the
    natural-log log-sum-exp of the scaled, masked scores [B,H,S] (-inf for rows without a key)."""
    B, H, S, D = q.shape
    out = torch.zeros(B, H, S, D, dtype=dtype)
    lse = torch.empty(B, H, S, dtype=dtype)
    scale = D ** -0.5 if sm_scale is None else sm_scale
    for b in range(B):
        for h in range(H):
            em = block_mask_to_element_mask(dynamic_map[b, h], qc_size[b, h], kc_size[b, h])
            s = (q[b, h].to(dtype) @ k[b, h].to(dtype).T) * scale
            s = s.masked_fill(~em, float("-inf"))
            w = torch.nan_to_num(torch.softmax(s, dim=-1), nan=0.0)
            out[b, h] = w @ v[b, h].to(dtype)
            lse[b, h] = torch.logsumexp(s, dim=-1)
    return (out, lse) if return_lse else out


# --------------------------------------------------------------------------------------------
# SVG1 executed masks (element-exact mask_mods)
# --------------------------------------------------------------------------------------------
def sparsity_to_width(sparsity, context_length, num_frame, frame_size):
    """hyvideo/utils.py:142-151 (identical in wan/cog)."""
    seq_len = context_length + num_frame * frame_size
    total_elements = seq_len ** 2
    sparsity = (sparsity * total_elements - 2 * seq_len * context_length) / total_elements
    width = seq_len * (1 - math.sqrt(1 - sparsity))
    return width / frame_size


def hy_band_width(mul, token_per_frame):
    """hyvideo/utils.py:24-25,33: floor(mul*P/128)*128."""
    return floor(mul * token_per_frame / 128) * 128


def wan_band_width(mul, token_per_frame):
    """wan/utils.py:29-33: ceil(mul*P/128)*128."""
    return ceil(mul * token_per_frame / 128) * 128


def hy_mask_mod(context_length, prompt_length, num_frames, token_per_frame, mul):
    """hyvideo/utils.py:20-44."""
    real_length = num_frames * token_per_frame + prompt_length
    W = hy_band_width(mul, token_per_frame)
    V = num_frames * token_per_frame

    def mod(q_idx, kv_idx):
        real = (kv_idx < real_length) & (q_idx < real_length)
        fake = (kv_idx >= real_length) & (q_idx >= real_length)
        band = (q_idx - kv_idx).abs() < W
        text_col = (V <= kv_idx) & (kv_idx < real_length)
        text_row = (V <= q_idx) & (q_idx < real_length)
        return (real & (band | text_col | text_row)) | fake

    return mod


def wan_mask_mod(num_frames, token_per_frame, mul):
    """wan/utils.py:25-41."""
    W = wan_band_width(mul, token_per_frame)

    def mod(q_idx, kv_idx):
        return (kv_idx < token_per_frame) | ((q_idx - kv_idx).abs() <= W)

    return mod


def cog_mask_mod(prompt_length, num_frames, token_per_frame, mul, attn_sink=False):
    """cog/utils.py:30-46."""
    W = hy_band_width(mul, token_per_frame)
    first_col = prompt_length + token_per_frame if attn_sink else prompt_length

    def mod(q_idx, kv_idx):
        return (kv_idx < first_col) | (q_idx < prompt_length) | ((q_idx - kv_idx).abs() < W)

    return mod


def generic_mask_fn(mode, m0, m1, m2):
    """The engine's own parametrisation (include/svgb200.h SVGB_MASK_*), restated for tests."""

    def mod(q_idx, kv_idx):
        d = (q_idx - kv_idx).abs()
        if mode == 1:
            real = (q_idx < m1) & (kv_idx < m1)
            fake = (q_idx >= m1) & (kv_idx >= m1)
            return (real & ((d < m2) | (kv_idx >= m0) | (q_idx >= m0))) | fake
        if mode == 2:
            return (kv_idx < m0) | (d <= m2)
        if mode == 3:
            return (kv_idx < m0) | (q_idx < m1) | (d < m2)
        return torch.ones_like(d, dtype=torch.bool)

    return mod


# --------------------------------------------------------------------------------------------
# SVG1 profiling masks + sample_mse
# --------------------------------------------------------------------------------------------
def profiling_mask_rows(mask_name, rows, layout, context_length, num_frame, frame_size, thres=None):
    """Rows `rows` of get_attention_mask(...) evaluated analytically -> bool [len(rows), S].

    hyvideo/utils.py:47-93 (layout 'hy': text last, band threshold (1.5*P)//128 blocks),
    wan/utils.py:63-110 (layout 'wan': no text, first-frame sink, threshold (2*P)//128).
    The reference paints 128-token blocks with |bi-bj| < thres for the spatial mask; the temporal
    mask is the same picture pushed through reshape(P,F,P,F).permute(1,0,3,2), i.e.
        temporal[f*P+p, f2*P+p2] = picture[p*F+f, p2*F+f2].
    For 'wan' the first-frame sink columns are painted BEFORE that permutation (wan/utils.py:95-108)
    so they are permuted too.  `thres` overrides the band threshold (blocks)."""
    F_, P_ = num_frame, frame_size
    V = F_ * P_
    S = context_length + V
    if thres is None:
        thres = (frame_size * (1.5 if layout == "hy" else 2)) // 128
    kv = torch.arange(V)
    ki = kv if mask_name == "spatial" else (kv % P_) * F_ + kv // P_
    out = torch.zeros(len(rows), S, dtype=torch.bool)
    for n, r in enumerate([int(x) for x in rows]):
        if layout == "hy" and r >= V:
            out[n, :] = True  # text rows see everything (utils.py:66,90)
            continue
        qi = r if mask_name == "spatial" else (r % P_) * F_ + r // P_
        band = (qi // 128 - ki // 128).abs() < thres
        if layout == "wan":
            band = band | (ki < P_)
        out[n, :V] = band
        if layout == "hy":
            out[n, V:] = True  # text columns (utils.py:67,91)
    return out


def profiling_mask_rows_cog(mask_name, rows, context_length, num_frame, frame_size, thres=None):
    """Rows of the CogVideoX profiling masks (text FIRST), svg/models/cog/utils.py:61-88, analytically.

    spatial : text rows / columns all-ones (:66-67); the 128-token block band |bi-bj| < (1.5*P)//128 is painted in
              ABSOLUTE coordinates from row / column 0 for blocks 0..ceil(F*P/128)-1 (:68-74, not offset by the text);
    temporal: the same band picture pushed through reshape(P,F,P,F).permute(1,0,3,2) on the video x video part only
              (:76-86); text rows and text columns stay ZERO (a sampled text row is fully masked).
    `thres` overrides the band threshold (blocks)."""
    F_, P_, ctx = num_frame, frame_size, context_length
    V = F_ * P_
    S = ctx + V
    if thres is None:
        thres = (frame_size * 1.5) // 128
    lim = math.ceil(V / 128) * 128
    kv = torch.arange(S)
    out = torch.zeros(len(rows), S, dtype=torch.bool)
    for n, r in enumerate([int(x) for x in rows]):
        if mask_name == "spatial":
            band = ((r // 128 - kv // 128).abs() < thres) & (kv < lim) & (r < lim)
            out[n] = band | (kv < ctx) | (r < ctx)
        else:
            if r < ctx:
                continue
            qv = r - ctx
            kvv = kv[ctx:] - ctx
            qi = (qv % P_) * F_ + qv // P_
            ki = (kvv % P_) * F_ + kvv // P_
            out[n, ctx:] = (qi // 128 - ki // 128).abs() < thres
    return out


def sample_mse(q, k, v, sampled_rows, masks_rows):
    """hyvideo/attention.py:375-399 in fp32.  q,k,v [cfg,H,S,D]; masks_rows: list of bool
    [n_rows, S] (rows of the profiling masks at sampled_rows) -> fp32 [n_masks, cfg, H]."""
    cfg, H, S, D = q.shape
    sq = q[:, :, sampled_rows, :].float()
    scores = sq @ k.float().transpose(-2, -1) / (D ** 0.5)
    golden = torch.softmax(scores, dim=-1) @ v.float()
    out = torch.zeros(len(masks_rows), cfg, H)
    for i, m in enumerate(masks_rows):
        s = scores.masked_fill(~m.view(1, 1, *m.shape), float("-inf"))
        hs = torch.softmax(s, dim=-1) @ v.float()
        out[i] = ((hs - golden) ** 2).mean(dim=(2, 3))
    return out


# --------------------------------------------------------------------------------------------
# ops-API BSR masks
# --------------------------------------------------------------------------------------------
def ref_gen_temporal_mask(num_frames, num_tokens_per_frame, multiplier):
    """test_sparse_attn.py:20-42 (block = P/10, centre distance < mul*P)."""
    assert num_tokens_per_frame % 10 == 0
    bs = num_tokens_per_frame // 10
    n = num_frames * num_tokens_per_frame // bs
    i = np.arange(n)[:, None] * bs + bs // 2
    j = np.arange(n)[None, :] * bs + bs // 2
    keep = np.abs(i - j) < multiplier * num_tokens_per_frame
    return np.where(keep, np.arange(n)[None, :], -1), (bs, bs)


def ref_gen_spatial_mask(num_frames, num_tokens_per_frame, multiplier):
    """test_sparse_attn.py:45-63 (frame granular, |i-j| <= mul or j == 0)."""
    i = np.arange(num_frames)[:, None]
    j = np.arange(num_frames)[None, :]
    keep = (np.abs(i - j) <= multiplier) | (j == 0)
    return np.where(keep, j, -1), (num_tokens_per_frame, num_tokens_per_frame)


def get_factor(num_tokens_per_frame):
    """wan/utils.py:113-127: largest divisor of P below 256."""
    for f in range(255, 0, -1):
        if num_tokens_per_frame % f == 0:
            return f
    raise ValueError


def ref_gen_temporal_mask_wan(num_frames, num_tokens_per_frame, multiplier, first_frame=True):
    """first_frame=True: svg/models/wan/utils.py:130-185 (band + every block whose centre lies in the first frame,
    :168); first_frame=False: svg/kernels/ops/attention_ops_wan.py:48-129 (band only)."""
    bs = get_factor(num_tokens_per_frame)
    n = num_frames * num_tokens_per_frame // bs
    i = np.arange(n)[:, None] * bs + bs // 2
    j = np.arange(n)[None, :] * bs + bs // 2
    keep = np.abs(i - j) < multiplier * num_tokens_per_frame
    if first_frame:
        keep = keep | (j <= num_tokens_per_frame)
    return np.where(keep, np.arange(n)[None, :], -1), (bs, bs)
