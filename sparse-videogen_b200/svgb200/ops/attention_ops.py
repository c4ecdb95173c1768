"""Mirror of svg/kernels/ops/attention_ops.py: BSR masks (indptr, indices, (R, C)) + the HunyuanVideo
text-FIRST sparse forward.  The reference runs four FlashInfer calls and merges LSE states (:140-197);
here text and video live in one variable-block map (text block x everything, video x text), one launch."""
from __future__ import annotations

import weakref
from dataclasses import dataclass
from typing import Optional, Tuple

import numpy as np
import torch

from .. import core

__all__ = ["_gen_temporal_mask", "_gen_spatial_mask", "FAMetadata", "init_sparse_attn", "sparse_attn_forward",
           "bsr_to_plan"]


def _bsr_from_keep(keep: np.ndarray, block_size, device):
    indptr = np.concatenate([[0], np.cumsum(keep.sum(1))]).astype(np.int32)
    cols = np.nonzero(keep)[1].astype(np.int32)
    cols = np.concatenate([cols, np.zeros(256, np.int32)])  # the reference pads 256 zeros (:52,:101)
    dev = device if device is not None else ("cuda" if torch.cuda.is_available() else "cpu")
    return torch.from_numpy(indptr).to(dev), torch.from_numpy(cols).to(dev), block_size


def _gen_temporal_mask(num_frames: int, num_tokens_per_frame: int, multiplier: float, device=None):
    """attention_ops.py:9-55: block = P/10, keep iff |centre_i - centre_j| < mul*P."""
    assert num_tokens_per_frame % 10 == 0
    bs = num_tokens_per_frame // 10
    assert (num_tokens_per_frame * num_frames) % bs == 0
    n = num_frames * num_tokens_per_frame // bs
    c = np.arange(n) * bs + bs // 2
    keep = np.abs(c[:, None] - c[None, :]) < multiplier * num_tokens_per_frame
    return _bsr_from_keep(keep, (bs, bs), device)


def _gen_spatial_mask(num_frames: int, num_tokens_per_frame: int, multiplier: int, device=None):
    """attention_ops.py:58-104: frame granular, keep iff |i-j| <= mul or j == 0."""
    assert multiplier >= 0, "width of sliding window must be at least one frame"
    assert num_frames > 0
    i = np.arange(num_frames)
    keep = (np.abs(i[:, None] - i[None, :]) <= multiplier) | (i[None, :] == 0)
    return _bsr_from_keep(keep, (num_tokens_per_frame, num_tokens_per_frame), device)


@dataclass
class FAMetadata:
    len_text_promt: int
    num_frames: int
    num_tokens_per_frame: int
    temporal_mask_metadata: Tuple[torch.Tensor, torch.Tensor, Tuple[int, int]]
    spatial_mask_metadata: Tuple[torch.Tensor, torch.Tensor, Tuple[int, int]]
    workspace: Optional[torch.Tensor] = None  # unused: plans own their workspace


def init_sparse_attn(len_text_prompt, num_frames, num_tokens_per_frame, temporal_multiplier, spatial_multiplier):
    """attention_ops.py:118-137."""
    return FAMetadata(len_text_prompt, num_frames, num_tokens_per_frame,
                      _gen_temporal_mask(num_frames, num_tokens_per_frame, temporal_multiplier),
                      _gen_spatial_mask(num_frames, num_tokens_per_frame, spatial_multiplier))


_plan_cache: dict = {}


def bsr_to_plan(indptr, indices, block_size, video_len, text_len, device) -> core.AttnPlan:
    """BSR over the video part (+ an all-to-all text prefix of `text_len`) -> one shared plan."""
    # cache per live BSR tensor object (a data_ptr can be recycled by the allocator: key on identity and
    # verify through a weak reference)
    key = (id(indptr), id(indices), tuple(block_size), video_len, text_len, str(device))
    hit = _plan_cache.get(key)
    if hit is not None and hit[0]() is indptr and hit[1]() is indices:
        return hit[2]
    R, C = block_size
    MB, NB = video_len // R, video_len // C
    ip = indptr.to(device=device, dtype=torch.long)
    nnz_rows = torch.repeat_interleave(torch.arange(MB, device=device), ip[1:] - ip[:-1])
    cols = indices.to(device=device, dtype=torch.long)[: nnz_rows.numel()]
    t = 1 if text_len > 0 else 0
    bm = torch.zeros(1, MB + t, NB + t, dtype=torch.bool, device=device)
    bm[0, nnz_rows + t, cols + t] = True
    row = torch.full((1, MB + t), R, dtype=torch.int32, device=device)
    col = torch.full((1, NB + t), C, dtype=torch.int32, device=device)
    if t:
        bm[0, 0, :] = True   # text rows see everything (o_text, :189-195)
        bm[0, :, 0] = True   # video rows see the text columns (o_image_r, :180-186)
        row[0, 0] = text_len
        col[0, 0] = text_len
    plan = core.plan_varblock(bm, row, col, video_len + text_len)  # owns its workspace: safe to cache
    plan.desc.items_stride = 0   # one map for every head: share the plan (svgb200.h, svgb_plan)
    _plan_cache[key] = (weakref.ref(indptr), weakref.ref(indices), plan)
    return plan


def sparse_attn_forward(q, k, v, metadata: FAMetadata, sparse_pattern: str = "temporal"):
    """attention_ops.py:140-197.  q,k,v [seq_len, H, D], text FIRST."""
    assert sparse_pattern in ["temporal", "spatial"]
    md = metadata.temporal_mask_metadata if sparse_pattern == "temporal" else metadata.spatial_mask_metadata
    indptr, indices, block_size = md
    T = metadata.len_text_promt
    plan = bsr_to_plan(indptr, indices, block_size, q.shape[0] - T, T, q.device)
    return core.attention(q, k, v, plan, layout="shd")
