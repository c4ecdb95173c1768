"""Mirror of svg/kernels/ops/attention_ops_wan.py and the BSR helpers of svg/models/wan/utils.py."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional, Tuple

import numpy as np
import torch

from .. import core
from .attention_ops import _bsr_from_keep, bsr_to_plan

__all__ = ["get_factor", "gen_temporal_mask", "WanFAMetadata", "wan_sparse_attn_forward",
           "flashinfer_sparse_attn_forward"]


def get_factor(num_frames: int, num_tokens_per_frame: int) -> int:
    """wan/utils.py:113-127: the largest divisor of P below 256."""
    for f in range(255, 0, -1):
        if num_tokens_per_frame % f == 0:
            return f
    raise ValueError(f"No factor found for {num_frames} * {num_tokens_per_frame}")


def gen_temporal_mask(num_frames: int, num_tokens_per_frame: int, multiplier: float, device=None,
                      first_frame: bool = False):
    """svg/kernels/ops/attention_ops_wan.py:48-93: the diagonal band only (block centres closer than mul*P).
    first_frame=True is the variant of svg/models/wan/utils.py:130-185, which also keeps every block whose centre lies
    in the first frame (`elif col_token_idx <= num_tokens_per_frame`, wan/utils.py:168) -- exported under the
    reference's name as svgb200.models.wan.gen_temporal_mask."""
    bs = get_factor(num_frames, num_tokens_per_frame)
    assert (num_tokens_per_frame * num_frames) % bs == 0
    n = num_frames * num_tokens_per_frame // bs
    c = np.arange(n) * bs + bs // 2
    keep = np.abs(c[:, None] - c[None, :]) < multiplier * num_tokens_per_frame
    if first_frame:
        keep = keep | (c[None, :] <= num_tokens_per_frame)
    return _bsr_from_keep(keep, (bs, bs), device)


@dataclass
class WanFAMetadata:
    num_frames: int
    num_tokens_per_frame: int
    temporal_mask_metadata: Tuple[torch.Tensor, torch.Tensor, Tuple[int, int]]
    workspace: Optional[torch.Tensor] = None


def wan_sparse_attn_forward(q, k, v, metadata: WanFAMetadata):
    """attention_ops_wan.py:141-181.  q,k,v [seq_len, H, D] (video only)."""
    indptr, indices, block_size = metadata.temporal_mask_metadata
    assert q.shape[0] % block_size[0] == 0, f"Query length {q.shape[0]} % block_size {block_size[0]} != 0"
    assert k.shape[0] % block_size[1] == 0, f"Key length {k.shape[0]} % block_size {block_size[1]} != 0"
    assert k.shape[0] == v.shape[0], f"Key length {k.shape[0]} != Value length {v.shape[0]}"
    plan = bsr_to_plan(indptr, indices, block_size, q.shape[0], 0, q.device)
    return core.attention(q, k, v, plan, layout="shd")


def flashinfer_sparse_attn_forward(q, k, v, temporal_mask_metadata):
    """wan/utils.py:188-238.  q,k,v [cfg, H, S, D] -> [cfg, H, S, D]; no layout round trip needed here."""
    indptr, indices, block_size = temporal_mask_metadata
    cfg, H, S, D = q.shape
    assert S % block_size[0] == 0 and S % block_size[1] == 0
    plan = bsr_to_plan(indptr, indices, block_size, S, 0, q.device)
    return core.attention(q, k, v, plan)
