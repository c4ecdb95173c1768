"""Mirror of svg/kernels/triton/permute.py (:82-170).

Differentiable in the permuted tensor when it requires grad: the backward of the gather is the scatter under the same
indices and vice versa (core._Permute); labels and sorted indices are constants."""
from __future__ import annotations

from typing import Optional

import torch

from . import core


# Upper bound on cluster ids when the caller does not say (the reference passes labels only).  Using a
# bound instead of labels.max() keeps the call free of host syncs; the reference configs use <= 1000.
MAX_CLUSTERS = 4096


def permute_tensor_by_labels_triton(tensor: torch.Tensor, labels: Optional[torch.Tensor], dim: int, *,
                                    sorted_indices: Optional[torch.Tensor] = None,
                                    num_clusters: Optional[int] = None):
    """Permute `tensor` [B,H,S,D] along dim 2 by ascending label.  Returns (permuted, sorted_indices int32
    [B*H, S]).  Ties keep token order (stable) — the reference's torch.argsort is unstable (:113)."""
    assert dim == 2, "permute_tensor_by_labels currently only supports dim==2 (sequence dimension)"
    assert tensor.dim() == 4, "Expected tensor shape [B,H,S,D]"
    assert tensor.is_cuda, "permute_tensor_by_labels requires CUDA tensors"
    B, H, S, D = tensor.shape
    if sorted_indices is not None:
        sorted_indices = sorted_indices.to(torch.int32).contiguous()
    else:
        assert labels is not None, "Either `labels` or `sorted_indices` must be provided."
        lab = labels.to(tensor.device).reshape(B * H, S)
        sorted_indices, _ = core.argsort_labels(lab, num_clusters or MAX_CLUSTERS)
    return core.permute_gather(tensor, sorted_indices), sorted_indices


def permute_by_sorted_indices(tensor, sorted_indices):
    return core.permute_gather(tensor, sorted_indices)


def apply_inverse_permutation_triton(permuted_tensor: torch.Tensor, sorted_indices: torch.Tensor, dim: int):
    """out[..., sorted_indices[s], :] = permuted[..., s, :]  (:131-170)."""
    assert dim == 2, "apply_inverse_permutation currently only supports dim==2"
    assert permuted_tensor.dim() == 4, "Expected tensor shape [B,H,S,D]"
    assert permuted_tensor.is_cuda, "apply_inverse_permutation requires CUDA tensors"
    return core.permute_scatter(permuted_tensor, sorted_indices)
