"""Mirror of the reference's svg/kmeans_utils.py operator names on top of the svgb200 kernels.

Same names, argument meaning and return conventions as the reference so svg.models.*.attention can be
pointed here by replacing module globals (svgb200.patch.install).  All tensors must be CUDA tensors;
nothing here falls back to eager PyTorch for the computation.
"""
from __future__ import annotations

import torch

from . import core


class LazyInt:
    """n_iter without a host sync: behaves like an int when (and only when) somebody reads it."""

    def __init__(self, t: torch.Tensor):
        self._t = t

    def __int__(self):
        return int(self._t.item())

    __index__ = __int__

    def __repr__(self):
        return f"LazyInt({int(self)})"

    def __eq__(self, other):
        return int(self) == int(other)


def density_calculation(dynamic_map, q_cluster_sizes, k_cluster_sizes):
    """svg/kmeans_utils.py:13-31 — [cfg,H,QC,KC], [cfg,H,QC], [cfg,H,KC] -> [cfg,H] float32."""
    cfg, H, QC, KC = dynamic_map.shape
    d = core.density(dynamic_map.reshape(cfg * H, QC, KC), q_cluster_sizes.reshape(cfg * H, QC),
                     k_cluster_sizes.reshape(cfg * H, KC))
    return d.view(cfg, H)


def euclid_assign_triton(x, centroids, x_sq, out=None, **_):
    """svg/kmeans_utils.py:562-625 — returns int64 labels like the reference (:595)."""
    lab = core.kmeans_assign(x, centroids, x_sq.float()).to(torch.int64)
    if out is not None:
        out.copy_(lab)
        return out
    return lab


def triton_centroid_update_sorted_euclid(x, cluster_ids, old_centroids, **_):
    """svg/kmeans_utils.py:375-421 -> (centroids in x.dtype, counts int32)."""
    c_new, counts, _ = core.kmeans_update(x, cluster_ids, old_centroids)
    return c_new, counts


def batch_kmeans_Euclid(x, n_clusters, max_iters=100, tol=1e-4, init_centroids=None, verbose=False):
    """svg/kmeans_utils.py:684-733.  x [B,N,D] 16-bit.  Returns (cluster_ids int64 [B,N], centroids
    [B,K,D], cluster_sizes int32 [B,K], n_iters).  The whole loop runs on the device without the
    reference's per-iteration host sync; n_iters is a LazyInt."""
    B, N, D = x.shape
    if init_centroids is None:
        idx = torch.randint(0, N, (B, n_clusters), device=x.device)  # GPU generator, like :708
        init_centroids = torch.gather(x, 1, idx[..., None].expand(-1, -1, D))
    init_centroids = init_centroids.reshape(B, n_clusters, D)
    labels, cents, counts, n_iter = core.kmeans_run(x, init_centroids, max_iters, tol)
    return labels.to(torch.int64), cents, counts, LazyInt(n_iter)


def batch_kmeans_Euclid_sorted(x, n_clusters, max_iters=100, tol=1e-4, init_centroids=None):
    """batch_kmeans_Euclid for the SAP cores: same clustering, labels stay int32 and the stable argsort of the labels
    comes back as a fifth value (the reference recomputes it with torch.argsort: permute_tensor_by_labels_triton, svg/kernels/triton/permute.py:83-128)."""
    B, N, D = x.shape
    if init_centroids is None:
        idx = torch.randint(0, N, (B, n_clusters), device=x.device)  # GPU generator, like :708
        init_centroids = torch.gather(x, 1, idx[..., None].expand(-1, -1, D))
    init_centroids = init_centroids.reshape(B, n_clusters, D)
    labels, cents, counts, n_iter, perm = core.kmeans_run(x, init_centroids, max_iters, tol, want_perm=True)
    return labels, cents, counts, LazyInt(n_iter), perm


def identify_dynamic_map(query_centroids, key_centroids, q_cluster_sizes, k_cluster_sizes, p, min_kc_ratio=0):
    """svg/kmeans_utils.py:864-896 -> bool [B,H,QC,KC]."""
    B, H, QC, D = query_centroids.shape
    KC = key_centroids.shape[2]
    preserve = int(min_kc_ratio * KC) if min_kc_ratio > 0 else 0
    m = core.dynamic_map(query_centroids.reshape(B * H, QC, D), key_centroids.reshape(B * H, KC, D),
                         k_cluster_sizes.reshape(B * H, KC), p, preserve)
    return m.view(B, H, QC, KC)


def _flashinfer_plan(q, block_mask_map, block_row_sz, block_col_sz):
    B, H, S, D = q.shape
    QC, KC = block_row_sz.shape[-1], block_col_sz.shape[-1]
    assert block_mask_map.shape == (B, H, QC, KC)
    dev = q.device
    return core.plan_varblock(block_mask_map.to(dev).reshape(B * H, QC, KC), block_row_sz.to(dev).reshape(B * H, QC),
                              block_col_sz.to(dev).reshape(B * H, KC), S)


def dynamic_block_sparse_fwd_flashinfer(q, k, v, block_mask_map, block_row_sz, block_col_sz, is_cpu=True):
    """svg/kmeans_utils.py:1319-1392.  q,k,v [B,H,S,D]; map bool [B,H,QC,KC]; sizes [B,H,QC]/[B,H,KC]
    (on CPU when is_cpu, like the reference's default; moved to the GPU here)."""
    plan = _flashinfer_plan(q, block_mask_map, block_row_sz, block_col_sz)
    return core.attention(q, k, v, plan)


def dynamic_block_sparse_fwd_triton(q, k, v, dynamic_map, qc_size, kc_size):
    """svg/kmeans_utils.py:1205-1316 (same semantics, same kernel here)."""
    return dynamic_block_sparse_fwd_flashinfer(q, k, v, dynamic_map, qc_size, kc_size, is_cpu=False)


def dynamic_block_sparse_fwd_flashinfer_fp8(q, k, v, block_mask_map, block_row_sz, block_col_sz, is_cpu=True):
    """dynamic_block_sparse_fwd_flashinfer in FP8: q, k, v (already in cluster order) quantised to e4m3 per head and
    run on the e4m3 kernel; head_dim 128 only; the result comes back in q.dtype."""
    from .models.common import fp8_attention

    return fp8_attention(q, k, v, _flashinfer_plan(q, block_mask_map, block_row_sz, block_col_sz))


def dynamic_block_sparse_fwd_triton_fp8(q, k, v, dynamic_map, qc_size, kc_size):
    """dynamic_block_sparse_fwd_triton in FP8 (see dynamic_block_sparse_fwd_flashinfer_fp8)."""
    return dynamic_block_sparse_fwd_flashinfer_fp8(q, k, v, dynamic_map, qc_size, kc_size, is_cpu=False)
