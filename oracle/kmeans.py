"""Oracle: flash-k-means, dynamic map, density.  TEST INFRASTRUCTURE ONLY.

Restates (relative to /root/reference/svg/kmeans_utils.py):
  density_calculation                   :13-31
  _euclid_assign_kernel                 :464-554   (torch formulation kept by the reference at :631-635)
  triton_centroid_update_sorted_euclid  :375-421
  _euclid_iter / batch_kmeans_Euclid    :629-643 / :684-733
  weighted_softmax / identify_dynamic_map  :852-896

Parity status: density / identify_dynamic_map are checked against the reference functions run on CPU
(tests/golden/make_golden.py -> reference_golden.npz).  The k-means kernels are Triton (GPU only, untested by the
reference): pinned by vectors recorded from the reference's own Triton kernels, its Lloyd loop and its GPU
identify_dynamic_map EXECUTED ON A GPU (tests/golden/make_golden_gpu.py -> kmeans_golden.npz; checked by
tests/test_golden_kmeans_cpu.py and, for the CUDA kernels, tests/test_reference_golden_gpu.py).

What those vectors showed (and why label parity is stated with a margin): the reference evaluates ||c||^2 as
`tl.sum(c_tile * c_tile, axis=0)` on bf16 tiles (svg/kmeans_utils.py:531) — products and the reduction stay in
bf16, in a layout / autotune-config dependent order.  Its labels differ from an exactly evaluated argmin on 2-3 % of
the points, and every one of those differences is explained by a per-centroid offset of at most ~2 bf16 ulps of
||c||^2.  Labels are therefore compared exactly on the points whose best / second-best distance gap exceeds
2 * ulp_bf16(max ||c||^2) (`assign_margin_threshold`), the rest is bounded through the inertia.
"""
from __future__ import annotations

import torch


def density_calculation(dynamic_map, q_cluster_sizes, k_cluster_sizes):
    """:13-31.  [cfg,H,QC,KC] bool, [cfg,H,QC], [cfg,H,KC] -> [cfg,H] (exact rational in float64)."""
    blk = q_cluster_sizes[..., :, None].double() * k_cluster_sizes[..., None, :].double()
    return ((blk * dynamic_map.double()).sum(dim=(2, 3)) / blk.sum(dim=(2, 3))).float()


def row_sqnorm(x: torch.Tensor) -> torch.Tensor:
    """x_sq = (x**2).sum(-1) in the input dtype (:704): squares rounded to bf16/fp16, summed with
    fp32 accumulation, result rounded to the input dtype; returned as fp32."""
    return (x ** 2).sum(dim=-1).float()


def euclid_assign(x: torch.Tensor, c: torch.Tensor, x_sq: torch.Tensor) -> torch.Tensor:
    """:464-554.  x [B,N,D], c [B,K,D] (16-bit), x_sq fp32 [B,N] -> labels int64 [B,N] plus the
    (best, second-best) distance margin used by tests to skip numerically ambiguous points.
    dist = max(0, x_sq + sum_d(round16(c*c)) - 2 * (x . c)),  first minimum wins."""
    # :531 `tl.sum(c_tile * c_tile, axis=0)`: 16-bit products, 16-bit result.  The reference's reduction order is
    # implementation-defined; this is the correctly rounded value of the same quantity (see the module docstring).
    cent_sq = (c * c).float().sum(dim=-1).to(c.dtype).float()
    cross = torch.einsum("bnd,bkd->bnk", x.float(), c.float())
    dist = (x_sq[:, :, None] + cent_sq[:, None, :] - 2.0 * cross).clamp_min(0.0)
    labels = dist.argmin(dim=-1)
    top2 = torch.topk(dist, k=min(2, dist.shape[-1]), dim=-1, largest=False).values
    margin = (top2[..., -1] - top2[..., 0]) if dist.shape[-1] > 1 else torch.full_like(top2[..., 0], 1e30)
    return labels, margin


def assign_margin_threshold(c: torch.Tensor) -> float:
    """Distance gap above which a label is independent of how ||c||^2 was rounded: twice the spacing of 16-bit floats
    at the magnitude of the largest ||c||^2 (the resolution of the reference's own centroid-norm term)."""
    import math

    m = float((c.float() ** 2).sum(-1).max())
    mant = 7 if c.dtype == torch.bfloat16 else 10
    return 2.0 * 2.0 ** (math.floor(math.log2(max(m, 1e-30))) - mant)


def centroid_update(x: torch.Tensor, labels: torch.Tensor, old_c: torch.Tensor):
    """:375-421.  fp32 mean of members; empty clusters keep the old centroid; cast to x dtype."""
    B, N, D = x.shape
    K = old_c.shape[1]
    sums = torch.zeros(B, K, D, dtype=torch.float32)
    sums.scatter_add_(1, labels[:, :, None].expand(-1, -1, D), x.float())
    cnts = torch.zeros(B, K, dtype=torch.int64)
    cnts.scatter_add_(1, labels, torch.ones_like(labels))
    mean = sums / cnts.clamp(min=1).unsqueeze(-1).float()
    new_c = torch.where((cnts == 0).unsqueeze(-1), old_c.float(), mean)
    return new_c.to(x.dtype), cnts.to(torch.int32)


def batch_kmeans_euclid(x, n_clusters, max_iters, tol=1e-4, init_centroids=None):
    """:684-733.  Returns (labels, centroids, sizes, n_iter) with the reference's exact control
    flow: labels/sizes come from the last assignment; centroids are the updated ones unless the loop
    broke on `shift < tol`, in which case they are the ones the last assignment was made against."""
    assert init_centroids is not None, "random init (:708) uses the GPU generator; pass centroids"
    x_sq = row_sqnorm(x)
    c = init_centroids
    it = 0
    for it in range(max_iters):
        labels, _ = euclid_assign(x, c, x_sq)
        c_new, sizes = centroid_update(x, labels, c)
        shift = (c_new.float() - c.float()).norm(dim=-1).max()
        if shift < tol:
            break
        c = c_new
    return labels, c, sizes, it + 1


def weighted_softmax(scores, weights):
    """:852-861."""
    dt = scores.dtype
    s = scores.float()
    w = weights.float()
    e = torch.exp(s - s.max(dim=-1, keepdim=True)[0])
    we = w * e
    return (we / we.sum(dim=-1, keepdim=True).clamp(min=1e-12)).to(dt)


def cuda_scan_log_threads(num_rows: int, row_size: int) -> int:
    """get_log_num_threads_x_inner_scan of torch's CUDA scan (ATen/native/cuda/ScanUtils.cuh:19-41, uint32 math)."""
    lx = 0
    while (1 << lx) < row_size:
        lx += 1
    ly = 0
    while (1 << ly) < num_rows:
        ly += 1
    v = ((9 + lx - ly) & 0xFFFFFFFF) // 2
    return min(max(4, v), 9)


def cumsum_like_torch_cuda(x: torch.Tensor, num_rows: int | None = None) -> torch.Tensor:
    """torch.cumsum(x, dim=-1) for a 16-bit tensor AS THE CUDA BACKEND COMPUTES IT — the reference runs
    identify_dynamic_map on the GPU, and `torch.cumsum` of a bf16 CUDA tensor is NOT an fp32 running sum:
    tensor_kernel_scan_innermost_dim (ScanUtils.cuh:300-360) scans blocks of 2*nx elements with a Sklansky network
    whose every `+` is a bf16 add (std::plus<BFloat16>), carrying the block total into element 0 of the next block.
    Near the top-p threshold (0.9, bf16 spacing 2^-8) single small probabilities are absorbed, so the GPU keeps
    systematically MORE clusters than an fp32-accumulated cumsum would (recorded reference maps: +5 of 1000 on
    average, up to +38).  nx = 2^cuda_scan_log_threads(rows, row_size): 16 at 24 heads x 400 q-centroids x 1000
    columns, up to 512 for a few short rows (2 rows x 1024 columns).  One row (numel == row_size) is not this scan:
    torch hands it to cub::DeviceScan, which associates the 16-bit adds differently."""
    dt = x.dtype
    shape = x.shape
    row = shape[-1]
    rows = x.numel() // row if num_rows is None else num_rows
    lg = cuda_scan_log_threads(rows, row)
    nx = 1 << lg
    blk = 2 * nx
    pad = (-row) % blk
    buf = torch.nn.functional.pad(x.reshape(-1, row), (0, pad)).clone()  # init = 0 beyond the row
    total = torch.zeros(buf.shape[0], dtype=dt)
    t = torch.arange(nx)
    for b0 in range(0, buf.shape[1], blk):
        seg = buf[:, b0:b0 + blk]
        seg[:, 0] = seg[:, 0] + total
        for m in range(lg + 1):
            s_ = 1 << m
            a = ((t >> m) << (m + 1)) | s_
            ti, si = a + (t % s_), a - 1
            seg[:, ti] = seg[:, ti] + seg[:, si]  # 16-bit add: rounds to the tensor dtype
        total = seg[:, blk - 1].clone()
    return buf[:, :row].reshape(shape)


def onehot_dynmap_inputs(BH, QC, KC, D, dtype, gen):
    """Inputs on which every step of identify_dynamic_map is exact, so any two implementations must agree bit for bit.
    Key centroid j is 64 * e_c(j), q centroid i is 64 * e_g(i) or zero: scores are 4096 / sqrt(D) ("live", c(j) = g(i))
    or 0 in every summation order and in both 16-bit types; dead columns sit >= 4096 / 16 = 256 below the row maximum,
    where fp32 exp underflows to exactly 0, live ones give exp(0) = 1; the live sizes sum exactly in fp32 (< 2^24), so
    prob_j = round16(fl32(w_j / W_i)).  What follows (sort, 16-bit scan, cut, scatter) is fixed by documented roundings.
    Direction 0 holds ~30 % of the keys, all of size 7 (a long run of equal probabilities across the top-p cut), 1 keys of
    size 0 (W = 0: the 1e-12 denominator keeps every column), 2 exactly one key, 3 none (a row that hits no key: all
    columns live); ~15 % of the q rows are zero (all columns live).  Returns qc [BH,QC,D], kc [BH,KC,D], k_sizes int32."""
    assert D >= 8
    r = torch.rand(BH, KC, generator=gen)
    c = torch.where(r < 0.30, 0, torch.where(r < 0.35, 1, torch.randint(4, D, (BH, KC), generator=gen)))
    sizes = torch.randint(0, 300, (BH, KC), generator=gen, dtype=torch.int32)
    sizes = torch.where(c == 0, 7, torch.where(c == 1, 0, sizes)).to(torch.int32)
    c[:, KC // 2] = 2
    sizes[:, KC // 2] = 100
    g = torch.randint(0, D, (BH, QC), generator=gen)
    lead = torch.tensor([-1, 0, 1, 2, 3])[:QC]  # zero row, then one row per special direction
    g = torch.where(torch.rand(BH, QC, generator=gen) < 0.15, -1, g)
    g[:, : lead.numel()] = lead
    kc = torch.zeros(BH, KC, D).scatter_(2, c[..., None], 64.0)
    qc = torch.zeros(BH, QC, D).scatter_(2, g.clamp(min=0)[..., None], 64.0) * (g >= 0)[..., None]
    return qc.to(dtype), kc.to(dtype), sizes


def identify_dynamic_map(qc, kc, q_sizes, k_sizes, p, min_kc_ratio=0.0, cumsum="cuda"):
    """:864-896 with the tie rule the engine defines (stable descending sort: the lower column
    index first).  qc [B,H,QC,D], kc [B,H,KC,D] in the model dtype (bf16): scores, probabilities and
    their running sum are all rounded to that dtype exactly as the reference's torch ops do ON THE GPU
    (cumsum="cuda": cumsum_like_torch_cuda; cumsum="cpu": torch's CPU kernel, an fp32 running sum rounded per
    element — what the reference computes when its tensors live on the CPU, pinned by reference_golden.npz)."""
    B, H, QC, D = qc.shape
    KC = kc.shape[2]
    scores = torch.matmul(qc, kc.transpose(-2, -1)) / (D ** 0.5)
    probs = weighted_softmax(scores, k_sizes.unsqueeze(-2).float())
    sorted_probs, sorted_idx = torch.sort(probs, dim=-1, descending=True, stable=True)
    cums = cumsum_like_torch_cuda(sorted_probs) if cumsum == "cuda" else torch.cumsum(sorted_probs, dim=-1)
    remove = cums > p
    remove[..., 1:] = remove[..., :-1].clone()
    remove[..., 0] = False
    if min_kc_ratio > 0:
        remove[..., : int(min_kc_ratio * KC)] = False
    out = torch.zeros(B, H, QC, KC, dtype=torch.bool)
    out.scatter_(-1, sorted_idx, ~remove)
    return out
