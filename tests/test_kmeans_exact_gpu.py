"""flash-k-means (csrc/kmeans.cu) at production shapes, one Lloyd iteration at a time, against float64 references.

Shapes: HunyuanVideo 720p ([1, 24, 119056, 128] bf16, 256 text rows last, V = 33 * 3600 = 118800 video rows clustered
in place as a strided view, 400 q- / 1000 k-centroids) and Wan 2.1 720p (S = 75600, 300 / 1000).  Each iteration t is
checked from the kernel's own state C_{t-1} (the loop is deterministic, so the run with max_iters = t reproduces the
first t - 1 iterations of every longer run), so an error cannot hide in a later iteration or cascade into one.

Label bound.  The assign kernel forms d_k = fl(fl(|x|^2 + |c_k|^2) - 2 s_k) with s_k = x.c_k accumulated in fp32 by
wgmma, and compares distances with the low 5 mantissa bits replaced by the in-group index.  With u = 2^-24,
A_k = sum_d |x_d c_kd| (>= |x.c_k|) and M_k = |x|^2 + |c_k|^2 + 2 A_k:
  - fl(|x|^2 + |c_k|^2) and the final subtraction each round once: <= u M_k each;
  - s_k: the D products are exact in fp32 (16-bit x 16-bit); the tensor core aligns / accumulates them in at most 2D
    steps, each losing at most 2u (truncation, not rounding) of a magnitude <= A_k: |e_s| <= 4 D u A_k, which enters
    d_k twice;
  - the packed index: < 32 ulp <= 2^-18 |d_k|, and |d_k| <= M_k (1 + 3u);
so |d_k(kernel) - d_k(exact)| <= E_k = (2u + 2^-18)(1 + 3u) M_k + 8 D u A_k, and clamping at 0 does not increase it.
The kernel's label l therefore satisfies d_l - E_l <= min_k (d_k + E_k) everywhere, and is the exact argmin k* wherever
every other centroid has d_k - E_k above that minimum.  |x|^2 and |c|^2 themselves are reproduced bit for bit (the
kernels' fp32 orders).  Bit-identical centroids (production's random-point initialisation draws a few) tie exactly;
the upper copy must never win, and is then left out of the argmin.
"""
import math

import numpy as np
import pytest
import torch

from oracle.layout import stable_argsort_labels

pytestmark = pytest.mark.gpu

U = 2.0 ** -24


def clustered_gpu(B, N, D, n_true, dtype, seed, noise=0.5):
    g = torch.Generator(device="cuda").manual_seed(seed)
    cent = torch.randn(B, n_true, D, generator=g, device="cuda") * 2.0
    lab = torch.randint(0, n_true, (B, N), generator=g, device="cuda")
    x = torch.gather(cent, 1, lab[..., None].expand(-1, -1, D))
    return (x + noise * torch.randn(B, N, D, generator=g, device="cuda")).to(dtype)


def random_point_init(x, K, seed, dup_pairs=()):
    """Production initialisation (kmeans_utils.batch_kmeans_Euclid_sorted: x[randint] rows), with index (lo, hi)
    pairs forced to draw the same point."""
    B, N, D = x.shape
    g = torch.Generator(device="cuda").manual_seed(seed)
    idx = torch.randint(0, N, (B, K), generator=g, device="cuda")
    for lo, hi in dup_pairs:
        idx[:, hi] = idx[:, lo]
    return torch.gather(x, 1, idx[..., None].expand(-1, -1, D)).contiguous()


def kernel_row_sqnorm(x):
    """|x|^2 as the assign kernel forms it from its point tile: 16-bit squares, fp32 sum in dimension order, rounded
    to the 16-bit type."""
    sq = (x * x).float()
    acc = torch.zeros(sq.shape[:-1], dtype=torch.float32, device=x.device)
    for d in range(sq.shape[-1]):
        acc = acc + sq[..., d]
    return acc.to(x.dtype).float()


def kernel_csq(c):
    """|c|^2 as csq_kernel forms it: lane l sums dims l, l + 32, ... in fp32, a 16-8-4-2-1 butterfly combines the 32
    lanes, the result is rounded to the 16-bit type."""
    B, K, D = c.shape
    sq = (c * c).float().reshape(B, K, D // 32, 32)
    acc = torch.zeros(B, K, 32, dtype=torch.float32, device=c.device)
    for i in range(D // 32):
        acc = acc + sq[..., i, :]
    o = 16
    while o >= 1:
        acc = acc[..., :o] + acc[..., o:2 * o]
        o //= 2
    return acc[..., 0].to(c.dtype).float()


def upper_duplicates(c):
    """[B, K] bool: row k equals (bit for bit) an earlier row of its head."""
    B, K, D = c.shape
    out = torch.zeros(B, K, dtype=torch.bool, device=c.device)
    for b in range(B):
        _, inv = torch.unique(c[b].view(torch.int16), dim=0, return_inverse=True)
        first = torch.full((K,), K, dtype=torch.long, device=c.device).scatter_reduce(
            0, inv, torch.arange(K, device=c.device), reduce="amin")
        out[b] = first[inv] != torch.arange(K, device=c.device)
    return out


def check_labels(x, c, lab, chunk=8192):
    """lab must be the exact argmin of the reference distance (oracle.kmeans.euclid_assign) against c wherever the
    error bounds E_k (module docstring) leave only one candidate, and a candidate everywhere; a point never goes to the
    upper copy of a duplicated centroid (lowest index wins ties).  Returns the fraction of points with several
    candidates (exempt from the exact comparison)."""
    B, N, D = x.shape
    xsq = kernel_row_sqnorm(x).double()
    csq = kernel_csq(c).double()
    cd = c.double()
    dup = upper_duplicates(c)
    exempt = 0
    for b in range(B):
        # an upper copy computes bit-identical distances, and must never win: then it can be left out of the argmin
        assert not bool(dup[b][lab[b].long()].any()), "a point went to the upper copy of a duplicated centroid"
        for r0 in range(0, N, chunk):
            xb = x[b, r0:r0 + chunk].double()
            xs = xsq[b, r0:r0 + chunk]
            dist = (xs[:, None] + csq[b][None, :] - 2.0 * (xb @ cd[b].T)).clamp_min(0.0)
            A = xb.abs() @ cd[b].abs().T  # sum_d |x_d c_d|, which bounds |x.c| and the tensor core's error
            E = (2 * U + 2.0 ** -18) * (1 + 3 * U) * (xs[:, None] + csq[b][None, :] + 2 * A) + 8 * D * U * A
            dist[:, dup[b]] = math.inf
            got = lab[b, r0:r0 + chunk].long()
            best, arg = dist.min(-1)
            hi = (dist + E).min(-1).values  # no centroid the kernel can rank first is above this
            lo = dist - E
            d_got = lo.gather(1, got[:, None])[:, 0]
            worst = int((d_got - hi).argmax())
            assert bool((d_got <= hi).all()), (
                f"head {b} point {r0 + worst}: label {int(got[worst])} at {float(dist[worst, got[worst]])}, minimum "
                f"{float(best[worst])} (label {int(arg[worst])}), bound {float(E[worst, got[worst]] + E[worst, arg[worst]])}")
            lo.scatter_(1, arg[:, None], math.inf)
            sure = lo.min(-1).values > hi  # only the exact argmin can come first
            assert torch.equal(got[sure], arg[sure]), f"head {b}: {int((got[sure] != arg[sure]).sum())} labels off"
            exempt += int((~sure).sum())
    return exempt / (B * N)


def check_update(x, lab, c_prev, c_new, counts):
    """counts = bincount(labels); c_new = float64 mean of the members rounded to the 16-bit type, within one 16-bit ulp
    plus the kernel's fp32 summation error (at most cnt + 32 additions -- 16 or 32 row-groups -- and one division,
    each <= u sum|x| / cnt after the division), identical on
    most entries; empty clusters keep c_prev bit for bit."""
    B, N, D = x.shape
    K = c_prev.shape[1]
    mant = 7 if x.dtype == torch.bfloat16 else 10
    for b in range(B):
        li = lab[b].long()
        cnt = torch.bincount(li, minlength=K)
        assert torch.equal(counts[b].long(), cnt)
        s = torch.zeros(K, D, dtype=torch.float64, device=x.device).index_add_(0, li, x[b].double())
        sa = torch.zeros(K, D, dtype=torch.float64, device=x.device).index_add_(0, li, x[b].double().abs())
        n = cnt.clamp(min=1).double()[:, None]
        mean = s / n
        ulp = torch.exp2(torch.floor(torch.log2(mean.abs().clamp(min=2.0 ** -14))) - mant)
        tol = ulp + (n + 33) * U * sa / n
        live = cnt > 0
        err = (c_new[b].double() - mean).abs()
        assert bool((err[live] <= tol[live]).all()), f"head {b}: centroid off by {float((err - tol)[live].max())}"
        differs = (c_new[b][live] != mean[live].float().to(x.dtype)).float().mean()
        assert differs < 5e-3, differs
        assert torch.equal(c_new[b][~live].view(torch.int16), c_prev[b][~live].view(torch.int16))


def check_iterations(x, init, iters, tol=-1.0):
    """Runs kmeans_run with max_iters = 1..iters and checks iteration t from (labels, centroids) of run t - 1."""
    from svgb200 import core

    c_prev = init
    exempt = []
    for t in range(1, iters + 1):
        lab, c, cnt, n_it, perm = core.kmeans_run(x, init, t, tol, want_perm=True)
        assert int(n_it.item()) == t
        exempt.append(check_labels(x, c_prev, lab))
        check_update(x, lab, c_prev, c, cnt)
        assert np.array_equal(perm.cpu().numpy(), stable_argsort_labels(lab.cpu().numpy()))
        c_prev = c
    return exempt


# ---- a. a strided view clusters exactly like its contiguous copy ---------------------------------------------------
HY_H, HY_S, HY_V, HY_D = 24, 119056, 118800, 128


@pytest.fixture(scope="module")
def hy_tokens(cuda):
    """[24, 119056, 128] bf16: clustered video rows, then 256 text rows holding a large finite value (a head-offset
    error pulls them into a centroid)."""
    t = torch.empty(HY_H, HY_S, HY_D, dtype=torch.bfloat16, device=cuda)
    t[:, :HY_V] = clustered_gpu(HY_H, HY_V, HY_D, 1000, torch.bfloat16, seed=7)
    t[:, HY_V:] = 1.0e4
    return t


def _same_run(x_view, init, iters):
    from svgb200 import core

    a = core.kmeans_run(x_view, init, iters, want_perm=True)
    b = core.kmeans_run(x_view.contiguous(), init, iters, want_perm=True)
    for name, u, v in zip(("labels", "centroids", "counts", "n_iter", "perm"), a, b):
        assert torch.equal(u.view(torch.int16) if u.dtype == torch.bfloat16 else u,
                           v.view(torch.int16) if v.dtype == torch.bfloat16 else v), f"{name} differ"


@pytest.mark.parametrize("iters", [1, 2, 4])
@pytest.mark.parametrize("K", [400, 1000])
def test_strided_view_matches_contiguous(hy_tokens, K, iters):
    x = hy_tokens[:, :HY_V]
    assert x.stride(0) == HY_S * HY_D and not x.is_contiguous()
    _same_run(x, random_point_init(x, K, seed=K), iters)


@pytest.mark.parametrize("iters", [1, 4])
def test_strided_view_matches_contiguous_one_head(hy_tokens, iters):
    x = hy_tokens[5:6, :HY_V]
    _same_run(x, random_point_init(x, 1000, seed=3), iters)


# ---- b. every Lloyd iteration at production size ----------------------------------------------------------------
@pytest.mark.parametrize("model,K", [("hy", 1000), ("hy", 400), ("wan", 1000), ("wan", 300)])
def test_lloyd_iterations_exact_production(cuda, hy_tokens, model, K):
    """Three heads, iterations 1-3, each from the kernel's previous state.  The initialisation is production's
    x[randint] with three forced duplicate pairs -- inside one 32-group, across groups of a chunk, across chunks (the
    last one padded at K = 1000 = 7 * 128 + 104) -- on top of the ones randint draws by itself."""
    if model == "hy":
        x = hy_tokens[:3, :HY_V]  # in place, heads S * D apart
    else:
        x = clustered_gpu(3, 75600, 128, 1000, torch.bfloat16, seed=11)
    pairs = [(3, 17), (5, 40), (7, K - 10)]
    init = random_point_init(x, K, seed=K + 1, dup_pairs=pairs)
    exempt = check_iterations(x, init, 3)
    print(f"{model} K={K}: exempt fraction per iteration {exempt}")
    # near-ties of init points drawn from one cluster: 0.13-0.29 % at iteration 1, less later (H100, both models)
    assert max(exempt) < 5e-3
    from svgb200 import core

    lab, c, cnt, _ = core.kmeans_run(x, init, 1, -1.0)
    for lo, hi in pairs:
        assert bool((cnt[:, hi] == 0).all()) and bool((cnt[:, lo] > 0).all())
        assert not bool((lab == hi).any())
        assert torch.equal(c[:, hi].view(torch.int16), init[:, hi].view(torch.int16))


# ---- c. edges -----------------------------------------------------------------------------------------------------
EDGE_DT = [(128, torch.bfloat16), (64, torch.float16)]


@pytest.mark.parametrize("D,dtype", EDGE_DT, ids=["d128-bf16", "d64-fp16"])
@pytest.mark.parametrize("N,K", [(37, 1), (128, 129), (129, 1000), (128 * 40 + 1, 4096), (128 * 40 + 1, 129),
                                 (37, 4096), (129, 1)])
def test_lloyd_iterations_exact_edges(cuda, N, K, D, dtype):
    """K at its limits (1, 4096), one partial centroid chunk (129), N around the 128-point tile; K > N gives a
    duplicate-rich initialisation."""
    x = clustered_gpu(2, N, D, 64, dtype, seed=N + K)
    init = random_point_init(x, K, seed=N * K)
    exempt = check_iterations(x, init, 2)
    assert max(exempt) < 3e-2  # a few hundred points: one near-tie weighs more


def test_kmeans_bytes_rejects_k_above_4096():
    import ctypes

    from svgb200._lib import lib

    n = ctypes.c_size_t()
    assert lib().svgb_kmeans_bytes(1, 128, 4096, 128, ctypes.byref(n)) == 0
    assert lib().svgb_kmeans_bytes(1, 128, 4097, 128, ctypes.byref(n)) != 0


@pytest.mark.parametrize("K", [129, 4096])
def test_identical_points_all_label_zero(cuda, K):
    from svgb200 import core

    g = torch.Generator(device=cuda).manual_seed(K)
    x = torch.randn(1, 1, 128, generator=g, device=cuda).to(torch.bfloat16).expand(2, 1000, 128).contiguous()
    init = x[:, :K] if K <= 1000 else x[:, :1].expand(2, K, 128).contiguous()
    lab, c, cnt, n_it, perm = core.kmeans_run(x, init, 3, want_perm=True)
    assert not bool(lab.any())
    assert bool((cnt[:, 0] == 1000).all()) and int(cnt.sum()) == 2000
    assert torch.equal(perm.cpu(), torch.arange(1000, dtype=torch.int32).expand(2, -1))


def test_early_exit(cuda):
    """tol = 1e9 stops after the first iteration; a tol between the first two shifts after the second.  Either way
    n_iter is right, the centroids are the ones the last assignment was made against (the loop breaks before
    `centroids = centroids_new`), and perm_out is the stable argsort of the returned labels, not of a stale iteration."""
    from svgb200 import core

    x = clustered_gpu(2, 128 * 40 + 1, 128, 64, torch.bfloat16, seed=5)
    init = random_point_init(x, 129, seed=6)
    runs = [core.kmeans_run(x, init, t, -1.0, want_perm=True) for t in (1, 2)]
    (l1, c1, n1, _, _), (l2, c2, n2, _, _) = runs

    def shift(a, b):  # the kernel's shift: 16-bit difference, norm rounded to 16 bit (within 1 % of this)
        return float((a.float() - b.float()).to(x.dtype).float().norm(dim=-1).max())

    s1, s2 = shift(c1, init), shift(c2, c1)
    assert s1 > 1.25 * s2 > 0, (s1, s2)  # the data give a tol that separates the two iterations
    for tol, it, lab, cnt, cent in ((1e9, 1, l1, n1, init), (math.sqrt(s1 * s2), 2, l2, n2, c1)):
        lab_e, c_e, cnt_e, n_e, perm_e = core.kmeans_run(x, init, 6, tol, want_perm=True)
        assert int(n_e.item()) == it
        assert torch.equal(c_e.view(torch.int16), cent.view(torch.int16))
        assert torch.equal(lab_e, lab) and torch.equal(cnt_e, cnt)
        assert np.array_equal(perm_e.cpu().numpy(), stable_argsort_labels(lab.cpu().numpy()))
    assert not torch.equal(l1, l2)  # a stale permutation would show
