"""GPU parity for the SVG2 front half (flash k-means, dynamic map) and SVG1 profiling (sample_mse).

The reference has no test for these (SURVEY §4); oracles restate svg/kmeans_utils.py:464-733,852-896 and
hyvideo/attention.py:375-399.  Integer outputs are compared exactly wherever the arithmetic is
well-conditioned; points whose best/second-best centroid distances differ by less than the fp32
summation noise are excluded (and counted).
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def clustered(BH, N, K, D, gen, noise=0.3, dtype=torch.bfloat16):
    cent = torch.randn(BH, K, D, generator=gen) * 2.0
    lab = torch.randint(0, K, (BH, N), generator=gen)
    x = torch.gather(cent, 1, lab[:, :, None].expand(-1, -1, D)) + noise * torch.randn(BH, N, D, generator=gen)
    return x.to(dtype), cent.to(dtype), lab


def test_row_sqnorm(cuda):
    from oracle.kmeans import row_sqnorm
    from svgb200 import core

    g = torch.Generator().manual_seed(0)
    x = torch.randn(3, 2000, 128, generator=g).bfloat16()
    got = core.row_sqnorm(x.to(cuda)).cpu()
    ref = row_sqnorm(x)
    # identical up to one bf16 ulp where the fp32 summation order crosses a rounding boundary
    assert (got != ref).float().mean() < 5e-3
    torch.testing.assert_close(got, ref, rtol=2 ** -7, atol=0)


@pytest.mark.parametrize("BH,N,K,D", [(2, 5000, 100, 128), (3, 3001, 300, 128), (2, 2048, 37, 64)])
def test_kmeans_assign(cuda, BH, N, K, D):
    from oracle import kmeans as ok
    from svgb200 import core

    g = torch.Generator().manual_seed(N)
    x, _, _ = clustered(BH, N, K, D, g)
    c = torch.randn(BH, K, D, generator=g).bfloat16()
    x_sq = ok.row_sqnorm(x)
    lab = core.kmeans_assign(x.to(cuda), c.to(cuda), x_sq.to(cuda)).cpu().long()
    ref, margin = ok.euclid_assign(x, c, x_sq)
    safe = margin > 1e-2
    assert safe.float().mean() > 0.98
    assert torch.equal(lab[safe], ref[safe])
    # everywhere: the chosen centroid is a (near-)minimiser
    cent_sq = (c * c).float().sum(-1).bfloat16().float()  # 16-bit ||c||^2, as the reference's kernel holds it (:531)
    cross = torch.einsum("bnd,bkd->bnk", x.float(), c.float())
    dist = (x_sq[:, :, None] + cent_sq[:, None, :] - 2 * cross).clamp_min(0)
    chosen = torch.gather(dist, 2, lab[:, :, None]).squeeze(-1)
    assert torch.all(chosen <= dist.min(-1).values + 2e-2)


def test_kmeans_update_deterministic_and_matches(cuda):
    from oracle import kmeans as ok
    from svgb200 import core

    g = torch.Generator().manual_seed(1)
    BH, N, K, D = 3, 7000, 120, 128
    x, c0, lab = clustered(BH, N, K, D, g)
    lab[0][lab[0] == 5] = 6  # an empty cluster keeps its old centroid
    c_new, counts, shift = core.kmeans_update(x.to(cuda), lab.to(cuda), c0.to(cuda))
    c_new2, _, _ = core.kmeans_update(x.to(cuda), lab.to(cuda), c0.to(cuda))
    assert torch.equal(c_new, c_new2)  # run-to-run bit-exact (reference uses fp32 atomics)
    ref_c, ref_n = ok.centroid_update(x, lab, c0)
    assert torch.equal(counts.cpu(), ref_n)
    assert torch.equal(c_new.cpu()[0, 5], c0[0, 5])
    torch.testing.assert_close(c_new.cpu().float(), ref_c.float(), rtol=2 ** -7, atol=1e-6)
    assert (c_new.cpu() != ref_c).float().mean() < 5e-3
    ref_shift = (ref_c - c0).norm(dim=-1).max().float()
    torch.testing.assert_close(shift.cpu()[0], ref_shift, rtol=2e-2, atol=1e-3)


def test_kmeans_run_matches_reference_control_flow(cuda):
    from oracle import kmeans as ok
    from svgb200 import core

    g = torch.Generator().manual_seed(2)
    BH, N, K, D = 2, 6000, 50, 128
    x, cent, _ = clustered(BH, N, K, D, g, noise=0.1)
    init = (cent.float() + 0.2 * torch.randn(BH, K, D, generator=g)).bfloat16()
    for iters in (1, 2, 6):
        lab, c, cnt, n_it = core.kmeans_run(x.to(cuda), init.to(cuda), iters)
        rl, rc, rn, rit = ok.batch_kmeans_euclid(x, K, iters, init_centroids=init)
        assert int(n_it.item()) == rit
        assert torch.equal(lab.cpu().long(), rl)
        assert torch.equal(cnt.cpu(), rn)
        torch.testing.assert_close(c.cpu().float(), rc.float(), rtol=2 ** -7, atol=1e-6)
    # early exit: start from a fixed point -> first shift is 0 < tol -> break with the OLD centroids
    _, c_fix, _, _ = ok.batch_kmeans_euclid(x, K, 30, init_centroids=init)
    lab, c, cnt, n_it = core.kmeans_run(x.to(cuda), c_fix.to(cuda), 10)
    rl, rc, rn, rit = ok.batch_kmeans_euclid(x, K, 10, init_centroids=c_fix)
    assert int(n_it.item()) == rit
    assert torch.equal(c.cpu(), rc) and torch.equal(lab.cpu().long(), rl)


@pytest.mark.parametrize("D,dtype", [(128, torch.bfloat16), (64, torch.float16)])
def test_kmeans_assign_exact_ties(cuda, D, dtype):
    """Duplicated centroids, as production's randint initialisation (kmeans_utils.py) draws them: every point that
    copies -- or lies near -- a duplicated centroid is equally far from both copies, and the documented rule
    (include/svgb200.h: lowest k wins ties) must pick the lower index.  The pairs sit inside one 32-group (3, 17),
    in two groups of one 128-chunk (5, 40) and in two chunks (7, 200), with K > 256.  Checked with a caller-supplied
    x_sq (svgb_kmeans_assign) and through one Lloyd iteration (svgb_kmeans_run: |x|^2 from shared memory), whose
    update leaves the higher copy empty with its old centroid."""
    from oracle import kmeans as ok
    from svgb200 import core

    g = torch.Generator().manual_seed(41)
    BH, N, K = 2, 4000, 300
    pairs = [(3, 17), (5, 40), (7, 200)]
    c = (torch.randn(BH, K, D, generator=g) * 2.0).to(dtype)
    for lo, hi in pairs:
        c[:, hi] = c[:, lo]
    x = (torch.gather(c.float(), 1, torch.randint(0, K, (BH, N, 1), generator=g).expand(-1, -1, D))
         + 0.3 * torch.randn(BH, N, D, generator=g))
    expect = torch.full((BH, N), -1, dtype=torch.long)
    n_tie = 0
    for lo, hi in pairs:
        for near in (False, True):  # 40 exact copies, then 40 points at distance ~0.05 * sqrt(D)
            sl = slice(n_tie, n_tie + 40)
            x[:, sl] = c[:, lo].float()[:, None] + (0.05 * torch.randn(BH, 40, D, generator=g) if near else 0)
            expect[:, sl] = lo
            n_tie += 40
    x = x.to(dtype)
    tie = expect >= 0
    # assign with the caller's x_sq
    x_sq = ok.row_sqnorm(x)
    lab = core.kmeans_assign(x.to(cuda), c.to(cuda), x_sq.to(cuda)).cpu().long()
    assert torch.equal(lab[tie], expect[tie]), f"{int((lab[tie] != expect[tie]).sum())} tied points off"
    ref, margin = ok.euclid_assign(x, c, x_sq)
    safe = (margin > 1e-2) & ~tie
    assert torch.equal(lab[safe], ref[safe])
    # one Lloyd iteration: |x|^2 from the point tile in shared memory, then the update
    lab1, c1, cnt1, _ = core.kmeans_run(x.to(cuda), c.to(cuda), 1)
    lab1, c1, cnt1 = lab1.cpu().long(), c1.cpu(), cnt1.cpu()
    assert torch.equal(lab1[tie], expect[tie])
    for lo, hi in pairs:
        assert bool((cnt1[:, hi] == 0).all()) and bool((cnt1[:, lo] >= 80).all())
        assert torch.equal(c1[:, hi], c[:, hi])  # an empty cluster keeps its old centroid


@pytest.mark.parametrize("QC,KC,dtype", [(40, 100, torch.bfloat16), (64, 1000, torch.bfloat16), (33, 257, torch.float16)])
def test_dynamic_map(cuda, QC, KC, dtype):
    from oracle import kmeans as ok
    from svgb200 import core

    g = torch.Generator().manual_seed(QC)
    H, D = 4, 128
    qc = torch.randn(1, H, QC, D, generator=g).to(dtype)
    kc = torch.randn(1, H, KC, D, generator=g).to(dtype)
    ks = torch.randint(0, 300, (1, H, KC), generator=g, dtype=torch.int32)
    qs = torch.randint(1, 300, (1, H, QC), generator=g, dtype=torch.int32)
    got = core.dynamic_map(qc[0].to(cuda), kc[0].to(cuda), ks[0].to(cuda), 0.9, int(0.1 * KC)).cpu()
    ref = ok.identify_dynamic_map(qc, kc, qs, ks, 0.9, 0.1)[0]
    assert got.shape == ref.shape
    row_diff = (got != ref).any(-1)
    # rows differ only when an fp32 summation-order difference crosses a 16-bit rounding boundary of a score
    assert row_diff.float().mean() < 0.06, row_diff.float().mean()
    assert (got != ref).sum(-1).max() <= 4
    assert torch.equal(got.sum(-1)[~row_diff], ref.sum(-1)[~row_diff])


@pytest.mark.parametrize("layout,ctx,F,P", [(0, 64, 5, 260), (1, 0, 6, 200)])
def test_sample_mse(cuda, layout, ctx, F, P):
    from oracle import attention as oa
    from svgb200 import core

    g = torch.Generator().manual_seed(3)
    H, D = 3, 128
    S = ctx + F * P
    q, k, v = (torch.randn(1, H, S, D, generator=g).bfloat16() for _ in range(3))
    rows = torch.randint(0, min(1000, F * P), (32,), generator=g)
    got = core.sample_mse(q[0].to(cuda), k[0].to(cuda), v[0].to(cuda), rows.to(cuda), layout, ctx, F, P).cpu()
    name = "hy" if layout == 0 else "wan"
    masks = [oa.profiling_mask_rows(m, rows, name, ctx, F, P) for m in ("spatial", "temporal")]
    ref = oa.sample_mse(q, k, v, rows, masks)[:, 0]
    torch.testing.assert_close(got, ref, rtol=3e-2, atol=1e-6)
    assert torch.equal(got.argmin(0), ref.argmin(0))
