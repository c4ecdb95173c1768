"""GPU parity tests for the wgmma attention path, through the C ABI, against the CPU oracle.

Grids follow the reference's own tests: svg/kernels/test/test_sparse_attn_dyn_blk_wan.py:74-133
(variable blocks; atol=rtol=1e-2) and test_sparse_attn.py:90-95 (fp16 5e-3, bf16 (3e-2, 2e-2)).
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

TOL = {torch.float16: dict(rtol=5e-3, atol=5e-3), torch.bfloat16: dict(rtol=3e-2, atol=2e-2)}
# lse: fp32 scores from exact 16-bit products and an fp32 row sum of ex2.approx terms (relative error ~1e-6) put the
# kernel's lse within ~1e-5 of the fp64 logsumexp of the same 16-bit inputs; 1e-3 / 1e-4 leaves room for the
# summation order of the logits, not for a wrong key set or scale
LSE_TOL = dict(rtol=1e-4, atol=1e-3)
# large logits (output ~ one key): P is rounded to the 16-bit type before P V and the output once more, so the error
# is relative to softmax(s) |V| of the row: two roundings of 2^-9 (bf16) / 2^-12 (fp16) each
REL = {torch.bfloat16: 2 * 2 ** -8, torch.float16: 2 * 2 ** -11}


def check_lse(lse, ref_lse, **tol):
    """kernel lse vs the fp64 logsumexp; rows without a key must be exactly -inf"""
    lse, ref_lse = lse.cpu().double().reshape(ref_lse.shape), ref_lse.double()
    empty = ref_lse == float("-inf")
    assert torch.equal(lse == float("-inf"), empty), "-inf rows differ"
    torch.testing.assert_close(lse[~empty], ref_lse[~empty], **(tol or LSE_TOL))


def check_relative(o, ref, ref_abs, rel):
    """|o - ref| <= rel * (softmax(s) |V|) row-wise scale: a bound that holds whatever the logit magnitude"""
    err = (o.double() - ref.double()).abs()
    bound = rel * ref_abs.double() + 1e-6
    assert bool((err <= bound).all()), f"max excess {float((err - bound).max())}"


def random_partition(seq_len, num_blocks, gen):
    """random_partition_batch (test_sparse_attn_dyn_blk_wan.py:8-35) for one head."""
    cuts = torch.randperm(seq_len - 1, generator=gen)[: num_blocks - 1] + 1
    cuts, _ = torch.sort(cuts)
    return torch.diff(torch.cat([torch.tensor([0]), cuts, torch.tensor([seq_len])])).to(torch.int32)


@pytest.mark.parametrize("D", [128, 64])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_selftest_tile(cuda, D, dtype):
    """One 128x128xD tile through the same descriptors as the attention kernel: S = Q K^T (SS,
    K-major) must be exact up to fp32 summation order; O = round16(S*scale) V (TS, MN-major V)."""
    from svgb200 import core

    g = torch.Generator().manual_seed(0)
    q = torch.randn(128, D, generator=g).to(dtype)
    k = torch.randn(128, D, generator=g).to(dtype)
    v = torch.randn(128, D, generator=g).to(dtype)
    p_scale = 0.0625
    s, o = core.selftest_tile(q.to(cuda), k.to(cuda), v.to(cuda), p_scale)
    torch.cuda.synchronize()
    s_ref = q.float() @ k.float().T
    torch.testing.assert_close(s.cpu(), s_ref, rtol=1e-4, atol=1e-3)
    p = (s.cpu() * p_scale).to(dtype).float()
    o_ref = p @ v.float()
    torch.testing.assert_close(o.cpu(), o_ref, rtol=1e-3, atol=2e-2)


def _run_varblock(cuda, H, D, S, MB, NB, density, dtype, seed, uniform_sizes=False, gather=False, sm_scale=None,
                  gain=1.0, hot_masked=False):
    """-> (o, ref, lse, ref_lse, ref_abs): kernel output, fp64 oracle (as fp32), kernel lse, fp64 logsumexp and the
    oracle's softmax(s) |V|.  gain scales q and k (logits ~ gain^2); hot_masked gives the keys of key block 0 the
    largest scores of every row and deselects that block everywhere."""
    from oracle.attention import dynamic_block_sparse_fwd
    from svgb200 import core

    g = torch.Generator().manual_seed(seed)
    if uniform_sizes:
        row = torch.full((H, MB), S // MB, dtype=torch.int32)
        col = torch.full((H, NB), S // NB, dtype=torch.int32)
    else:
        row = torch.stack([random_partition(S, MB, g) for _ in range(H)])
        col = torch.stack([random_partition(S, NB, g) for _ in range(H)])
    bmap = torch.rand(H, MB, NB, generator=g) > density  # same polarity as the reference test (:101)
    q = torch.randn(1, H, S, D, generator=g) * gain
    k = torch.randn(1, H, S, D, generator=g) * gain
    v = torch.randn(1, H, S, D, generator=g).to(dtype)
    if hot_masked:
        u = torch.randn(D, generator=g)
        q = q + 2 * u
        for h in range(H):
            k[0, h, : int(col[h, 0])] = 5 * u  # scores ~ +110 against ~N(0, 5) elsewhere
        bmap[:, :, 0] = False
    q, k = q.to(dtype), k.to(dtype)
    plan = core.plan_varblock(bmap.to(cuda), row.to(cuda), col.to(cuda), S, gather=gather)
    o, lse = core.attn_fwd(q.to(cuda), k.to(cuda), v.to(cuda), plan, return_lse=True, sm_scale=sm_scale)
    torch.cuda.synchronize()
    args = (bmap[None], row[None], col[None], sm_scale)
    ref, ref_lse = dynamic_block_sparse_fwd(q, k, v, *args, return_lse=True, dtype=torch.float64)
    ref_abs = dynamic_block_sparse_fwd(q, k, v.abs(), *args, dtype=torch.float64) if (gain != 1 or hot_masked) else None
    return o.float().cpu(), ref.float(), lse.cpu().view(1, H, S), ref_lse, ref_abs


@pytest.mark.parametrize("D", [128, 64])
@pytest.mark.parametrize("S", [256, 4096])
@pytest.mark.parametrize("MB,NB", [(10, 50), (20, 100)])
@pytest.mark.parametrize("density", [0.2, 0.7, 0.9])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_variable_block_sparse_attention(cuda, D, S, MB, NB, density, dtype):
    """Reference grid of test_sparse_attn_dyn_blk_wan.py (heads folded to 2 per case)."""
    o, ref, lse, ref_lse, _ = _run_varblock(cuda, 2, D, S, MB, NB, density, dtype, seed=hash((D, S, MB, NB)) % 1000)
    torch.testing.assert_close(o, ref, atol=1e-2, rtol=1e-2)
    check_lse(lse, ref_lse)


@pytest.mark.parametrize("D", [128, 64])
@pytest.mark.parametrize("S,MB,NB", [(256, 10, 50), (4096, 20, 100), (1000, 7, 33)])
@pytest.mark.parametrize("density", [0.2, 0.7])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_variable_block_gather_path(cuda, D, S, MB, NB, density, dtype):
    """Same grid through the row-gather kernel path (cp.async producers, exactly-full chunks)."""
    o, ref, lse, ref_lse, _ = _run_varblock(cuda, 2, D, S, MB, NB, density, dtype, seed=hash((D, S, MB)) % 1000,
                                            gather=True)
    torch.testing.assert_close(o, ref, atol=1e-2, rtol=1e-2)
    check_lse(lse, ref_lse)


@pytest.mark.parametrize("gather", [False, True])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("variant", [("sm_scale", 0.05), ("sm_scale", 0.3), ("gain", 4.5), ("hot_masked", 1.0)])
def test_variable_block_scale_and_large_logits(cuda, variant, dtype, gather):
    """A caller's sm_scale (C ABI / core.attn_fwd) multiplies the logits of both the output and the lse.  With an
    input gain of 4.5 the scaled logits span more than 100 (exp over- / underflows in fp32 without the running-max
    subtraction); with hot_masked the largest score of every row sits on a MASKED key (a max taken before masking
    underflows every allowed p).  Large-logit cases are checked with a bound relative to softmax(s) |V|."""
    name, val = variant
    kw = {name: val if name != "hot_masked" else True}
    o, ref, lse, ref_lse, ref_abs = _run_varblock(cuda, 2, 128, 4096, 20, 100, 0.5, dtype, seed=31, gather=gather,
                                                  **kw)
    check_lse(lse, ref_lse)
    if ref_abs is None:
        torch.testing.assert_close(o, ref, atol=1e-2, rtol=1e-2)
    else:
        check_relative(o, ref, ref_abs, REL[dtype])
    if name == "gain":
        finite = ref_lse[ref_lse > float("-inf")]
        assert float(finite.max() - finite.min()) > 50  # lse spread; the logits themselves span > 100


def test_gather_path_fused_permutation(cuda):
    """q_rows / kv_rows / o_rows = cluster argsorts: SVG2 attention straight on the un-permuted tensors equals
    masked attention under  allowed(i, j) = map[qlabel(i), klabel(j)]  (and equals the permute->attend->
    inverse-permute pipeline of hyvideo/attention.py:628-655,778-783); lse lands on the output rows, -inf for the
    query cluster that sees nothing."""
    _gather_fused_permutation(cuda, "bhsd")


def test_gather_path_fused_permutation_shd(cuda):
    """The same fused-permutation gather in the [S, H, D] layout (row gathers with row stride H*D)."""
    _gather_fused_permutation(cuda, "shd")


def _gather_fused_permutation(cuda, layout):
    from svgb200 import core

    g = torch.Generator().manual_seed(21)
    H, S, D, QC, KC = 3, 1500, 128, 9, 31
    q, k, v = (torch.randn(1, H, S, D, generator=g).to(torch.bfloat16) for _ in range(3))
    ql = torch.randint(0, QC, (H, S), generator=g)
    kl = torch.randint(0, KC, (H, S), generator=g)
    kl[0][kl[0] == 3] = 4  # an empty key cluster
    bm = torch.rand(H, QC, KC, generator=g) > 0.5
    bm[1, 2, :] = False     # a query cluster that sees nothing
    qperm, qcnt = core.argsort_labels(ql.to(cuda), QC)
    kperm, kcnt = core.argsort_labels(kl.to(cuda), KC)
    plan = core.plan_varblock(bm.to(cuda), qcnt, kcnt, S, gather=True)
    if layout == "shd":
        qs, ks_, vs = (t[0].permute(1, 0, 2).contiguous().to(cuda) for t in (q, k, v))
        o, lse = core.attn_fwd(qs, ks_, vs, plan, layout="shd", q_rows=qperm, kv_rows=kperm, o_rows=qperm,
                               return_lse=True)
        o = o.float().cpu().permute(1, 0, 2)[None]
    else:
        o, lse = core.attn_fwd(q.to(cuda), k.to(cuda), v.to(cuda), plan, q_rows=qperm, kv_rows=kperm, o_rows=qperm,
                               return_lse=True)
        o = o.float().cpu()
    for h in range(H):
        allowed = bm[h][ql[h]][:, kl[h]]
        s = (q[0, h].double() @ k[0, h].double().T) * D ** -0.5
        s = s.masked_fill(~allowed, float("-inf"))
        w = torch.nan_to_num(torch.softmax(s, -1), nan=0.0)
        torch.testing.assert_close(o[0, h], (w @ v[0, h].double()).float(), atol=1e-2, rtol=1e-2)
        check_lse(lse[h], torch.logsumexp(s, -1))
    assert torch.all(o[0, 1][ql[1] == 2] == 0)


def test_variable_block_long_uniform(cuda):
    """8192 tokens, 4 heads, uniform clusters (exercises 2-tile items and multi-chunk runs)."""
    o, ref, lse, ref_lse, _ = _run_varblock(cuda, 4, 128, 8192, 32, 64, 0.5, torch.bfloat16, seed=3, uniform_sizes=True)
    torch.testing.assert_close(o, ref, atol=1e-2, rtol=1e-2)
    check_lse(lse, ref_lse)


def test_variable_block_empty_rows_and_blocks(cuda):
    """Empty clusters are legal and q-rows with no selected key must return 0 (SURVEY App.B #4)."""
    from oracle.attention import dynamic_block_sparse_fwd
    from svgb200 import core

    g = torch.Generator().manual_seed(7)
    H, S, D = 2, 1024, 128
    row = torch.tensor([[0, 300, 0, 500, 224], [1024, 0, 0, 0, 0]], dtype=torch.int32)
    col = torch.tensor([[100, 0, 400, 24, 0, 500], [0, 0, 0, 1000, 0, 24]], dtype=torch.int32)
    bmap = torch.rand(H, 5, 6, generator=g) > 0.5
    bmap[0, 3, :] = False  # a q-block that sees nothing
    bmap[1, 0, :] = True
    q, k, v = (torch.randn(1, H, S, D, generator=g).to(torch.bfloat16) for _ in range(3))
    plan = core.plan_varblock(bmap.to(cuda), row.to(cuda), col.to(cuda), S)
    o = core.attn_fwd(q.to(cuda), k.to(cuda), v.to(cuda), plan).float().cpu()
    ref = dynamic_block_sparse_fwd(q, k, v, bmap[None], row[None], col[None])
    torch.testing.assert_close(o, ref, atol=1e-2, rtol=1e-2)
    assert torch.all(o[0, 0, 300:800] == 0)


def test_dense_equals_sdpa(cuda):
    """map = all ones, one block: the dense fall-back (b11)."""
    from svgb200 import core

    g = torch.Generator().manual_seed(11)
    H, S, D = 3, 1000, 128  # S not a multiple of 128: tail chunk + OOB rows
    q, k, v = (torch.randn(1, H, S, D, generator=g).to(torch.bfloat16) for _ in range(3))
    one = torch.ones(H, 1, 1, dtype=torch.bool)
    sz = torch.full((H, 1), S, dtype=torch.int32)
    plan = core.plan_varblock(one.to(cuda), sz.to(cuda), sz.to(cuda), S)
    o, lse = core.attn_fwd(q.to(cuda), k.to(cuda), v.to(cuda), plan, return_lse=True)
    ref = torch.nn.functional.scaled_dot_product_attention(q.float(), k.float(), v.float())
    torch.testing.assert_close(o.float().cpu(), ref, **TOL[torch.bfloat16])
    s = (q.float() @ k.float().transpose(-1, -2)) * D ** -0.5
    torch.testing.assert_close(lse.cpu().view(1, H, S), torch.logsumexp(s, -1), rtol=1e-3, atol=1e-3)


BAND_CASES = [
    # (mode, F, P, ctx, prompt_len, mul) -- small analogues of HY (text last), WAN (sink), COG (text first)
    ("hy", 6, 200, 48, 20, 1.4),
    ("hy", 5, 333, 64, 64, 0.9),
    ("wan", 7, 180, 0, 0, 1.2),
    ("cog", 4, 260, 40, 40, 1.1),
]


def _band(case):
    from oracle import attention as oa
    from svgb200 import core

    mode, F, P, ctx, plen, mul = case
    if mode == "hy":
        return oa.hy_mask_mod(ctx, plen, F, P, mul), (core.MASK_HY, F * P, F * P + plen, oa.hy_band_width(mul, P))
    if mode == "wan":
        return oa.wan_mask_mod(F, P, mul), (core.MASK_WAN, P, 0, oa.wan_band_width(mul, P))
    return oa.cog_mask_mod(plen, F, P, mul), (core.MASK_COG, plen, plen, oa.hy_band_width(mul, P))


@pytest.mark.parametrize("case", BAND_CASES)
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_band_attention_matches_mask_mod(cuda, case, dtype):
    """SVG1 executed mask: element-exact mask_mod semantics (hyvideo/utils.py:20-44 etc.), output and lse."""
    _band_case(cuda, case, dtype, 128)


@pytest.mark.parametrize("case", BAND_CASES)
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_band_attention_head_dim_64(cuda, case, dtype):
    """The same band plans with head_dim 64 (64-wide P V tiles, one 128-byte panel per row)."""
    _band_case(cuda, case, dtype, 64)


def _band_case(cuda, case, dtype, D):
    from oracle import attention as oa
    from svgb200 import core

    mode, F, P, ctx, plen, mul = case
    S = ctx + F * P
    mod, args = _band(case)
    g = torch.Generator().manual_seed(5)
    H = 2
    q, k, v = (torch.randn(1, H, S, D, generator=g).to(dtype) for _ in range(3))
    plan = core.plan_band(*args, H, S, cuda)
    o, lse = core.attn_fwd(q.to(cuda), k.to(cuda), v.to(cuda), plan, return_lse=True)
    ref, ref_lse = oa.masked_attention_bhsd(q[0], k[0], v[0], mod, return_lse=True, dtype=torch.float64)
    torch.testing.assert_close(o.float().cpu(), ref.float()[None], **TOL[dtype])
    check_lse(lse, ref_lse)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("variant", [("sm_scale", 0.05), ("sm_scale", 0.3), ("gain", 4.5), ("hot_masked", 1.0)])
def test_band_scale_and_large_logits(cuda, variant, dtype):
    """Band plan (Wan mask, element-mask chunks) under a caller's sm_scale, logits spanning more than 100, and the
    largest scores on masked keys (the last frame, outside the band of the early rows): output within a bound
    relative to softmax(s) |V|, lse against the fp64 logsumexp."""
    from oracle import attention as oa
    from svgb200 import core

    case = ("wan", 7, 180, 0, 0, 1.2)
    mod, args = _band(case)
    F, P = case[1], case[2]
    S, H, D = F * P, 2, 128
    name, val = variant
    g = torch.Generator().manual_seed(13)
    gain = val if name == "gain" else 1.0
    q = torch.randn(1, H, S, D, generator=g) * gain
    k = torch.randn(1, H, S, D, generator=g) * gain
    v = torch.randn(1, H, S, D, generator=g).to(dtype)
    if name == "hot_masked":
        u = torch.randn(D, generator=g)
        q = q + 2 * u
        k[:, :, S - P:] = 5 * u  # scores ~ +110; masked for every row farther than W from the last frame
    q, k = q.to(dtype), k.to(dtype)
    sm = val if name == "sm_scale" else None
    plan = core.plan_band(*args, H, S, cuda)
    o, lse = core.attn_fwd(q.to(cuda), k.to(cuda), v.to(cuda), plan, return_lse=True, sm_scale=sm)
    ref, ref_lse = oa.masked_attention_bhsd(q[0], k[0], v[0], mod, sm_scale=sm, return_lse=True, dtype=torch.float64)
    check_lse(lse, ref_lse)
    if name == "sm_scale":
        torch.testing.assert_close(o.float().cpu(), ref.float()[None], **TOL[dtype])
    else:
        ref_abs = oa.masked_attention_bhsd(q[0], k[0], v[0].abs(), mod, sm_scale=sm, dtype=torch.float64)
        check_relative(o.float().cpu()[0], ref, ref_abs, REL[dtype])


def test_shd_layout_and_scatter_rows(cuda):
    """[S,H,D] addressing (ops API) and the fused inverse-permutation store."""
    from oracle.attention import dynamic_block_sparse_fwd
    from svgb200 import core

    g = torch.Generator().manual_seed(9)
    H, S, D = 3, 768, 64
    row = torch.stack([random_partition(S, 4, g) for _ in range(H)])
    col = torch.stack([random_partition(S, 9, g) for _ in range(H)])
    bmap = torch.rand(H, 4, 9, generator=g) > 0.4
    q, k, v = (torch.randn(S, H, D, generator=g).to(torch.float16) for _ in range(3))
    plan = core.plan_varblock(bmap.to(cuda), row.to(cuda), col.to(cuda), S)
    o = core.attn_fwd(q.to(cuda), k.to(cuda), v.to(cuda), plan, layout="shd").float().cpu()
    ref = dynamic_block_sparse_fwd(*(t.permute(1, 0, 2)[None] for t in (q, k, v)), bmap[None], row[None], col[None])
    torch.testing.assert_close(o.permute(1, 0, 2)[None], ref, atol=1e-2, rtol=1e-2)
    # scatter rows: o2[h, perm[h, s]] = o[h, s]
    perm = torch.stack([torch.randperm(S, generator=g) for _ in range(H)]).to(torch.int32)
    qb, kb, vb = (t.permute(1, 0, 2).contiguous()[None] for t in (q, k, v))
    o2 = core.attn_fwd(qb.to(cuda), kb.to(cuda), vb.to(cuda), plan, o_rows=perm.to(cuda)).float().cpu()
    expect = torch.empty_like(ref)
    expect[0].scatter_(1, perm.long()[:, :, None].expand(-1, -1, D), ref[0])
    torch.testing.assert_close(o2, expect, atol=1e-2, rtol=1e-2)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("layout", ["bhsd", "shd"])
def test_transposed_tail_kernel_edge_sizes(cuda, dtype, layout):
    """Tails of a variable-block plan (the last r % 256 <= 128 rows of a q-block), paired two per CTA as dual items.
    q-block sizes are chosen to hit every split of `r % 256` (plan_items_kernel): tails of 1 / 15 / 16 / 17 /
    33 / 48 / 64 rows, longer tails (65..128), 128 + 33, a partial two-tile item, an empty q-block, a q-block that
    selects no key block at all (-> zeros) and an odd number of tails (one CTA with a single tail); ragged key
    blocks so that chunks have every width; output through a row scatter for the bhsd layout."""
    from oracle.attention import dynamic_block_sparse_fwd
    from svgb200 import core

    g = torch.Generator().manual_seed(5)
    H, D = 2, 128
    rows = [257, 15, 64, 128 + 33, 300, 48, 17, 0, 64 + 256, 1, 16, 33, 100, 128, 200]
    S = sum(rows)
    row = torch.tensor([rows, rows[::-1]], dtype=torch.int32)
    KC = 23
    col = torch.stack([random_partition(S, KC, g) for _ in range(H)])
    bmap = torch.rand(H, len(rows), KC, generator=g) < 0.45
    bmap[0, 1, :] = False       # a short tail that attends nothing
    bmap[1, 3, :] = True        # and one that attends everything
    q, k, v = (torch.randn(1, H, S, D, generator=g).to(dtype) for _ in range(3))
    plan = core.plan_varblock(bmap.to(cuda), row.to(cuda), col.to(cuda), S)
    ref, ref_lse = dynamic_block_sparse_fwd(q, k, v, bmap[None], row[None], col[None], return_lse=True,
                                            dtype=torch.float64)
    ref = ref.float()
    if layout == "bhsd":
        perm = torch.stack([torch.randperm(S, generator=g) for _ in range(H)]).to(torch.int32)
        o, lse = core.attn_fwd(q.to(cuda), k.to(cuda), v.to(cuda), plan, o_rows=perm.to(cuda), return_lse=True)
        o, lse = o.float().cpu(), lse.cpu()
        o = torch.stack([o[0, h][perm[h].long()] for h in range(H)])[None]  # undo the scatter (lse follows o)
        lse = torch.stack([lse[h][perm[h].long()] for h in range(H)])[None]
    else:
        qs, ks_, vs = (t[0].permute(1, 0, 2).contiguous().to(cuda) for t in (q, k, v))
        o, lse = core.attn_fwd(qs, ks_, vs, plan, layout="shd", return_lse=True)
        o = o.float().cpu().permute(1, 0, 2)[None]
    torch.testing.assert_close(o, ref, **TOL[dtype])
    check_lse(lse, ref_lse)  # the tail that selects nothing: -inf
    r0 = rows[0]
    assert torch.all(o[0, 0, r0:r0 + rows[1]] == 0)
