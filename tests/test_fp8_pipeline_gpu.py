"""FP8 (e4m3) through every layer: the row-gather kernel path (svgb_attn_fwd on a gather plan / core.attn_fwd_fp8 with
q_rows / kv_rows), the SVG1 and SVG2 cores with fp8=True, and patch.install(..., fp8=True).

Kernel results are compared with the fp64 oracle on the de-quantised inputs at the FP8 tolerances of
tests/test_fp8_gpu.py (rtol 8e-2 / atol 4e-2, LSE as FP8_LSE); everything the FP8 mode leaves 16-bit (profiling,
k-means, maps, permutations, dense branch) is compared bit for bit with the 16-bit core."""
import pytest
import torch

pytestmark = pytest.mark.gpu

FP8_TOL = dict(rtol=8e-2, atol=4e-2)
FP8_LSE = dict(rtol=1e-3, atol=5e-3)


def _deq(x8, s):
    H = s.numel()
    return x8.view(torch.float8_e4m3fn).double().cpu() * s.cpu().double().view(1, H, 1, 1)


def _check_lse(lse, ref_lse):
    lse, ref_lse = lse.cpu().double().reshape(ref_lse.shape), ref_lse.double()
    empty = ref_lse == float("-inf")
    assert torch.equal(lse == float("-inf"), empty), "-inf rows differ"
    torch.testing.assert_close(lse[~empty], ref_lse[~empty], **FP8_LSE)


def _clusters(cuda, H, S, QC, KC, g):
    """Random labels with an empty query cluster (head 0), an empty key cluster (head 1), a query cluster that
    selects nothing and one that selects everything (head 2) -> (map, q_perm, q_counts, k_perm, k_counts)."""
    from svgb200 import core

    ql = torch.randint(0, QC, (H, S), generator=g)
    kl = torch.randint(0, KC, (H, S), generator=g)
    ql[0][ql[0] == 5] = 6
    kl[1][kl[1] == 3] = 4
    bm = torch.rand(H, QC, KC, generator=g) < 0.4
    bm[2, 7, :] = False
    bm[2, 8, :] = True
    qperm, qcnt = core.argsort_labels(ql.to(cuda), QC)
    kperm, kcnt = core.argsort_labels(kl.to(cuda), KC)
    return bm, qperm, qcnt, kperm, kcnt


def _scaled_qkv(H, S, D, g):
    """Heads whose q / v scales differ by ~300x, so a scale read from the wrong head fails."""
    fq, fv = torch.tensor([0.03, 10.0, 1.0])[:H], torch.tensor([10.0, 0.03, 1.0])[:H]
    q = (torch.randn(1, H, S, D, generator=g) * fq.view(1, H, 1, 1)).bfloat16()
    k = torch.randn(1, H, S, D, generator=g).bfloat16()
    v = (torch.randn(1, H, S, D, generator=g) * fv.view(1, H, 1, 1)).bfloat16()
    return q, k, v, fv


def test_fp8_gather_matches_oracle(cuda):
    """FP8 gather with q_rows / kv_rows / o_rows on random cluster permutations vs the fp64 oracle on de-quantised
    inputs; rows of the q-cluster that selects nothing give output 0 and an LSE of exactly -inf."""
    from oracle import attention as oa
    from svgb200 import core

    g = torch.Generator().manual_seed(31)
    H, S, D, QC, KC = 3, 6000, 128, 37, 101
    bm, qperm, qcnt, kperm, kcnt = _clusters(cuda, H, S, QC, KC, g)
    q, k, v, fv = _scaled_qkv(H, S, D, g)
    (q8, sq), (k8, sk), (v8, sv) = (core.quantize_e4m3(t.to(cuda)) for t in (q, k, v))
    plan = core.plan_varblock(bm.to(cuda), qcnt, kcnt, S, gather=True)
    o, lse = core.attn_fwd_fp8(q8, k8, v8, sq, sk, sv, plan, q_rows=qperm, kv_rows=kperm, o_rows=qperm,
                               return_lse=True)
    o, lse = o.float().cpu(), lse.cpu()
    qp, kp = qperm.cpu().long(), kperm.cpu().long()
    qd, kd, vd = _deq(q8, sq), _deq(k8, sk), _deq(v8, sv)
    # the oracle runs in cluster order: gather the de-quantised rows, and read the kernel's output through q_perm
    qd = torch.stack([qd[0, h, qp[h]] for h in range(H)])[None]
    kd = torch.stack([kd[0, h, kp[h]] for h in range(H)])[None]
    vd = torch.stack([vd[0, h, kp[h]] for h in range(H)])[None]
    ref, ref_lse = oa.dynamic_block_sparse_fwd(qd, kd, vd, bm[None], qcnt.cpu()[None], kcnt.cpu()[None],
                                               return_lse=True, dtype=torch.float64)
    o = torch.stack([o[0, h, qp[h]] for h in range(H)])
    lse = torch.stack([lse[h, qp[h]] for h in range(H)])
    empty_rows = ref_lse[0, 2] == float("-inf")
    assert bool(empty_rows.any())
    assert bool((o[2][empty_rows] == 0).all())
    for h in range(H):
        torch.testing.assert_close(o[h] / fv[h], (ref[0, h] / fv[h]).float(), **FP8_TOL)
    _check_lse(lse, ref_lse[0])


def test_fp8_gather_fused_permutation_is_exact(cuda):
    """Gathering e4m3 rows through q_rows / kv_rows is bit-identical to running the same plan with identity rows on
    the same bytes permuted beforehand."""
    from svgb200 import core

    g = torch.Generator().manual_seed(32)
    H, S, D, QC, KC = 3, 5000, 128, 29, 77
    bm, qperm, qcnt, kperm, kcnt = _clusters(cuda, H, S, QC, KC, g)
    q, k, v, _ = _scaled_qkv(H, S, D, g)
    (q8, sq), (k8, sk), (v8, sv) = (core.quantize_e4m3(t.to(cuda)) for t in (q, k, v))
    plan = core.plan_varblock(bm.to(cuda), qcnt, kcnt, S, gather=True)
    o1, l1 = core.attn_fwd_fp8(q8, k8, v8, sq, sk, sv, plan, q_rows=qperm, kv_rows=kperm, o_rows=qperm,
                               return_lse=True)

    def permuted(x8, perm):  # e4m3 bytes moved as 16-bit pairs
        return core.permute_gather(x8.view(torch.int16), perm).view(torch.uint8)
    q8p, k8p, v8p = permuted(q8, qperm), permuted(k8, kperm), permuted(v8, kperm)
    o2, l2 = core.attn_fwd_fp8(q8p, k8p, v8p, sq, sk, sv, plan, o_rows=qperm, return_lse=True)
    assert torch.equal(o1.view(torch.int16), o2.view(torch.int16))
    assert torch.equal(l1, l2)


def test_census_fp8_gather_plan(cuda):
    """The census of tests/test_attention_census_gpu.py (q = 0, one-hot key-identity V) on an FP8 gather plan with
    q_rows / kv_rows / o_rows: every row's output bit for bit and exp(lse) against the key count."""
    from oracle import census as oc
    from svgb200 import core
    from test_attention_census_gpu import bound_ok, check_census

    g = torch.Generator().manual_seed(33)
    H, S, D, QC, KC = 3, 6000, 128, 37, 101
    bm, qperm, qcnt, kperm, kcnt = _clusters(cuda, H, S, QC, KC, g)
    plan = core.plan_varblock(bm.to(cuda), qcnt, kcnt, S, gather=True)
    cnt, n = [], []
    for h in range(H):
        c, nn = oc.scatter_rows(*oc.blockmap_census(bm[h], qcnt[h].cpu(), kcnt[h].cpu(), D, kperm[h].cpu()),
                                qperm[h].cpu())
        cnt.append(c)
        n.append(nn)
    bound_ok(cnt, torch.bfloat16)
    q8 = torch.zeros(1, H, S, D, dtype=torch.uint8, device=cuda)
    k8, sk = core.quantize_e4m3(torch.randn(1, H, S, D, device=cuda).bfloat16())
    sq = torch.tensor([0.5, 3.0, 1.0], device=cuda)
    sv = torch.ones(H, device=cuda)
    for enc in oc.ENCODINGS:
        v8 = oc.identity_values(S, D, enc, H, torch.float8_e4m3fn, cuda).view(torch.uint8)
        o, lse = core.attn_fwd_fp8(q8, k8, v8, sq, sk, sv, plan, q_rows=qperm, kv_rows=kperm, o_rows=qperm,
                                   return_lse=True)
        check_census(o[0], lse, cnt, n, enc, "fp8 gather plan")


def test_rows_need_a_gather_plan(cuda):
    from svgb200 import core

    H, S, D = 1, 512, 128
    q8 = torch.zeros(1, H, S, D, dtype=torch.uint8, device=cuda)
    s = torch.ones(H, device=cuda)
    sz = torch.tensor([[S]], dtype=torch.int32, device=cuda)
    plan = core.plan_varblock(torch.ones(H, 1, 1, dtype=torch.bool, device=cuda), sz, sz, S)
    rows = torch.arange(S, dtype=torch.int32, device=cuda)[None]
    with pytest.raises(core.SvgbError, match="gather plan"):
        core.attn_fwd_fp8(q8, q8, q8, s, s, s, plan, q_rows=rows)


# ---------------------------------------------------------------------------------------------------------------
# cores
# ---------------------------------------------------------------------------------------------------------------
def _clustered_inputs(cuda, H, S, D, seed, dtype=torch.bfloat16):
    g = torch.Generator(device=cuda).manual_seed(seed)
    q, k, v = (torch.randn(1, H, S, D, device=cuda, generator=g) for _ in range(3))
    base = torch.randn(1, H, 16, D, device=cuda, generator=g) * 1.5
    which = torch.randint(0, 16, (S,), device=cuda, generator=g)
    return (q * 0.7 + base[:, :, which]).to(dtype), (k * 0.7 + base[:, :, which]).to(dtype), v.to(dtype)


def _labels_from(perm, sizes):
    lab = torch.empty(perm.shape[0], dtype=torch.long, device=perm.device)
    lab[perm.long()] = torch.repeat_interleave(torch.arange(sizes.shape[0], device=perm.device), sizes.long())
    return lab


def _sap_pair(model, cuda, **kw):
    from svgb200.models import hyvideo as hy
    from svgb200.models import wan

    common = dict(num_q_centroids=12, num_k_centroids=40, top_p_kmeans=0.9, min_kc_ratio=0.1, kmeans_iter_init=3,
                  kmeans_iter_step=2, **kw)
    if model == "wan":
        F, P, ctx = 6, 400, 0
        make = lambda fp8: wan.WanSAPCore(F, P, fp8=fp8, **common)  # noqa: E731
    else:
        F, P, ctx = 4, 300, 64
        make = lambda fp8: hy.HunyuanSAPCore(ctx, F, P, prompt_length=20, fp8=fp8, **common)  # noqa: E731
    return make(False), make(True), ctx + F * P


@pytest.mark.parametrize("model", ["wan", "hunyuan"])
def test_sap_core_fp8_keeps_the_16bit_maps(cuda, model):
    """WanSAPCore / HunyuanSAPCore with fp8=True against the 16-bit core on identical inputs and identical initial
    centroids, over a cold and a warm step: map, sizes and both permutations bit-identical; sampled rows of the FP8
    output agree with the fp64 oracle on the de-quantised inputs under the engine's map."""
    from svgb200 import core

    H, D = 3, 128
    ref_core, fp8_core, S = _sap_pair(model, cuda)
    q, k, v = _clustered_inputs(cuda, H, S, D, 40)
    (q8, sq), (k8, sk), (v8, sv) = (core.quantize_e4m3(t) for t in (q, k, v))
    qd, kd, vd = _deq(q8, sq)[0], _deq(k8, sk)[0], _deq(v8, sv)[0]
    rows = torch.randint(0, S, (64,), generator=torch.Generator().manual_seed(1))
    rows[0] = S - 1  # a text row (HunyuanVideo)
    for step in range(2):
        torch.manual_seed(step)
        o_ref = ref_core.sparse_core(q, k, v)
        torch.manual_seed(step)
        o = fp8_core.sparse_core(q, k, v)
        assert o.dtype == torch.bfloat16 and o.shape == o_ref.shape
        for name in ("dynamic_map", "q_sizes", "k_sizes", "q_sorted_indices", "k_sorted_indices"):
            assert torch.equal(fp8_core.last[name], ref_core.last[name]), name
        m, rs, cs = (fp8_core.last[x] for x in ("dynamic_map", "q_sizes", "k_sizes"))
        qperm, kperm = fp8_core.last["q_sorted_indices"], fp8_core.last["k_sorted_indices"]
        for h in range(H):
            ql, kl = _labels_from(qperm[h], rs[h]).cpu(), _labels_from(kperm[h], cs[h]).cpu()
            allowed = m[h].cpu()[ql[rows]][:, kl]
            s = (qd[h, rows] @ kd[h].T) * D ** -0.5
            w = torch.nan_to_num(torch.softmax(s.masked_fill(~allowed, float("-inf")), -1), nan=0.0)
            torch.testing.assert_close(o[0, h, rows].float().cpu(), (w @ vd[h]).float(), **FP8_TOL)


def test_svg1_core_fp8_equals_the_hand_built_chain(cuda):
    """HunyuanSVG1Core(fp8=True): the same head choice as the 16-bit core, and an output equal bit for bit to
    placement -> quantise -> attn_fwd_fp8 on the band plan -> inverse placement."""
    from svgb200 import core
    from svgb200.models import hyvideo as hy

    H, F, P, ctx, plen, D = 4, 5, 260, 64, 20, 128
    S = ctx + F * P
    kw = dict(num_sampled_rows=32, sample_mse_max_row=1000)
    ref_core = hy.HunyuanSVG1Core(ctx, plen, F, P, H, D, 0.25, cuda, **kw)
    fp8_core = hy.HunyuanSVG1Core(ctx, plen, F, P, H, D, 0.25, cuda, fp8=True, **kw)
    q, k, v = _clustered_inputs(cuda, H, S, D, 41)
    k[:, :2] = (k[:, :2].float() * 0.2 + q[:, :2].float()).to(k.dtype)  # heads with local structure
    rows = torch.randint(0, 1000, (32,), generator=torch.Generator().manual_seed(2))
    best = torch.argmin(fp8_core.sample_mse(q, k, v, rows), dim=0)
    assert torch.equal(best, torch.argmin(ref_core.sample_mse(q, k, v, rows), dim=0))
    o = fp8_core.sparse_core(q, k, v, sampled_rows=rows)
    placed = [torch.empty_like(t) for t in (q, k, v)]
    core.head_placement([q, k, v], placed, best, ctx, F, P)
    (q8, sq), (k8, sk), (v8, sv) = (core.quantize_e4m3(t) for t in placed)
    hid = core.attn_fwd_fp8(q8, k8, v8, sq, sk, sv, fp8_core.block_mask.plan)
    want = torch.empty_like(q)
    core.head_placement([hid], [want], best, ctx, F, P, inverse=True)
    assert torch.equal(o.view(torch.int16), want.view(torch.int16))


def test_dense_branch_is_the_16bit_one(cuda):
    """fp8=True leaves the dense branch of both cores untouched: bit-identical to the 16-bit cores."""
    from svgb200.models import hyvideo as hy

    H, F, P, ctx, plen, D = 2, 4, 150, 40, 17, 128
    S = ctx + F * P
    q, k, v = _clustered_inputs(cuda, H, S, D, 42)
    cu = torch.tensor([0, F * P + plen, S], dtype=torch.int32, device=cuda)
    t = torch.tensor([950.0])
    outs = []
    for fp8 in (False, True):
        svg1 = hy.HunyuanSVG1Core(ctx, plen, F, P, H, D, 0.3, cuda, first_times_fp=900, fp8=fp8)
        sap = hy.HunyuanSAPCore(ctx, F, P, num_q_centroids=6, num_k_centroids=12, top_p_kmeans=0.9, min_kc_ratio=0.1,
                                kmeans_iter_init=3, kmeans_iter_step=1, prompt_length=plen, first_times_fp=900,
                                fp8=fp8)
        outs.append((svg1.attention_core_logic(q, k, v, t, 0, (cu, cu, S, S)),
                     sap.attention_core_logic(q, k, v, t, 0, (cu, cu, S, S))))
    for a, b in zip(*outs):
        assert torch.equal(a, b)


def test_fp16_in_fp16_out(cuda):
    """The FP8 kernel writes bf16; the cores hand fp16 callers fp16."""
    from svgb200.models import wan

    H, F, P, D = 2, 4, 300, 128
    S = F * P
    q, k, v = _clustered_inputs(cuda, H, S, D, 43, torch.float16)
    sap = wan.WanSAPCore(F, P, num_q_centroids=8, num_k_centroids=20, top_p_kmeans=0.9, min_kc_ratio=0.1,
                         kmeans_iter_init=3, kmeans_iter_step=1, fp8=True)
    svg1 = wan.WanSVG1Core(F, P, H, D, 0.3, cuda, dtype=torch.float16, num_sampled_rows=16, sample_mse_max_row=S,
                           fp8=True)
    for c in (sap, svg1):
        o = c.sparse_core(q, k, v)
        assert o.dtype == torch.float16 and bool(torch.isfinite(o).all())


def test_head_dim_64_is_rejected(cuda):
    from svgb200 import core
    from svgb200.models import cog

    ctx, F, P, H, D = 40, 4, 200, 2, 64
    S = ctx + F * P
    svg1 = cog.CogSVG1Core(ctx, F, P, H, D, 0.3, cuda, fp8=True)
    q = torch.randn(1, H, S, D, device=cuda).bfloat16()
    with pytest.raises(core.SvgbError, match="head_dim 128"):
        svg1.sparse_core(q, q, q)


# ---------------------------------------------------------------------------------------------------------------
# drop-in patch
# ---------------------------------------------------------------------------------------------------------------
def test_install_fp8_calls_equal_the_core_calls(cuda):
    """install(..., fp8=True) on a stand-in of a reference attention module: the installed flex_attention and
    dynamic_block_sparse_fwd_flashinfer / _triton equal quantise + attn_fwd_fp8 bit for bit."""
    import types

    from svgb200 import core, patch
    from svgb200.models import wan

    mod = types.ModuleType("svg.models.wan.attention")
    for name in ("flex_attention", "dynamic_block_sparse_fwd_flashinfer", "dynamic_block_sparse_fwd_triton"):
        setattr(mod, name, None)
    patch.install(mod, fp8=True)
    H, F, P, D = 2, 5, 300, 128
    S = F * P
    q, k, v = _clustered_inputs(cuda, H, S, D, 44)
    (q8, sq), (k8, sk), (v8, sv) = (core.quantize_e4m3(t) for t in (q, k, v))
    bm = wan.prepare_flexattention(1, H, D, torch.bfloat16, cuda, 0, 0, F, P, diag_width=1.2, multiplier=1.2)
    want = core.attn_fwd_fp8(q8, k8, v8, sq, sk, sv, bm.plan)
    assert torch.equal(mod.flex_attention(q, k, v, block_mask=bm).view(torch.int16), want.view(torch.int16))
    g = torch.Generator().manual_seed(45)
    QC, KC = 7, 19

    def part(n):
        cuts = torch.sort(torch.randperm(S - 1, generator=g)[: n - 1] + 1)[0]
        return torch.diff(torch.cat([torch.tensor([0]), cuts, torch.tensor([S])])).to(torch.int32)
    row = torch.stack([part(QC) for _ in range(H)])[None]
    col = torch.stack([part(KC) for _ in range(H)])[None]
    m = torch.rand(1, H, QC, KC, generator=g) < 0.5
    plan = core.plan_varblock(m[0].to(cuda), row[0].to(cuda), col[0].to(cuda), S)
    want = core.attn_fwd_fp8(q8, k8, v8, sq, sk, sv, plan)
    for fn in (mod.dynamic_block_sparse_fwd_flashinfer, mod.dynamic_block_sparse_fwd_triton):
        assert torch.equal(fn(q, k, v, m, row, col).view(torch.int16), want.view(torch.int16))
