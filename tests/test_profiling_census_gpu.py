"""Exact census of the SVG1 profiling masks (MASK_PROF_*, the element masks of sample_mse) run through band plans.

Same method as test_attention_census_gpu.py (oracle/census.py): q = 0 and a one-hot key-identity V make the kernel's
output and LSE a bit-exact function of the key set each row executed.  The expected key sets come from the oracle's
restatement of the reference's get_attention_mask (oracle.attention.profiling_mask_rows / profiling_mask_rows_cog),
never from the engine, so one key wrongly kept or dropped anywhere fails.  Every sample_mse profiling pass runs these
masks on chunks that are all element-masked.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu


def prof_params(layout, name, ctx, F, P):
    """(mode, m0, m1, m2) of the profiling mask as sample_mse builds it (sample_mse.cu)."""
    from svgb200 import core

    modes = {"hy": (core.MASK_PROF_HY_S, core.MASK_PROF_HY_T), "wan": (core.MASK_PROF_WAN_S, core.MASK_PROF_WAN_T),
             "cog": (core.MASK_PROF_COG_S, core.MASK_PROF_COG_T)}
    mode = modes[layout][name == "temporal"]
    thres = (2 * P) // 128 if layout == "wan" else int(1.5 * P / 128.0)
    return mode, F, P, (thres | (ctx << 12)) if layout == "cog" else thres


def oracle_rows(layout, name, ctx, F, P, rows):
    """bool [len(rows), S] on the CPU"""
    from oracle import attention as oa

    if layout == "cog":
        return oa.profiling_mask_rows_cog(name, rows, ctx, F, P)
    return oa.profiling_mask_rows(name, rows, layout, ctx, F, P)


def run_prof_census(cuda, layout, name, ctx, F, P, H, D, rows=None):
    """Kernel over all S rows with the band plan of the profiling mask; compares `rows` (default: all of them)."""
    from oracle import census as oc
    from svgb200 import core

    S = ctx + F * P
    rows = torch.arange(S) if rows is None else rows
    plan = core.plan_band(*prof_params(layout, name, ctx, F, P), H, S, cuda)
    q = torch.zeros(1, H, S, D, dtype=torch.float16, device=cuda)
    k = torch.randn(1, H, S, D, device=cuda).half()
    m = torch.cat([oracle_rows(layout, name, ctx, F, P, rows[i:i + 1024]).to(cuda) for i in range(0, len(rows), 1024)])
    n = m.sum(1).cpu()
    for enc in oc.ENCODINGS:
        codes = oc.key_codes(S, D, enc, cuda)
        cnt = torch.zeros(len(rows), D, device=cuda).index_add_(1, codes, m.float()).to(torch.int32).cpu()
        assert int(cnt.max()) < oc.COUNT_LIMIT[torch.float16]
        exp_o = oc.expected_output(cnt, n, torch.float16)
        v = oc.identity_values(S, D, enc, H, torch.float16, cuda)
        o, lse = core.attn_fwd(q, k, v, plan, return_lse=True)
        rc = rows.to(cuda)
        for h in range(H):
            oh = o[0, h, rc].cpu()
            lh = lse[h, rc].cpu().double()
            bad_o = (oh.view(torch.int16) != exp_o.view(torch.int16)).any(1)
            bad_l = torch.where(n > 0, ~((lh.exp() - n.double()).abs() < 0.5), lh != float("-inf"))
            bad = bad_o | bad_l
            if bool(bad.any()):
                i = int(bad.nonzero()[0])
                raise AssertionError(
                    f"{layout} {name} ctx={ctx} F={F} P={P} D={D}, encoding {enc}: {int(bad.sum())} rows differ, first "
                    f"(head {h}, row {int(rows[i])}): expected {int(n[i])} keys, exp(lse) = {float(lh[i].exp()):.3f}")


@pytest.mark.parametrize("name", ["spatial", "temporal"])
@pytest.mark.parametrize("case", [
    # layout, ctx, F, P.  P = 200, 180, 260, 80: frames that do not line up with the 128-key chunks;
    # P = 80 gives thres = 0 (HY keeps only the text; COG temporal rows see no key at all)
    ("hy", 48, 6, 200), ("hy", 64, 5, 256), ("hy", 20, 9, 80), ("wan", 0, 7, 180), ("wan", 0, 4, 384),
    ("cog", 40, 4, 260), ("cog", 226, 3, 1350), ("cog", 20, 9, 80)])
@pytest.mark.parametrize("D", [64, 128])
def test_census_profiling_small(cuda, case, name, D):
    layout, ctx, F, P = case
    run_prof_census(cuda, layout, name, ctx, F, P, 2, D)


@pytest.mark.parametrize("name", ["spatial", "temporal"])
def test_census_profiling_hunyuan_720p(cuda, name):
    """One head at HunyuanVideo 720p (S = 256 + 33 x 3600, P = 3600 = 28 x 128 + 16): every text row, the rows at
    the edges of frames and of 128-row blocks, and 2048 random video rows."""
    ctx, F, P = 256, 33, 3600
    V = F * P
    g = torch.Generator().manual_seed(3)
    edges = torch.cat([torch.arange(0, V, P), torch.arange(P - 1, V, P), torch.arange(0, V, 128), torch.arange(127, V, 128)])
    rows = torch.cat([torch.randint(0, V, (2048,), generator=g), edges, torch.arange(V, V + ctx)]).unique()
    run_prof_census(cuda, "hy", name, ctx, F, P, 1, 128, rows)
