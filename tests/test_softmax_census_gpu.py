"""Exact census of the attention kernel's online softmax, on every row of every head (oracle/softmax.py).

Integer Q and K put every score on an integer grid with hot keys 160 (after c) above cold ones, and keys that rise in
t along the kernel's visit order: rows meet cold keys first, are wiped to exactly 0 by the alpha of their first hot
chunk, and then rescale by 1/2 .. 1/8 as the max rises.  Every p, alpha and partial sum is exact, so the output must
equal round16(O * (1/l * v_scale)) of the closed form BIT FOR BIT and the lse must lie within log2f's one-ulp error of
(M c + log2 l) ln 2.  A wrong alpha, a rescale of the wrong chunk or row, a stale l, a P packed from the wrong chunk
or in the wrong format, or a wrong per-head scale changes bits; a correct reordering of the chunk loop does not.
The budget, coverage and sensitivity of every case are shown on the CPU (tests/test_softmax_census_cpu.py).

Together the cases run all ten kernel instantiations: D 64 / 128 x bf16 / fp16 x TMA / row gather, and e4m3 with both
loaders.  The three premise tests are the smallest cases of the facts the design rests on, so that a failure points
at the premise rather than at the chunk loop.
"""
import pytest
import torch

from oracle import softmax as sm

pytestmark = pytest.mark.gpu

DT = {"bf16": torch.bfloat16, "fp16": torch.float16}


def _plan(cuda, case):
    from svgb200 import core
    from svgb200.ops import attention_ops

    if "bsr" in case.notes:
        F, P, text, Rb = case.notes["bsr"]
        plan = attention_ops.bsr_to_plan(case.notes["indptr"], case.notes["indices"], (Rb, Rb), F * P, text, cuda)
        assert plan.desc.items_stride == 0
        return plan
    if case.mod is not None:
        return core.plan_band(*case.band, case.H, case.S, cuda)
    return core.plan_varblock(case.bm.to(cuda), case.rows.to(cuda), case.cols.to(cuda), case.S, gather=case.gather)


def check(cuda, case, o, lse, what):
    """o [H, S, D] and lse [H, S] in output-row order against the closed form; names the first differing
    (head, row, column)."""
    o, lse = o.cpu(), lse.cpu()
    for h in range(case.H):
        O, l, m_raw, budget = sm.expected(case, h, device=cuda)
        assert float(budget.max()) < sm.BUDGET, f"{what}: head {h} leaves the exact range"
        O, l, m_raw = sm.to_output_rows(case, h, O, l, m_raw)
        exp_o = sm.expected_output(O, l, case.vs[h], o.dtype)
        lo, hi = sm.lse_bounds(m_raw, l, case.c[h])
        bad_o = (o[h].view(torch.int16) != exp_o.view(torch.int16)).any(1)
        got = lse[h]
        bad_l = torch.where(l > 0, ~((got >= lo) & (got <= hi)), got != float("-inf"))
        bad = bad_o | bad_l
        if bool(bad.any()):
            r = int(bad.nonzero()[0])
            col = int((o[h, r].view(torch.int16) != exp_o[r].view(torch.int16)).nonzero()[0]) if bad_o[r] else 0
            raise AssertionError(
                f"{what}: first differing (head {h}, row {r}, column {col}) of {int(bad_o.sum())} output rows and "
                f"{int(bad_l.sum())} lse rows: expected {float(exp_o[r, col])!r} (O = {float(O[r, col])!r}, "
                f"l = {float(l[r])!r}), kernel {float(o[h, r, col])!r}; lse expected in [{float(lo[r])!r}, "
                f"{float(hi[r])!r}] (exact {float(sm.exact_lse(m_raw[r:r + 1], l[r:r + 1], case.c[h])[0])!r}), "
                f"kernel {float(got[r])!r}")


def run(cuda, case, dtype, what, sm_scale=1.0, layout="bhsd"):
    """16-bit inputs; sm_scale is the target c (every head's c must be it)."""
    from svgb200 import core

    scale = sm.scale_for(sm_scale)
    assert all(c == sm.kernel_c(scale) for c in case.c)
    plan = _plan(cuda, case)
    q, k, v = (t.to(dtype).to(cuda) for t in case.tensors())
    kw = dict(return_lse=True, sm_scale=scale)
    if case.o_rows is not None:
        kw["o_rows"] = case.o_rows.to(cuda)
    if case.gather:
        kw["q_rows"], kw["kv_rows"] = case.q_rows.to(cuda), case.kv_rows.to(cuda)
    if layout == "shd":
        q, k, v = (t.transpose(0, 1).contiguous() for t in (q, k, v))
        o, lse = core.attn_fwd(q, k, v, plan, layout="shd", **kw)
        o = o.transpose(0, 1)
    else:
        o, lse = core.attn_fwd(q[None], k[None], v[None], plan, **kw)
        o = o[0]
    check(cuda, case, o, lse, what)


def run_fp8(cuda, case, what):
    """e4m3 inputs with the per-head scales of oracle.softmax (FP8_QS, FP8_KS, FP8_VS); c = 1 from sm_scale."""
    from svgb200 import core

    scale = sm.scale_for(1.0)
    assert case.c == sm.FP8_C and case.vs == sm.FP8_VS
    plan = _plan(cuda, case)
    q8, k8, v8 = (t.to(torch.float8_e4m3fn).view(torch.uint8)[None].to(cuda) for t in case.tensors())
    qs, ks, vs = (torch.tensor(x, dtype=torch.float32, device=cuda) for x in (sm.FP8_QS, sm.FP8_KS, sm.FP8_VS))
    kw = {}
    if case.o_rows is not None:
        kw["o_rows"] = case.o_rows.to(cuda)
    if case.gather:
        kw["q_rows"], kw["kv_rows"] = case.q_rows.to(cuda), case.kv_rows.to(cuda)
    o, lse = core.attn_fwd_fp8(q8, k8, v8, qs, ks, vs, plan, return_lse=True, sm_scale=scale, **kw)
    check(cuda, case, o[0], lse, what)


# --------------------------------------------------------------------------------------------
# premises, each in its own one-chunk case
# --------------------------------------------------------------------------------------------
def test_premise_ex2_exact_at_integers(cuda):
    """(a) ex2.approx.ftz.f32 gives 2^x exactly at x in {-3, .., 0} and 0 at x <= -157: four hot keys per row with
    p = 1/8 .. 1, each alone in its V column (V = identity), and 124 cold keys whose p must be 0."""
    run(cuda, sm.premise_case("ex2"), torch.bfloat16, "premise ex2")


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("D", [64, 128])
def test_premise_wgmma_accumulation_exact(cuda, D, dtype):
    """(b) the 16-bit P V wgmma sums integer products exactly while every partial sum is representable: p = 1 for all
    128 keys and V in [-4, 4]."""
    run(cuda, sm.premise_case("accum", D), DT[dtype], f"premise accumulation D={D} {dtype}")


def test_premise_e4m3_qk_exact(cuda):
    """(c) the e4m3 Q K^T wgmma is exact for integer scores below 2^9: one hot key per row (scores up to 326), so
    O = v_r * v_scale, l = 1 and the lse is M c ln 2 itself; c = 2 on head 0 and 1/2 on head 1."""
    run_fp8(cuda, sm.premise_case("e4m3_qk"), "premise e4m3 Q K^T")


# --------------------------------------------------------------------------------------------
# band plans
# --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("name", list(sm.BAND))
def test_softmax_band(cuda, name, D, dtype):
    """HunyuanVideo (text last), Wan (sink), CogVideoX with and without the sink, the generic widths 254 / 255 and mode
    NONE, at S not a multiple of 128; two heads."""
    run(cuda, sm.band_case(name, D=D), DT[dtype], f"band {name} D={D} {dtype}")


def test_softmax_band_hunyuan_720p(cuda):
    """HunyuanVideo 720p: S = 119 056, D = 128, bf16, 30 % density, one head; regions of 4096 keys."""
    run(cuda, sm.band_case("hy720", H=1), torch.bfloat16, "band HunyuanVideo 720p")


@pytest.mark.parametrize("c", [0.5, 2.0])
def test_softmax_scale(cuda, c):
    """sm_scale giving c = 1/2 and c = 2 exactly: the scale reaches the exponents unrounded (HunyuanVideo band)."""
    run(cuda, sm.band_case("hy", c=[c, c]), torch.bfloat16, f"band hy c={c}", sm_scale=c)


# --------------------------------------------------------------------------------------------
# variable-block, gather and shared plans
# --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("D", [64, 128])
def test_softmax_varblock(cuda, D, dtype):
    """Variable-block TMA plan: q_sizes edge sizes (every r % 256 class, empty q-blocks, an odd tail count, so one
    CTA runs a single stream), runs across empty key blocks, an all-empty q-block; output through o_rows."""
    run(cuda, sm.varblock_case(D=D), DT[dtype], f"varblock D={D} {dtype}")


def test_softmax_varblock_shd(cuda):
    """The same plan in the [S, H, D] layout of the ops API."""
    run(cuda, sm.varblock_case(), torch.bfloat16, "varblock shd", layout="shd")


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("D", [64, 128])
def test_softmax_gather(cuda, D, dtype):
    """Row-gather plan through q_rows / kv_rows / o_rows (cluster argsorts), with an empty query and key cluster, a
    query cluster that sees nothing and one that sees everything."""
    run(cuda, sm.gather_case(D=D), DT[dtype], f"gather D={D} {dtype}")


def test_softmax_bsr_shared_plan(cuda):
    """One BSR plan for both heads (items_stride = 0)."""
    run(cuda, sm.bsr_case(), torch.bfloat16, "shared BSR plan")


# --------------------------------------------------------------------------------------------
# FP8 (e4m3): per-head q_scale * k_scale = 2 and 1/2, v_scale 1/2 and 2
# --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["band", "varblock", "gather"])
def test_softmax_fp8(cuda, kind):
    if kind == "band":
        case = sm.band_case("hy", c=sm.FP8_C, vs=sm.FP8_VS)
    elif kind == "varblock":
        case = sm.varblock_case(c=sm.FP8_C, vs=sm.FP8_VS)
    else:
        case = sm.gather_case(c=sm.FP8_C, vs=sm.FP8_VS)
    run_fp8(cuda, case, f"fp8 {kind}")

