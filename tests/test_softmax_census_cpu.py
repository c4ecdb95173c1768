"""CPU proof that the softmax census (tests/test_softmax_census_gpu.py, oracle/softmax.py) is exact and sees the bugs
it is meant to see.

  * the scale constants give c exactly, and the e4m3 scale products are exact powers of two;
  * every GPU case is exact: integer inputs representable in its formats, a hot / cold gap of at least 150 after c,
    and every row's partial sums inside the 2^22 budget;
  * coverage: on the kernel's visit order, most rows with keys are wiped by their first hot chunk and then rescale at
    least twice by a partial alpha; some rows only ever see cold keys, some see no key, and band rows of an item's
    second stream are covered;
  * the chunk-loop simulation reproduces the closed form on every row it visits (oracle.softmax.coverage);
  * sensitivity: outputs of oracle mutants of the chunk loop differ from the true ones, in output bits or beyond the
    lse tolerance, on a stated fraction of rows.
"""
import numpy as np
import pytest
import torch

from oracle import softmax as sm


@pytest.mark.parametrize("c", [0.5, 1.0, 2.0])
def test_scale_constant_gives_c_exactly(c):
    s = sm.scale_for(c)
    assert sm.kernel_c(s) == c
    assert float(np.float32(s)) == s  # an fp32 value: the C ABI's float carries it unchanged
    for nb in (np.nextafter(np.float32(s), np.float32(0)), np.nextafter(np.float32(s), np.float32(4))):
        assert sm.kernel_c(float(nb)) != c


def test_fp8_scales_are_exact():
    """e4m3 heads: q_scale * k_scale = 2 and 1/2, different v_scales, all powers of two, so c stays exact."""
    assert sm.FP8_C == [2.0, 0.5]
    assert sm.FP8_VS[0] != sm.FP8_VS[1]
    for x in sm.FP8_QS + sm.FP8_KS + sm.FP8_VS:
        assert np.log2(x) == int(np.log2(x))


# (builder, input formats, row stride of the coverage walk, stated coverage)
CASES = {
    "hy": (lambda: sm.band_case("hy"), ("bf16", "fp16"), 1, 0.75),
    "wan": (lambda: sm.band_case("wan"), ("bf16", "fp16"), 1, 0.65),
    "cog": (lambda: sm.band_case("cog"), ("bf16", "fp16"), 1, 0.79),
    "cog_sink": (lambda: sm.band_case("cog_sink"), ("bf16", "fp16"), 1, 0.79),
    "generic_254": (lambda: sm.band_case("generic_254"), ("bf16", "fp16"), 1, 0.59),
    "generic_255": (lambda: sm.band_case("generic_255"), ("bf16", "fp16"), 1, 0.51),
    "none": (lambda: sm.band_case("none"), ("bf16", "fp16"), 1, 0.70),
    "hy720": (lambda: sm.band_case("hy720", H=1), ("bf16",), 467, 0.90),
    "hy_c0.5": (lambda: sm.band_case("hy", c=[0.5, 0.5]), ("bf16",), 1, 0.75),
    "hy_c2": (lambda: sm.band_case("hy", c=[2.0, 2.0]), ("bf16",), 1, 0.75),
    "varblock": (lambda: sm.varblock_case(), ("bf16", "fp16"), 7, 0.90),
    "gather": (lambda: sm.gather_case(), ("bf16", "fp16"), 7, 0.90),
    "bsr": (lambda: sm.bsr_case(), ("bf16",), 1, 0.72),
    "fp8_band": (lambda: sm.band_case("hy", c=sm.FP8_C, vs=sm.FP8_VS), ("e4m3",), 1, 0.75),
    "fp8_varblock": (lambda: sm.varblock_case(c=sm.FP8_C, vs=sm.FP8_VS), ("e4m3",), 7, 0.90),
    "fp8_gather": (lambda: sm.gather_case(c=sm.FP8_C, vs=sm.FP8_VS), ("e4m3",), 7, 0.90),
    "premise_ex2": (lambda: sm.premise_case("ex2"), ("bf16",), 1, None),
    "premise_accum": (lambda: sm.premise_case("accum"), ("bf16", "fp16"), 1, None),
    "premise_e4m3_qk": (lambda: sm.premise_case("e4m3_qk"), ("e4m3",), 1, None),
}
FMT = {"bf16": torch.bfloat16, "fp16": torch.float16, "e4m3": torch.float8_e4m3fn}


@pytest.mark.parametrize("name", list(CASES))
def test_case_is_exact(name):
    """Inputs exact in every format the case runs in, the hot / cold gap >= 150 after c, the budget below 2^22 (on
    every row; the HunyuanVideo 720p case on every 97th row here and on all rows in the GPU test)."""
    build, fmts, _, _ = CASES[name]
    case = build()
    assert int(case.kcls.max()) < case.D - 1 and int(case.kt.max()) <= case.R
    for h in range(case.H):
        a, b = sm.qk_ints(case.c[h])
        e = b * case.c[h]
        assert 16 * a * case.c[h] == sm.GAP and sm.GAP - e * case.R >= sm.MIN_GAP
        # every score is below 2^9 (the e4m3 premise) and a tier spans at most 2^(e R)
        assert 16 * a + b * case.R < 512 and e * case.R <= 6
    for f in fmts:
        for t in case.tensors():
            assert torch.equal(t.to(FMT[f]).float(), t), f
    rows = list(range(0, case.S, 97)) if case.S > 100000 else None
    for h in range(case.H):
        budget = sm.expected(case, h, row_ids=rows)[3]
        assert float(budget.max()) < sm.BUDGET


@pytest.mark.parametrize("name", [n for n, c in CASES.items() if c[3] is not None])
def test_coverage(name):
    """The stated fraction of rows with keys is wiped and then partially rescaled at least twice with O != 0, in the
    kernel's visit order (the order does not depend on D or the format).  Every case has cold-only rows."""
    build, _, stride, frac = CASES[name]
    case = build()
    st = sm.coverage(case, stride)
    assert st["covered"] >= frac * st["keyed"], st
    assert st["cold_only"] > 0, st
    if case.mod is not None:
        assert st["stream1"] > 0, st
    if name in ("varblock", "gather"):
        assert st["keyless"] > 0, st


# --------------------------------------------------------------------------------------------
# sensitivity on oracle mutants
# --------------------------------------------------------------------------------------------
def _differs(case, h, r, O, l, m, O2, l2, m2):
    """Whether a mutant's (O2, l2, m2) of one row shows in the output bits or beyond the lse tolerance."""
    out = sm.expected_output(torch.tensor(O)[None], torch.tensor([l]), case.vs[h], torch.bfloat16)
    out2 = sm.expected_output(torch.tensor(O2)[None], torch.tensor([l2]), case.vs[h], torch.bfloat16)
    if not torch.equal(out.view(torch.int16), out2.view(torch.int16)):
        return True
    mr = torch.tensor([m / case.c[h]])
    lo, hi = sm.lse_bounds(mr, torch.tensor([l], dtype=torch.float64), case.c[h])
    lo2, hi2 = sm.lse_bounds(torch.tensor([m2 / case.c[h]]), torch.tensor([l2], dtype=torch.float64), case.c[h])
    return bool(hi2[0] < lo[0] or lo2[0] > hi[0])


# mutant -> stated fraction of rows with keys whose output or lse changes (band hy and varblock cases)
MUTANTS = {"prev_alpha": 0.6, "l_once": 0.6, "drop_hot": 0.9}


@pytest.mark.parametrize("case_name", ["hy", "varblock"])
@pytest.mark.parametrize("mutant", list(MUTANTS))
def test_chunk_loop_mutants_are_seen(mutant, case_name):
    """O rescaled with the previous chunk's alpha; l not rescaled at the row's last partial rescale; the row's first
    hot key dropped."""
    case = sm.band_case("hy") if case_name == "hy" else sm.varblock_case()
    stride = 1 if case_name == "hy" else 9
    keyed = seen = 0
    for h in range(case.H):
        for r in range(0, case.S, stride):
            O, l, m, _ = sm.simulate(case, h, r)
            if l == 0:
                continue
            keyed += 1
            O2, l2, m2, _ = sm.simulate(case, h, r, mutant)
            seen += _differs(case, h, r, O, l, m, O2, l2, m2)
    assert seen >= MUTANTS[mutant] * keyed, (seen, keyed)


def test_wrong_head_v_scale_is_seen():
    """Head h scaled by the other head's v_scale (1/2 against 2): every row with a nonzero output changes."""
    case = sm.band_case("hy", c=sm.FP8_C, vs=sm.FP8_VS)
    for h in range(case.H):
        O, l, _, _ = sm.expected(case, h)
        right = sm.expected_output(O, l, case.vs[h], torch.bfloat16)
        wrong = sm.expected_output(O, l, case.vs[h ^ 1], torch.bfloat16)
        nz = (right != 0).any(1)
        assert bool(nz.float().mean() > 0.99)
        assert bool((right.view(torch.int16) != wrong.view(torch.int16)).any(1)[nz].all())
