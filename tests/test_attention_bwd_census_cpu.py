"""The premises of the backward censuses (oracle/bwd_census.py), without a GPU: the lse encoding, the representability
of every key-census value, and per gradient-census case its budget, exactness, coverage and the sensitivity of its
expected bits to the kernel bugs the census is meant to catch (oracle mutants)."""
import numpy as np
import pytest
import torch

from oracle import bwd_census as bc
from oracle import census as oc
from oracle import softmax as osm


def test_lse_round_trip():
    """For every integer L in [-4, 8], lse_for(L) is an fp32 value whose fp32(lse * fp32(log2 e)) is exactly L: the
    kernel's log2-domain lse is an integer, so exp2(c s - L) is exact at the integer exponents of the censuses."""
    for L in range(-4, 9):
        x = np.float32(bc.lse_for(L))
        assert np.float32(x * osm.LOG2E) == np.float32(L), L
        assert abs(float(x) - L * np.log(2)) < 1e-6


def key_cases():
    """(what, S, D, dtype) of every key-census run of tests/test_attention_bwd_census_gpu.py"""
    out = []
    for kind, density in bc.KEY_BAND_FULL:
        out.append((f"band {kind} {density}", bc.key_band_case(kind, density)[2], 128, torch.float16))
    for case in bc.KEY_BAND_SMALL:
        S = bc.key_band_case(case)[2]
        out += [(f"band {case}", S, D, dt) for D in (64, 128) for dt in (torch.bfloat16, torch.float16)]
    out.append(("varblock hunyuan", 256 + 33 * 3600, 128, torch.float16))
    out.append(("varblock wan", 21 * 3600, 128, torch.float16))
    out.append(("varblock small", 6000, 128, torch.bfloat16))
    out.append(("shared BSR", 40 + 8 * 300, 128, torch.float16))
    return out


def test_key_census_representable():
    """No count of a key-census table can exceed the number of positions that share one code (column_bound), and every
    value the closed form takes up to that bound (count x 1/4, 1/2 or 1, either sign) is exact in the output format.
    So one key wrongly kept or dropped changes stored bits.  fp16 holds counts to 2047, bf16 to 256 (both bounds are
    tight: one more is not exact)."""
    for dt, m in bc.MAX_COUNT.items():
        assert bc.key_counts_representable(m, dt)
        assert not bc.key_counts_representable(m + 2, dt)
    worst = {}
    for what, S, D, dt in key_cases():
        bound = max(oc.column_bound(S, D // 2, enc) for enc in oc.ENCODINGS)
        assert bound <= bc.MAX_COUNT[dt], f"{what}: D={D} {dt}: a count may reach {bound}"
        worst[dt] = max(worst.get(dt, 0), bound)
    print(f"largest possible count: {worst[torch.float16]} (fp16, limit 2047), {worst[torch.bfloat16]} (bf16, limit 256)")


def grad_cases():
    out = [bc.grad_band_case(n, D=D) for n in bc.GRAD_BAND for D in (64, 128)]
    out += [bc.grad_band_case("hy", c=c) for c in (0.5, 2.0)]
    out += [bc.grad_varblock_case(D=D) for D in (64, 128)]
    out += [bc.grad_varblock_case(H=4), bc.grad_bsr_case()]
    return out


@pytest.mark.parametrize("case", grad_cases(), ids=lambda c: f"{c.name}-D{c.D}-H{c.H}-c{c.c}")
def test_grad_census_case(case):
    """Budget: for every gradient element the sum of |terms| stays below 2^24 granules of 1/8, so the fp32 accumulators
    are exact in any order.  Representability: the inputs are exact in bf16 and fp16, every P is in {1/8, .., 1} and
    every dS a multiple of 1/8 of magnitude <= 8 (exact in bf16).  Coverage: the share of allowed pairs with dS != 0,
    and the keyless rows and unreached keys of the variable-block maps."""
    for t in (case.q, case.k, case.v, case.o, case.do):
        for dt in (torch.bfloat16, torch.float16):
            assert torch.equal(t.to(dt).float(), t)
    _, b = osm.qk_ints(case.c)
    e = b * case.c
    t = case.k[:, :, case.D - 1]
    assert int(t.min()) >= 0 and e * float(t.max()) <= 2 and set(case.L.unique().tolist()) <= {2, 3}
    assert bool((case.q[:, :, case.D - 1] == b).all())
    cols = torch.arange(case.D - 1)
    for h in range(case.H):  # the score is b t_j alone: Q and K live on disjoint columns below D - 1
        assert not bool(((case.q[h, :, : case.D - 1] != 0).any(0) & (case.k[h, :, : case.D - 1] != 0).any(0)).any())
    nz = (case.q[:, :, :-1] != 0).any(1) | (case.k[:, :, :-1] != 0).any(1)
    assert bool(nz.any(0)[cols].all()), "some column of dQ or dK is zero on every head"
    allowed = nonzero = keyless = unreached = 0
    budget = 0.0
    for h in range(case.H):
        _, bud, st = bc.grad_exact(case, h)
        assert st["ds_exact"] and st["ds_max"] <= 8
        assert max(bud) < bc.BUDGET, f"head {h}: budget {bud}"
        budget = max(budget, max(bud))
        allowed += st["allowed"]
        nonzero += st["ds_nonzero"]
        keyless += st["keyless"]
        unreached += st["unreached"]
    if case.bm is not None and "bsr" not in case.notes:
        assert keyless > 0 and unreached > 0
    assert nonzero > 0.5 * allowed
    print(f"{case.name} D={case.D} H={case.H} c={case.c}: budget {budget:.0f} of {bc.BUDGET} granules; dS != 0 on "
          f"{nonzero / max(allowed, 1):.3f} of {allowed} allowed pairs; {keyless} keyless rows, {unreached} unreached keys")


@pytest.mark.parametrize("case", [bc.grad_band_case("cog", D=128), bc.grad_varblock_case(D=128)],
                         ids=["band-cog", "varblock"])
def test_grad_census_mutants(case):
    """Each oracle mutant (a restated kernel bug) changes the expected bits of a large share of the rows of at least
    one gradient: the neighbouring row's lse or delta, delta over only the first 64 columns, dK stored without
    sm_scale, dV stored with it, one allowed pair dropped per row."""
    ref = [bc.grad_expected(case, h, torch.bfloat16) for h in range(case.H)]
    lines = []
    for m in bc.MUTANTS:
        frac = []
        for g in range(3):
            changed = sum(int((bc.grad_expected(case, h, torch.bfloat16, mutant=m)[g].float() != ref[h][g].float())
                              .any(1).sum()) for h in range(case.H))
            frac.append(changed / (case.H * case.S))
        lines.append(f"{m}: dq {frac[0]:.3f} dk {frac[1]:.3f} dv {frac[2]:.3f}")
        assert max(frac) > 0.25, f"{case.name}: mutant {m} changes too few rows ({lines[-1]})"
    print(f"{case.name}: share of rows whose expected bits change, per mutant: " + "; ".join(lines))


def test_grad_band_lists_cross_the_stream_switch():
    """The key-major plans of the gradient census's band cases (restated from the mask: one list per 256-key item,
    shared by its two streams) have stream-0 lists of odd and of even length followed by a stream 1, so the kernel's
    stage parity and the stationary-tile barrier phase are both exercised across the stream switch.  (Mode NONE gives
    every key the same list of all 9 query chunks.)"""
    seen = {}
    for name in bc.GRAD_BAND:
        case = bc.grad_band_case(name)
        mode, m0, m1, _ = case.band
        items = torch.tensor([[[r, min(n, 128), 0, 0], [r + 128, max(n - 128, 0), 0, 0]]
                              for r, n in bc.band_items(mode, m0, m1, case.S, True)])
        lens = torch.tensor([w.numel() for w, _ in bc.band_t_lists(items, case.mod, case.S, "cpu")])
        items[:, :, 3] = lens[:, None]
        st = bc.plan_stats(items)
        seen[name] = {k for k in ("odd", "even", "one") if st[k]}
        assert st["two"] and st["odd"] and (st["even"] or name == "none"), f"{name}: {st}"
    print(f"key-major band plans: {seen}")
