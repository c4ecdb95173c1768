"""The split KV-cache census of oracle/kvsplit_census.py on the CPU: its predicate and split rule against the host mirrors
of the single plan, the premises of every GPU case of tests/kvsplit_cases.py, the rows the cases must contain, the
merge bound against a perturbed fp32 emulation of the merge, and that every MUTATION of the flow is caught by some GPU
case."""
import math

import numpy as np
import pytest
import torch

import block_causal_mask as bcm
import kvcache_mask as km
import kvsplit_cases as kc
from oracle import census as oc
from oracle import kvsplit_census as ks

OUT = {"bf16": torch.bfloat16, "fp16": torch.float16, "e4m3": torch.bfloat16, "e4m3_rows": torch.bfloat16}


@pytest.mark.parametrize("name", list(kc.MASKS))
def test_predicate_and_row_sets_match_the_mirrors(name):
    mask = kc.MASKS[name]
    for L, Sq in ((700, 300), (90, 200), (0, 5)):
        for i in range(Sq):
            p = L - Sq + i
            if mask.block:
                want = [bcm.allowed(p, kv, mask.sink, mask.block, mask.first_block, mask.window) for kv in range(L)]
            else:
                want = [km.allowed(p, kv, mask.sink, mask.left, mask.right) for kv in range(L)]
            assert [mask.allowed(p, kv) for kv in range(L)] == want, (name, L, i)
            a1, b0, b1 = (int(x[0]) for x in mask.row_sets(np.array([p]), L))
            got = [kv < a1 or b0 <= kv < b1 for kv in range(L)]
            assert got == want, (name, L, i)


@pytest.mark.parametrize("name", list(kc.MASKS))
def test_split_lists_concatenate_to_the_single_mirror(name):
    """Split s of every item keeps a piece of the single plan's list (tests/kvcache_mask.py, tests/block_causal_mask.py):
    concatenated in split order they give it back, with every chunk's elem flag."""
    mask = kc.MASKS[name]
    Ls, Sq = [1500, 0, 90, 777], 300
    if mask.block:
        items, _ = bcm.kv_plan(Ls, Sq=Sq, new_len=0, nblocks=4, block_rows=2048, sink=mask.sink, block=mask.block,
                               first_block=mask.first_block, window=mask.window)
    else:
        items, _ = km.plan(Ls, Sq=Sq, new_len=0, nblocks=4, block_rows=2048, sink=mask.sink,
                           left=min(mask.left, 10 ** 9), right=mask.right)
    case = ks.Case("mirror", Ls, Sq, 1, 1, 64, "bf16", "contig", mask, 1)
    single = [(r0, nr, [(j, elem) for _, _, elem, j in ch]) for _, r0, nr, ch in items]
    assert ks.plan_lists(case, 1) == single
    for n in (2, 3, 5, 40):
        split = ks.plan_lists(case, n)
        for i, (r0, nr, chunks) in enumerate(single):
            parts = [split[s * len(single) + i] for s in range(n)]
            assert all(p[:2] == (r0, nr) for p in parts)
            assert [c for p in parts for c in p[2]] == chunks, (name, n, i)


@pytest.mark.parametrize("case", kc.ALL, ids=lambda c: c.name)
def test_premises(case):
    """Inputs exact in their format, the counts below the census limits, every split's sum below 2^22, the splits'
    counts summing to the mask's, and no empty visited chunk (so the cut over visited chunks is the cut over kept ones)."""
    n = kc.splits(case)
    ns_, cnt, N = ks.key_census(case, n)
    assert np.array_equal(ns_.sum(0), N)
    assert int(ns_.max(initial=0)) < 1 << 22
    assert int(cnt.max(initial=0)) < oc.COUNT_LIMIT[OUT[case.fmt]], case.name
    assert ks.visited_all_live(case), case.name
    # one-hot V and power-of-two row scales 2^d, d in [-2, 6]: the stored bytes 2^-d are exact e4m3, bf16 and fp16
    for d in range(-2, 7):
        x = torch.tensor([2.0 ** -d])
        assert float(x.to(torch.float8_e4m3fn).float() * 2.0 ** d) == 1.0
    for dt in (torch.bfloat16, torch.float16):
        assert float(torch.ones(1).to(dt)) == 1.0
    for hk in range(case.Hkv):
        codes = ks.key_codes(max(case.Ls + [1]), case.D, hk)
        assert codes.min() >= 0 and codes.max() < case.D


def test_coverage_of_the_required_rows():
    """Across the GPU cases: a row whose only keys lie in a split other than 0, one whose live splits are not adjacent,
    one that no split sees, an empty trailing split (n > nvis), and an item whose pieces leave a split without keys for
    a row between two live ones."""
    seen = dict(late_only=0, gap=0, keyless=0, empty_split=0)
    for case in kc.SMALL:
        n = kc.splits(case)
        ns_, _, N = ks.key_census(case, n)
        live = ns_ > 0
        first = np.where(live.any(0), live.argmax(0), -1)
        seen["late_only"] += int(((first > 0) & (N > 0)).sum())
        seen["keyless"] += int((N == 0).sum())
        last = np.where(live.any(0), n - 1 - live[::-1].argmax(0), -1)
        seen["gap"] += int(((last - first + 1 > live.sum(0)) & (N > 0)).sum())
        seen["empty_split"] += sum(1 for _, _, ch in ks.plan_lists(case, n) if not ch)
    assert all(v > 0 for v in seen.values()), seen


@pytest.mark.parametrize("case", kc.SMALL[::3] + kc.PRODUCTION[:1], ids=lambda c: c.name)
def test_bound_holds_against_a_perturbed_fp32_merge(case):
    """Every expf result moved by up to 2 ulp and every logf by up to 1 ulp, at random, in 6 draws: the emulated o is
    always one of the 16-bit values the bound admits, and its lse within beta_l."""
    n = kc.splits(case)
    ns_, cnt, _ = ks.key_census(case, n)
    o_p, l_p = ks.partials_fp32(ns_, cnt, case.G)
    y, beta, lse, beta_l = ks.bound(o_p, l_p)
    dt = OUT[case.fmt]
    rng = np.random.default_rng(case.seed)
    for draw in range(6):
        o, l = ks.merge_fp32(o_p, l_p, rng=rng if draw else None)
        o16 = ks.round16(o, dt)
        assert bool(ks.admissible(o16, y, beta, dt).all()), (case.name, draw)
        assert bool((np.abs(o.astype(np.float64) - y) <= beta).all()), (case.name, draw)
        fin = np.isfinite(lse)
        assert np.array_equal(fin, np.isfinite(l))
        assert bool((np.abs(l[fin].astype(np.float64) - lse[fin]) <= beta_l[fin]).all()), (case.name, draw)


def test_lse_bound_identifies_the_count_at_production_length():
    """At N = 32 760 keys the merge bound beta_l (~2.5e-6) and the partials' own lse error together stay below
    0.4 ln((N + 1) / N) (3.1e-5): exp(lse) rounds to N."""
    case = kc.PRODUCTION[0]
    n = kc.splits(case)
    ns_, cnt, N = ks.key_census(case, n)
    o_p, l_p = ks.partials_fp32(ns_, cnt, case.G)
    lo, hi = ks.lse_partial_bounds(ns_, case.Hq)
    sigma = np.maximum(hi - lo, 0)
    _, _, lse, beta_l = ks.bound(o_p, l_p, sigma)
    step = ks.lse_count_margin(kc.WAN_L)
    fin = np.isfinite(lse)
    worst = float((beta_l[fin] + np.abs(lse[fin] - np.log(N[None].repeat(case.Hq, 0)[fin]))).max())
    # exp(lse) rounds to N while |lse - ln N| < ln(1 + 1 / (2N)) ~ step / 2
    assert float(beta_l[fin].max()) < 0.25 * step and worst < 0.4 * step, (float(beta_l[fin].max()), worst, step)


def _softmax(i):
    """(case name, o_part, lse_part, lo, hi, budget) of softmax census case i: the closed-form partials, the lse as the
    kernel forms it with a correctly rounded log2f"""
    base, mask, n, fmt = kc.softmax_case(i)
    o, lo, hi, lse, budget = ks.softmax_partials(base, mask, n)
    return f"softmax_{kc.SOFTMAX[i][0]}_n{n}_{fmt}{base.D}", o, lse, lo, hi, budget


_SOFTMAX = {}


def _softmax_cached(i):
    if i not in _SOFTMAX:
        _SOFTMAX[i] = _softmax(i)
    return _SOFTMAX[i]


def _merge_catch(o_p, l_p, mo, ml):
    """How a merged (mo, ml) differs from the merge of (o_p, l_p): (kind, None) for a non-finite value or a miss where
    the value is exact (rows without keys, zero outputs), (kind, margin in bounds) elsewhere; None when inside 10
    bounds everywhere"""
    y, beta, lse, beta_l = ks.bound(o_p, l_p)
    with np.errstate(invalid="ignore", over="ignore"):
        d = np.abs(mo.astype(np.float64) - y)
        d = np.where(np.isnan(d), np.inf, d)
        fin = np.isfinite(lse)
        dl = np.where(fin, np.abs(ml.astype(np.float64) - np.where(fin, lse, 0)), np.where(ml == lse, 0, np.inf))
        dl = np.where(np.isnan(dl), np.inf, dl)
    if np.isinf(d).any():
        return "merged o, not finite", None
    if np.isinf(dl).any():
        return "merged lse, not finite or -inf where finite (or the reverse)", None
    # where the bound is only the subnormal floor (y = 0: rows without keys, zero outputs) the value must be exact
    pos_o, pos_l = beta > 2.0 ** -140, beta_l > 0
    m_o = float((d[pos_o] / beta[pos_o]).max(initial=0))
    m_l = float((dl[pos_l] / beta_l[pos_l]).max(initial=0))
    if max(m_o, m_l) >= 10:
        return ("merged o", m_o) if m_o >= m_l else ("merged lse", m_l)
    if (d[~pos_o] > 2.0 ** -140).any():
        return "merged o, exactly 0 expected", None
    if (dl[~pos_l] > 0).any():
        return "merged lse, exact value expected", None
    return None


def _mutation_report(mut):
    """(case name, how it is caught, margin) of the first GPU case that catches the mutation, or None: the key census
    cases first, then (merge mutations) the softmax census cases"""
    for case in kc.SMALL:
        n = kc.splits(case)
        lists, o_p, l_p, o, l = ks.simulate(case, n)
        mlists, mo_p, ml_p, mo, ml = ks.simulate(case, n, mut)
        if mlists != lists:
            return case.name, "split lists", None
        if not (np.array_equal(mo_p, o_p) and np.array_equal(ml_p, l_p)):
            bad_o = ~(mo_p == o_p)  # NaN never matches
            bad_l = ~(ml_p == l_p)
            return case.name, f"partials ({int(bad_o.sum())} o, {int(bad_l.sum())} lse)", None
        c = _merge_catch(o_p, l_p, mo, ml)
        if c:
            return (case.name,) + c
    if mut in ks.RULE + ks.EPILOGUE:
        return None
    for i in range(len(kc.SOFTMAX)):
        name, o_p, l_p, _, _, _ = _softmax_cached(i)
        mo, ml = ks.merge_fp32(o_p, l_p, mutation=mut)
        c = _merge_catch(o_p, l_p, mo, ml)
        if c:
            return (name,) + c
    return None


@pytest.mark.parametrize("mut", [m for m in ks.MUTATIONS if m != "piece_over_kept"])
def test_every_mutation_is_caught(mut):
    rep = _mutation_report(mut)
    assert rep is not None, f"{mut}: no GPU case catches it"
    print(f"{mut}: caught by {rep[0]} through the {rep[1]}" + (f", margin {rep[2]:.3g} x bound" if rep[2] else ""))


@pytest.mark.parametrize("mut", ["no_max", "m_first_live"])
def test_merge_range_mutations_need_the_softmax_census(mut):
    """With q = 0 every lse_s is ln(n_s) <= 10.4: a merge without the max, or with m from the first live split, passes
    every key census case, and only the softmax census, whose hot and cold splits lie over 100 nats apart, sees it."""
    for case in kc.SMALL:
        n = kc.splits(case)
        _, o_p, l_p, _, _ = ks.simulate(case, n)
        _, _, _, mo, ml = ks.simulate(case, n, mut)
        assert _merge_catch(o_p, l_p, mo, ml) is None, case.name
    assert any(_merge_catch(*_softmax_cached(i)[1:3], *ks.merge_fp32(*_softmax_cached(i)[1:3], mutation=mut))
               for i in range(len(kc.SOFTMAX)))


@pytest.mark.parametrize("i", range(len(kc.SOFTMAX)))
def test_softmax_census_premises(i):
    """Every split's partial sums stay below the census budget (a split without a row's hot keys makes its cold tier
    live), the kernel-rounded lse lies in lse_bounds, and some row has a hot and a cold split more than 100 nats
    apart."""
    from oracle import softmax as sm

    name, o_p, l_p, lo, hi, budget = _softmax_cached(i)
    assert budget < sm.BUDGET, name
    fin = np.isfinite(lo)
    assert np.array_equal(np.isfinite(l_p), fin)
    assert bool(((l_p[fin] >= lo[fin]) & (l_p[fin] <= hi[fin])).all()), name
    lam = np.where(fin, l_p, np.nan)
    with np.errstate(invalid="ignore"):
        spread = np.nanmax(lam, 0) - np.nanmin(lam, 0)
    assert float(np.nanmax(spread)) > 100, (name, float(np.nanmax(spread)))
    assert float(np.nanmax(lam)) > 100, name


@pytest.mark.parametrize("i", range(len(kc.SOFTMAX)))
def test_bound_holds_on_the_softmax_census(i):
    """The perturbed fp32 merge of the softmax census partials stays inside the bound (the cold splits' weights flush
    to 0 beside a hot one)."""
    name, o_p, l_p, _, _, _ = _softmax_cached(i)
    y, beta, lse, beta_l = ks.bound(o_p, l_p)
    dt = OUT[kc.SOFTMAX[i][2]]
    rng = np.random.default_rng(i)
    for draw in range(4):
        o, l = ks.merge_fp32(o_p, l_p, rng=rng if draw else None)
        assert bool(ks.admissible(ks.round16(o, dt), y, beta, dt).all()), (name, draw)
        assert bool((np.abs(o.astype(np.float64) - y) <= beta).all()), (name, draw)
        fin = np.isfinite(lse)
        assert np.array_equal(fin, np.isfinite(l))
        assert bool((np.abs(l[fin].astype(np.float64) - lse[fin]) <= beta_l[fin]).all()), (name, draw)


def test_cut_over_kept_chunks_is_equivalent_here():
    """Cutting the kept list instead of the visited one differs only when a visited chunk holds no allowed key, which
    neither rule produces (module docstring): on every case the mutation leaves the lists unchanged."""
    for case in kc.SMALL:
        n = kc.splits(case)
        assert ks.plan_lists(case, n, "piece_over_kept") == ks.plan_lists(case, n), case.name


def test_bound_is_tight_enough_to_matter():
    """The bound sits well below the 16-bit output spacing and the suite's old 2e-2 tolerance."""
    case = kc.SMALL[5]
    n = kc.splits(case)
    ns_, cnt, _ = ks.key_census(case, n)
    o_p, l_p = ks.partials_fp32(ns_, cnt, case.G)
    y, beta, _, beta_l = ks.bound(o_p, l_p)
    assert float(beta.max()) < 1e-6 and float(beta_l.max()) < 1e-5
    assert math.isfinite(float(beta.max()))
