"""CPU proof that the rectangular censuses (tests/test_attention_rect_census_gpu.py) are right and sharp before any GPU
time is spent:

  * square regression: with Skv = S the generalised oracles give today's tables bit for bit;
  * brute force: rectangular key tables, transposed tables and the softmax and gradient closed forms against plain fp64
    loops over the [Sq, Skv] mask on small shapes;
  * every case of tests/rect_census_cases.py is exact in each format (inputs, hot / cold gap, per-row budgets of 2^22
    forward and 2^24 backward, counts inside the range where one key shows), and covers the rows the chunk loop must
    handle: wipes followed by partial rescales, cold-only rows, keyless rows and unreached keys;
  * sensitivity: top-left alignment, the last key dropped, the last key chunk's valid count taken from Sq, the
    transposed table built over one length, and the gradient mutants drop_pair / lse_next each change stored bits (or
    move an lse past its bound) on at least one row of every case they apply to."""
import math

import pytest
import torch

import rect_census_cases as rc
from oracle import bwd_census as bc
from oracle import census as oc
from oracle import softmax as sm

# --------------------------------------------------------------------------------------------
# square regression
# --------------------------------------------------------------------------------------------
def test_square_band_and_blockmap_tables_unchanged():
    """band_census, band_tables, blockmap_census and blockmap_tables with Skv = S equal the calls without it."""
    args, mod, S = bc.key_band_case(("generic_cog", 3, 130, 129, 1031))
    a, b = oc.band_census(mod, S, 64, "cpu"), oc.band_census(mod, S, 64, "cpu", Skv=S)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    a, b = bc.band_tables(mod, S, 128, "cpu"), bc.band_tables(mod, S, 128, "cpu", Skv=S)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    case = bc.grad_varblock_case(D=128)
    for h in range(case.H):
        a = oc.blockmap_census(case.bm[h], case.rows[h], case.cols[h], 64)
        b = oc.blockmap_census(case.bm[h], case.rows[h], case.cols[h], 64, Skv=case.S)
        assert all(torch.equal(x, y) for x, y in zip(a, b))
        a = bc.blockmap_tables(case.bm[h], case.rows[h], case.cols[h], 128)
        b = bc.blockmap_tables(case.bm[h], case.rows[h], case.cols[h], 128, Skv=case.S)
        assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_square_grad_case_unchanged():
    """_grad_inputs, the mask and the stored gradients of a case with Skv = S equal the square case's."""
    sq = bc.grad_band_case("cog", D=64)
    g = torch.Generator().manual_seed(0)
    rect = bc.GradCase(sq.name, sq.S, sq.D, sq.H, sq.c, *bc._grad_inputs(sq.H, sq.S, sq.D, sq.c, g, Skv=sq.S),
                       band=sq.band, mod=sq.mod, Skv=sq.S)
    for x, y in zip((sq.q, sq.k, sq.v, sq.o, sq.do, sq.L), (rect.q, rect.k, rect.v, rect.o, rect.do, rect.L)):
        assert torch.equal(x, y)
    for h in range(sq.H):
        assert torch.equal(sq.mask(h), rect.mask(h))
        for x, y in zip(bc.grad_expected(sq, h, torch.bfloat16), bc.grad_expected(rect, h, torch.bfloat16)):
            assert torch.equal(x.view(torch.int16), y.view(torch.int16))


def test_square_softmax_case_unchanged():
    """A softmax case with Skv = S gives the square case's tensors and closed form (band and block-map paths)."""
    import dataclasses

    for case in (sm.band_case("cog"), sm.varblock_case()):
        rect = dataclasses.replace(case, Skv=case.S)
        assert all(torch.equal(x, y) for x, y in zip(case.tensors(), rect.tensors()))
        for h in range(case.H):
            assert all(torch.equal(x, y) for x, y in zip(sm.expected(case, h), sm.expected(rect, h)))


# --------------------------------------------------------------------------------------------
# brute force on small shapes
# --------------------------------------------------------------------------------------------
def _small_masks():
    g = torch.Generator().manual_seed(3)
    out = [("random", torch.rand(37, 53, generator=g) < 0.4), ("random_t", torch.rand(61, 29, generator=g) < 0.5)]
    m = torch.rand(37, 53, generator=g) < 0.4
    m[5] = False
    m[:, 7] = False
    out.append(("holes", m))
    return out


@pytest.mark.parametrize("name,m", _small_masks(), ids=lambda x: x if isinstance(x, str) else "")
def test_key_tables_brute_force(name, m):
    """cnt[i, d] = #{j allowed for i : code(j) = d} and cnt_t[j, d] = #{i allowed for j : code(i) = d} by loops, for
    both encodings; band_tables and blockmap_tables (a block map with one-element blocks) agree."""
    Sq, Skv = m.shape
    D = 8
    mod = lambda q, k: m[q, k]  # noqa: E731
    cnt, n, cnt_t = bc.band_tables(mod, Sq, 2 * D, "cpu", Skv=Skv)
    for enc in oc.ENCODINGS:
        ck, cq = oc.key_codes(Skv, D, enc).tolist(), oc.key_codes(Sq, D, enc).tolist()
        want, want_t = torch.zeros(Sq, D, dtype=torch.long), torch.zeros(Skv, D, dtype=torch.long)
        for i in range(Sq):
            for j in range(Skv):
                if m[i, j]:
                    want[i, ck[j]] += 1
                    want_t[j, cq[i]] += 1
        assert torch.equal(cnt[enc].long(), want) and torch.equal(cnt_t[enc].long(), want_t)
    assert torch.equal(n, m.sum(1))
    ones_q, ones_k = torch.ones(Sq, dtype=torch.int32), torch.ones(Skv, dtype=torch.int32)
    b = bc.blockmap_tables(m, ones_q, ones_k, 2 * D, Skv=Skv)
    assert all(torch.equal(x.long(), y.long()) for x, y in zip(b, (cnt, n, cnt_t)))
    r = oc.rect_census(m, ones_q, ones_k, D)
    assert torch.equal(r[0], b[0].long()) and torch.equal(r[1], n)


@pytest.mark.parametrize("name,m", _small_masks(), ids=lambda x: x if isinstance(x, str) else "")
def test_softmax_closed_form_brute_force(name, m):
    """oracle.softmax.expected on an Sq x Skv predicate against fp64 softmax(c s ln 2) @ V of the case's own tensors
    (the cold tier's weight beside a hot key is 2^-150, far below the tolerance), and lse against log-sum-exp."""
    Sq, Skv = m.shape
    mod = lambda q, k: m.to(torch.as_tensor(q).device)[q, k]  # noqa: E731
    case = sm.mask_case("small", mod, Sq, Skv, D=16, H=2, L=11, C=3)
    q, k, v = (t.double() for t in case.tensors())
    for h in range(case.H):
        O, l, m_raw, _ = sm.expected(case, h)
        s = (q[h] @ k[h].T) * case.c[h] * math.log(2)
        s = s.masked_fill(~m, -math.inf)
        lse = torch.logsumexp(s, 1)
        p = torch.exp(s - lse[:, None]).nan_to_num(0.0)
        live = m.any(1)
        ref = p @ v[h]
        got = O / l.clamp(min=1e-300)[:, None]
        assert torch.allclose(got[live], ref[live], rtol=1e-12, atol=1e-12)
        assert torch.allclose(sm.exact_lse(m_raw, l, case.c[h])[live], lse[live], rtol=1e-12, atol=1e-12)
        assert bool((l[~live] == 0).all())


@pytest.mark.parametrize("name,m", _small_masks(), ids=lambda x: x if isinstance(x, str) else "")
def test_gradient_closed_form_brute_force(name, m):
    """bwd_census.grad_exact on an Sq x Skv mask against scalar loops: P_ij = 2^(e t_j - L_i), dS_ij = P_ij (dO_i . V_j
    - dO_i . O_i), dQ_i = sum_j dS_ij K_j, dK_j = sum_i dS_ij Q_i, dV_j = sum_i P_ij dO_i."""
    Sq, Skv = m.shape
    D = 8
    case = bc.grad_rect_case("small", Sq, Skv, D=D, H=1, mod=lambda q, k: m[q, k])
    (aq, ak, av), _, _ = bc.grad_exact(case, 0)
    q, k, v, o, do = (t[0].double() for t in (case.q, case.k, case.v, case.o, case.do))
    L = case.L[0].double()
    _, b = sm.qk_ints(case.c)
    dq, dk, dv = torch.zeros(Sq, D, dtype=torch.float64), torch.zeros(Skv, D, dtype=torch.float64), \
        torch.zeros(Skv, D, dtype=torch.float64)
    for i in range(Sq):
        delta = float((do[i] * o[i]).sum())
        for j in range(Skv):
            if m[i, j]:
                p = 2.0 ** (b * case.c * float(k[j, D - 1]) - float(L[i]))
                ds = p * (float(do[i] @ v[j]) - delta)
                dq[i] += ds * k[j]
                dk[j] += ds * q[i]
                dv[j] += p * do[i]
    assert torch.equal(aq, dq) and torch.equal(ak, dk) and torch.equal(av, dv)


# --------------------------------------------------------------------------------------------
# the cases: geometry, exactness, coverage
# --------------------------------------------------------------------------------------------
def test_case_geometry():
    """Sq % 128 != Skv % 128 on every case; last chunks of 1, 64, 65 and 127 columns on both sides, Sq < Skv and
    Sq > Skv, a key side shorter than one chunk; keyless rows and unreached keys; in the block-causal case with
    Lq > Lk, the queries placed before the segment's first key see exactly keys [0, F) of it."""
    cases = rc.CASES + [rc.WAN720_TEXT, rc.WAN480_CHUNK]
    assert all(c.Sq % 128 != c.Skv % 128 for c in cases)
    for side in ("Sq", "Skv"):
        widths = {(getattr(c, side) - 1) % 128 + 1 for c in cases}
        assert {1, 64, 65, 127} <= widths, (side, widths)
    assert any(c.Sq < c.Skv for c in cases) and any(c.Sq > c.Skv for c in cases) and min(c.Skv for c in cases) < 128
    keyless = unreached = 0
    for c in rc.CASES:
        m = c.dense(0)
        keyless += int((~m.any(1)).sum())
        unreached += int((~m.any(0)).sum())
    assert keyless > 0 and unreached > 0
    c = rc.BY_NAME["block_ahead"]
    sink, C_, F, W = c.args
    lq, lk = c.cu_q[1], c.cu_k[1]
    assert lq > lk and F < C_
    m = c.dense(0)
    ahead = lq - lk  # queries qi < Lq - Lk sit before key 0
    want = torch.zeros(c.Skv, dtype=torch.bool)
    want[:F] = True
    assert bool((m[:ahead] == want).all()) and not bool((m[ahead:lq, :F] == 0).all())


def test_kvcache_predicates_match_the_host_mirrors():
    """The KV-cache cases' tensor predicates equal kvcache_mask.allowed / block_causal_mask.allowed at p = i + L - Sq."""
    import block_causal_mask as bm
    import kvcache_mask as km

    for c in rc.CASES:
        if c.kind != "kvcache":
            continue
        m = c.dense(0)
        kv = c.kv
        for i in range(0, c.Sq, 37):
            p = i + c.Skv - c.Sq
            for j in range(0, c.Skv, 7):
                if kv["mask"] == "block":
                    want = bm.allowed(p, j, kv["sink"], kv["C"], kv["F"], kv["W"])
                else:
                    want = km.allowed(p, j, kv["sink"], rc.BIG if kv["mask"] == "causal" else kv["left"], 0)
                assert bool(m[i, j]) == want, (c.name, i, j)


def _softmax_cases():
    return [(c.name, c) for c in rc.CASES] + [("wan720_text", rc.WAN720_TEXT), ("wan480_chunk", rc.WAN480_CHUNK)]


# name -> stated share of rows with keys that are wiped by their first hot chunk and then rescaled at least twice, on
# the kernel's visit order.  A row needs hot keys over three chunks for that, so short key sides and rows that see a
# few hundred keys score low; vb_1151x65's 65 keys are one chunk, where the rescales fall inside the chunk.
COVERAGE = {"vb_1000x600": 0.0, "vb_333x1200": 0.2, "vb_1151x65": 0.0, "local_holes": 0.5, "local_sink_window": 0.6,
            "local_short_tail": 0.01, "block_ahead": 0.4, "block_window_sink": 0.9, "block_one_query": 0.1,
            "kv_causal_contig": 1.0, "kv_causal_paged": 0.9, "kv_window_contig": 0.35, "kv_window_paged": 0.7,
            "kv_block_contig": 0.6, "kv_block_paged": 0.9, "wan720_text": 0.9, "wan480_chunk": 0.9}
STRIDE = {"wan720_text": 997, "wan480_chunk": 97}


@pytest.mark.parametrize("name,case", _softmax_cases(), ids=lambda x: x if isinstance(x, str) else "")
def test_softmax_case_exact_and_covered(name, case):
    """Inputs exact in bf16 and fp16, the hot / cold gap >= 150 after c, every row's partial sums below 2^22 (every
    row; the production shapes on a stride), and the share of rows wiped by their first hot chunk and then rescaled at
    least twice, with cold-only rows, on the kernel's visit order (the simulation equals the closed form on every
    visited row)."""
    s = case.softmax_case(128)
    assert int(s.kcls.max()) < s.D - 1 and int(s.kt.max()) <= s.R
    for h in range(s.H):
        a, b = sm.qk_ints(s.c[h])
        assert sm.GAP - b * s.c[h] * s.R >= sm.MIN_GAP
    for t in s.tensors():
        for dt in (torch.bfloat16, torch.float16):
            assert torch.equal(t.to(dt).float(), t)
    stride, frac = STRIDE.get(name, 1 if case.Sq * case.Skv < 2e6 else 5), COVERAGE[name]
    rows = list(range(0, s.S, stride))
    for h in range(s.H):
        budget = sm.expected(s, h, row_ids=rows)[3] if s.mod is not None else sm.expected(s, h)[3]
        assert float(budget.max()) < sm.BUDGET
    st = sm.coverage(s, stride)
    print(f"{name}: {st}")
    assert st["covered"] >= frac * st["keyed"] and (st["cold_only"] > 0 or case.Sq < 13), st


@pytest.mark.parametrize("name", rc.BACKWARD + ["wan480_chunk"])
def test_backward_case_exact(name):
    """Key census: every count stays where it is exact in bf16 (fp16 for the production shape, whose counts pass 256).
    Gradient census: budgets below 2^24 granules, every dS a multiple of 1/8 of magnitude <= 8, dS != 0 on most allowed
    pairs."""
    case = rc.WAN480_CHUNK if name == "wan480_chunk" else rc.BY_NAME[name]
    dt = torch.float16 if name == "wan480_chunk" else torch.bfloat16
    for D in (64, 128):
        for enc in oc.ENCODINGS:
            bound = max(oc.column_bound(case.Sq, D // 2, enc), oc.column_bound(case.Skv, D // 2, enc))
            assert bound <= bc.MAX_COUNT[dt], (D, enc, bound)
        if name == "wan480_chunk":
            continue
        gc = case.grad_case(D)
        for h in range(gc.H):
            _, bud, st = bc.grad_exact(gc, h)
            assert max(bud) < bc.BUDGET and st["ds_exact"] and st["ds_max"] <= 8
            assert st["ds_nonzero"] > 0.5 * st["allowed"]


# --------------------------------------------------------------------------------------------
# sensitivity
# --------------------------------------------------------------------------------------------
def _key_rows_seen(cnt, n, cnt2, n2, dt):
    """rows whose forward key census output bits or key count (exp(lse) names n exactly) differ"""
    bad = n != n2
    for enc in oc.ENCODINGS:
        a = oc.expected_output(cnt[enc], n, dt).view(torch.int16)
        b = oc.expected_output(cnt2[enc], n2, dt).view(torch.int16)
        bad |= (a != b).any(1)
    return int(bad.sum())


def _bwd_rows_seen(tab, tab2, Sq, Skv, D, dt):
    seen = 0
    for enc in oc.ENCODINGS:
        e = bc.key_expected(tab[0][enc], tab[2][enc], Sq, D, enc, Skv=Skv)
        e2 = bc.key_expected(tab2[0][enc], tab2[2][enc], Sq, D, enc, Skv=Skv)
        seen += sum(int((x.to(dt).float() != y.to(dt).float()).any(1).sum()) for x, y in zip(e, e2))
    return seen


def _softmax_rows_seen(s, s2, dt):
    O, l, m_raw, _ = sm.expected(s, 0)
    O2, l2, m2, _ = sm.expected(s2, 0)
    a = sm.expected_output(O, l, s.vs[0], dt).view(torch.int16)
    b = sm.expected_output(O2, l2, s.vs[0], dt).view(torch.int16)
    lo, hi = sm.lse_bounds(m_raw, l, s.c[0])
    lo2, hi2 = sm.lse_bounds(m2, l2, s.c[0])
    moved = (hi2 < lo) | (lo2 > hi) | ((l > 0) != (l2 > 0))
    return int(((a != b).any(1) | moved).sum())


def _grad_rows_seen(gc, gc2, dt):
    e, e2 = bc.grad_expected(gc, 0, dt), bc.grad_expected(gc2, 0, dt)
    return sum(int((x.float() != y.float()).any(1).sum()) for x, y in zip(e, e2))


@pytest.mark.parametrize("mutant", rc.MASK_MUTANTS)
def test_mask_mutants_are_seen(mutant):
    """On every case where the mutant changes the mask of head 0: the forward key census (both formats) and, with a
    backward, the backward key census and the gradient census each change stored bits or move an
    lse past its bound on at least one row; the softmax census does so on at least half of those cases."""
    applied, softmax_seen = [], 0
    for c in rc.CASES:
        if not c.applies(mutant) or torch.equal(c.dense(0), c.dense(0, mutant)):
            continue
        applied.append(c.name)
        D = 64
        t = oc.band_census(c.mod(0), c.Sq, D, "cpu", Skv=c.Skv)
        t2 = oc.band_census(c.mod(0, mutant), c.Sq, D, "cpu", Skv=c.Skv)
        for dt in (torch.bfloat16, torch.float16):
            assert _key_rows_seen(*t, *t2, dt) > 0, (c.name, dt)
        s = c.softmax_case(D)
        softmax_seen += _softmax_rows_seen(s, c.with_mask(s, mutant), torch.bfloat16) > 0
        if c.backward:
            tab = bc.band_tables(c.mod(0), c.Sq, D, "cpu", Skv=c.Skv)
            tab2 = bc.band_tables(c.mod(0, mutant), c.Sq, D, "cpu", Skv=c.Skv)
            assert _bwd_rows_seen(tab, tab2, c.Sq, c.Skv, D, torch.bfloat16) > 0, c.name
            gc = c.grad_case(D)
            assert _grad_rows_seen(gc, c.with_mask(gc, mutant), torch.bfloat16) > 0, c.name
    print(f"{mutant}: seen on {applied}; the softmax census sees it on {softmax_seen}")
    assert len(applied) >= 4
    # the softmax census sees only a row's live tier: a dropped key that is cold beside hot ones does not show there
    assert softmax_seen >= len(applied) // 2


def test_transposed_table_over_one_length_is_seen():
    """The backward's transposed table built over the square min(Sq, Skv) (keys and queries past it dropped, as a
    one-length oracle or kernel would) changes dK / dV bits on every case with a backward."""
    for name in rc.BACKWARD:
        c = rc.BY_NAME[name]
        D, S = 64, min(c.Sq, c.Skv)
        tab = bc.band_tables(c.mod(0), c.Sq, D, "cpu", Skv=c.Skv)
        sq_t, _ = oc.band_census(lambda kk, qq: c.mod(0)(qq, kk), S, D // 2, "cpu", Skv=S)
        wrong = torch.zeros_like(tab[2])
        wrong[:, :S] = sq_t
        assert _bwd_rows_seen(tab, (tab[0], tab[1], wrong), c.Sq, c.Skv, D, torch.bfloat16) > 0, name


@pytest.mark.parametrize("mutant", ["drop_pair", "lse_next"])
def test_gradient_mutants_are_seen(mutant):
    """bwd_census's drop_pair (the first allowed key of every row) and lse_next (the next row's lse) on the rectangular
    masks: stored dQ, dK or dV bits change on a large share of the rows of every case with a backward."""
    for name in rc.BACKWARD:
        gc = rc.BY_NAME[name].grad_case(64)
        ref = bc.grad_expected(gc, 0, torch.bfloat16)
        mut = bc.grad_expected(gc, 0, torch.bfloat16, mutant=mutant)
        changed = sum(int((x.float() != y.float()).any(1).sum()) for x, y in zip(ref, mut))
        assert changed > 0.1 * gc.S, (name, changed)
