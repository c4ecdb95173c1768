"""CPU proof that the pre-attention backward census (tests/test_rowwise_bwd_census_gpu.py, oracle/rowwise_bwd.py) is
exact and sees the bugs it is meant to see.

  * premises, for every case the GPU file runs (on its live rows; the others have dn = 0 and dx = 0): x, dn and dx
    exact in the 16-bit dtype; the closed form equal to the backward computed from first principles; dx never 0 and
    far enough from a rounding boundary that an rsqrtf a few ulps off cannot move it; mean(u) != 0 on LayerNorm rows;
    every row sum and every dgamma / dbeta sum below 2^24 quanta; eps absorbed; quarter-turn tables inverted exactly
    by the transpose;
  * geometry: the oracle's grid helpers against prep.cu's constants and the workspace sizes its C entry points
    report, and the grid crossings each case claims;
  * sensitivity: mutants of the formulas (a divisor N - 1, a dropped term, the hidden row divided by D, gamma indexed
    by column % D, dgamma summing u x^, the RoPE range off by one, the last partial dropped or doubled, stats of the
    other batch) change the expected bits.
"""
import ctypes as C
import re
from pathlib import Path

import pytest
import torch

from oracle import rowwise as rw
from oracle import rowwise_bwd as rb

ROOT = Path(__file__).resolve().parent.parent
DTYPES = (torch.bfloat16, torch.float16)
CHUNK = 1 << 21


def rope_t(dy, c, s, rope):
    """The kernels' RoPE transpose (prep.cu rope_apply<true> / rope_apply_complex<.., true>) in float64."""
    dy, c, s = dy.double(), c.double(), s.double()
    a, b = dy[..., 0::2], dy[..., 1::2]
    if rope == 2:
        return torch.stack([a * c + b * s, b * c - a * s], -1).flatten(-2)
    ce, co, se, so = c[..., 0::2], c[..., 1::2], s[..., 0::2], s[..., 1::2]
    return torch.stack([a * ce + b * so, b * co - a * se], -1).flatten(-2)


# ---- premises ----------------------------------------------------------------------------------------------------
class Premises:
    """Accumulates the element-wise premises of one case over chunks of its live rows."""

    def __init__(self, N, dtype, layer, hidden):
        self.N, self.dtype, self.layer, self.hidden = N, dtype, layer, hidden
        self.ag = torch.zeros(N, dtype=torch.float64)
        self.ab = torch.zeros(N, dtype=torch.float64)
        self.ratio = float("inf")
        self.rows = 0

    def add(self, c, g):
        dt, x, dn, dx, xh = self.dtype, c["x"], c["dn"], c["dx"], c["xh"]
        if x.shape[0] == 0:
            return
        assert rw.exact_in(x, dt) and rw.row_sums_ok(x, self.layer)
        assert rw.exact_in(dn, dt) and rw.exact_in(dx, dt)
        assert bool((dx != 0).all()), "a live row's dx has a 0"
        assert torch.equal(rb.norm_bwd(x, dn, g, layer=self.layer), dx), "closed form != first principles"
        ok, ratio = rw.norm_margin_ok(dx, rb.margin_scale(c), dt)
        assert ok, ratio
        self.ratio = min(self.ratio, ratio)
        if self.layer:
            assert bool((c["u"].mean(-1).abs() >= 1 / 16).all()), "mean(u) = 0 on a LayerNorm row"
        # every term of every fp32 sum a multiple of its quantum, the sums below 2^24 quanta
        t = dn * xh
        for v, q in ((dn, rb.Q_DB), (t, rb.Q_DG)):
            assert torch.equal(torch.round(v / q), v / q)
        ux = c["u"] * x.double()                                    # the hidden stats pass sums u x (quantum 1/16)
        assert torch.equal(torch.round(ux * 16), ux * 16) and float((ux.abs().sum(-1) * 16).max()) < rb.SUM_LIMIT
        self.ag += t.abs().sum(0)
        self.ab += dn.abs().sum(0)
        self.rows += x.shape[0]

    def done(self):
        assert float(self.ag.max()) / rb.Q_DG < rb.SUM_LIMIT and float(self.ab.max()) / rb.Q_DB < rb.SUM_LIMIT
        assert self.rows > 0
        return self.ratio, float(self.ag.max()) / rb.Q_DG / rb.SUM_LIMIT


def row_case_premises(layer, n, dtype, m, seed):
    g = rb.gamma(seed, n)
    p = Premises(n, rw.DT[dtype], layer, False)
    for r0 in range(0, m, CHUNK):
        idx = torch.arange(r0, min(m, r0 + CHUNK))
        lv = rb.row_live(seed, idx, m, n)
        idx = idx[lv]
        p.add(rb.rows(seed, idx, n, g, layer=layer), g)
    # the forced rows are live
    assert bool(rb.row_live(seed, rb.row_forced(m, n), m, n).all())
    return p.done()


def prep_case_premises(B, S, H, D, norm, rope, lo, n, dtype, seed):
    N = H * D if norm == 3 else D
    tok = rb.prep_live(seed, B, S, H, D, norm, lo, n).nonzero()[:, 0]
    out = []
    for i in range(2):
        g = rb.gamma(seed * 3 + i, N)
        p = Premises(N, rw.DT[dtype], norm == 2, norm == 3)
        step = max(1, CHUNK // (H * D))
        for t0 in range(0, tok.shape[0], step):
            tk = tok[t0:t0 + step]
            idx = tk if norm == 3 else (tk[:, None] * H + torch.arange(H)).reshape(-1)
            p.add(rb.rows(seed * 3 + i, idx, N, g, layer=norm == 2), g)
        out.append(p.done())
    return min(o[0] for o in out), max(o[1] for o in out)


def report(capsys, what, ratio, fill):
    with capsys.disabled():
        print(f"\n  {what}: margin / error bound >= {ratio:.3g}, largest dgamma sum {fill:.3f} of 2^24 quanta", end="")


@pytest.mark.parametrize("layer, n, dtype, m, seed", rb.ROW_CASES + rb.ROW_CASES_HY + rb.AUTOGRAD_ROW_CASES)
def test_row_norm_case_premises(layer, n, dtype, m, seed, capsys):
    report(capsys, f"{'layer' if layer else 'rms'} n {n} {dtype} m {m}", *row_case_premises(layer, n, dtype, m, seed))


PREP_ALL = rb.PREP_CASES + rb.PREP_CASES_THRESHOLD + rb.HIDDEN_CASES + rb.PREP_CASES_FULL


@pytest.mark.parametrize("B, S, H, D, norm, rope, lo, n, dtype, seed",
                         [c[:10] for c in PREP_ALL] + rb.AUTOGRAD_PREP_CASES)
def test_prep_case_premises(B, S, H, D, norm, rope, lo, n, dtype, seed, capsys):
    report(capsys, f"prep B {B} S {S} H {H} D {D} norm {norm} rope {rope} {dtype}",
           *prep_case_premises(B, S, H, D, norm, rope, lo, n, dtype, seed))


def test_eps_absorbed_at_the_census_variances():
    """fp32(var + eps) == var: RMS (eps 1e-6) at every census variance, LayerNorm (1e-5) at var 256 and 1024; at var
    64 LayerNorm's eps is not absorbed, which is why its rows keep to LN_JS."""
    f32 = lambda v: torch.tensor(v, dtype=torch.float32)  # noqa: E731
    for j in rw.JS:
        var = 16.0 * 4 ** j
        assert f32(var) + f32(rb.RMS_EPS) == f32(var)
    for j in rb.LN_JS:
        var = 16.0 * 4 ** j
        assert f32(var) + f32(rb.LN_EPS) == f32(var)
    assert f32(64.0) + f32(rb.LN_EPS) != f32(64.0)
    assert min(rb.LN_JS) >= 2


def test_e_vectors_and_closed_form():
    """Every e is orthogonal to 1 and to its block, so over any row mean(u x^) = m0 and mean(u) = mean(c)."""
    E, Bk = rb.E_VECS, rw.BLOCKS
    assert torch.equal(E.sum(-1), torch.zeros(E.shape[:2]))
    assert torch.equal((E * Bk[:, None, :]).sum(-1), torch.zeros(E.shape[:2]))
    assert bool((E.abs().sum(-1) > 0).all())
    for layer in (False, True):
        for N in (32, 256, 5120) if not layer else (32, 256):
            g = rb.gamma(1, N)
            c = rb.rows(1, torch.arange(300), N, g, layer=layer)
            assert torch.equal((c["u"] * c["xh"]).mean(-1), c["m0"])
            assert torch.equal(c["u"] * 1, c["dn"] * g)
            assert set(c["m0"].tolist()) == set(rb.M0S)
    assert {abs(v) for v in rb.GAMMAS} == {0.5, 1.0, 2.0}
    assert set(rb.gamma(0, 4096).tolist()) == set(rb.GAMMAS)


def test_dead_rows_give_zero():
    g = rb.gamma(2, 64)
    idx = torch.arange(500)
    lv = idx % 3 == 0
    c = rb.rows(2, idx, 64, g, layer=True, live=lv)
    assert bool((c["dn"][~lv] == 0).all() and (c["dx"][~lv] == 0).all())
    assert bool((c["dx"][lv] != 0).all())
    assert torch.equal(rb.norm_bwd(c["x"], c["dn"], g, layer=True), c["dx"])


@pytest.mark.parametrize("rope", [1, 2])
def test_quarter_turn_tables_invert_exactly(rope):
    """The kernels' transpose of dy = RoPE(dn) is dn exactly, and no rotated row uses the identity."""
    D, n = 128, 300
    c, s = rb.quarter_tables(4, n, D, rope)
    pairs = set(zip(c.flatten().tolist(), s.flatten().tolist()))
    assert pairs == set(rb.QUARTER) and (1.0, 0.0) not in pairs
    if rope == 1:
        assert torch.equal(c[:, 0::2], c[:, 1::2]) and torch.equal(s[:, 0::2], s[:, 1::2])
    dn = rb.rows(4, torch.arange(3 * n), D, rb.gamma(4, D), layer=False)["dn"].view(3, n, D)
    dy = rb.rotate(dn, c, s, rope)
    assert torch.equal(rope_t(dy, c, s, rope), dn)
    assert bool((dy != dn).any(-1).all())                     # every rotated row moves


# ---- geometry ----------------------------------------------------------------------------------------------------
def test_constants_match_prep_cu():
    src = (ROOT / "sparse-videogen_b200" / "csrc" / "prep.cu").read_text()
    assert re.search(r"constexpr int kBwdCtas = 148 \* 4;", src)
    assert re.search(r"constexpr int kHiddenThreads = 128;", src)
    assert re.search(r"constexpr int kThreads = 256;", src)
    assert re.search(r"#define SVGB_PREP_UNROLL 4\b", src)
    assert rb.BWD_CTAS == 592 and rb.HIDDEN_THREADS == 128 and rb.THREADS == 256 and rb.UNROLL == 4


@pytest.fixture(scope="module")
def lib():
    import importlib.util

    spec = importlib.util.spec_from_file_location("svgb200_build", ROOT / "sparse-videogen_b200" / "build.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.build_lib()
    from svgb200 import _lib

    return _lib.lib()


def align(v):
    return -(-v // 256) * 256


def test_geometry_matches_the_workspace_sizes(lib):
    """The C entry points size their workspaces from row_blocks, prep_bwd_blocks and hidden_splits: the oracle's
    helpers give the same sizes on every case shape, and around the caps."""
    nb = C.c_size_t()
    rows = {(c[3], c[1]) for c in rb.ROW_CASES + rb.ROW_CASES_HY}
    rows |= {(m, n) for n in rw.NORM_NS for m in (rb.row_threshold(n) - rb.rpb(n) * 4, rb.row_threshold(n) + 1)}
    for m, n in rows:
        assert lib.svgb_row_norm_bwd_bytes(m, n, C.byref(nb)) == 0
        assert nb.value == align(4 * 2 * n * rb.row_blocks(m, n)), (m, n)
    for c in PREP_ALL + [(1, 5, 7, 64, 1), (3, 9999, 2, 128, 2), (600, 2, 1, 256, 1), (2, 300, 40, 128, 3)]:
        B, S, H, D, norm = c[:5]
        assert lib.svgb_qkv_prep_bwd_bytes(B, S, H, D, norm, C.byref(nb)) == 0
        if norm in (1, 2):
            assert nb.value == 2 * align(4 * 2 * D * rb.prep_bwd_blocks(B, S, D) * B), c
        else:
            assert nb.value == 2 * align(4 * H * D * rb.hidden_splits(B, S, H, D)) + 2 * align(8 * B * S), c


def test_cases_cross_the_grids():
    """Each case crosses the boundary it is there for."""
    for layer, n, dt, m, seed in rb.ROW_CASES:
        assert rb.row_passes(m, n) == (2 if m > rb.row_threshold(n) else 1)
    for n in rw.NORM_NS:
        one, dead, below, above = rb.row_norm_rows(n)
        assert one == 1 and dead < rb.rpb(n) and rb.row_blocks(dead, n) == 1
        assert rb.row_passes(below, n) == 1 and rb.row_passes(above, n) == 2
        assert below % (rb.rpb(n) * rb.UNROLL) and above % (rb.rpb(n) * rb.UNROLL)
    assert rb.row_passes(rw.HY_NORM_ROWS, rw.HY_NORM_N) == 76
    for c in rb.PREP_CASES_THRESHOLD:
        B, S, D = c[0], c[1], c[3]
        assert S % rb.rpb(D) and rb.prep_passes(B, S, D) == (2 if S > rb.prep_threshold(B, D) else 1)
    assert {rb.prep_passes(c[0], c[1], c[3]) for c in rb.PREP_CASES_THRESHOLD} == {1, 2}
    for B, S, H, D, *_ in rb.HIDDEN_CASES:
        assert (H * D // 8) % rb.HIDDEN_THREADS                          # threads past H * LPR return early
    spl = [(B * S, rb.hidden_splits(B, S, H, D)) for B, S, H, D, *_ in rb.HIDDEN_CASES]
    assert any(T == s for T, s in spl) and any(T > 3 * s for T, s in spl)  # one token per split, and many
    crossing = 0
    for B, S, H, D, *_ in rb.HIDDEN_CASES:
        per = -(-B * S // rb.hidden_splits(B, S, H, D))
        crossing += B == 2 and S % per != 0
    assert crossing >= 2
    assert any(rb.hidden_cols(H, D) > 1 for B, S, H, D, *_ in rb.HIDDEN_CASES)
    wan = rb.PREP_CASES_FULL[0]
    assert rb.hidden_splits(1, wan[1], wan[2], wan[3]) == 118 and rb.prep_passes(1, wan[1], wan[3]) == 8
    hy = rb.PREP_CASES_FULL[1]
    assert rb.prep_passes(1, hy[1], hy[3]) == 13 and hy[1] - hy[7] == rw.HY_TXT


def test_forced_rows_cover_the_boundaries():
    """walk_ends / split_ends against a direct enumeration of each CTA's rows / each split's tokens."""
    for units, group, grid in ((1000, 8, 7), (37905, 16, 592), (5, 8, 1), (4757, 16, 296)):
        cta = torch.arange(units) // group % grid
        want = set()
        for b in range(grid):
            r = (cta == b).nonzero()[:, 0]
            if r.numel():
                want |= {int(r[0]), int(r[-1])}
        assert set(rb.walk_ends(units, group, grid).tolist()) == want
    for T, splits in ((2002, 592), (400, 400), (1000, 197)):
        per = -(-T // splits)
        sp = torch.arange(T) // per
        want = set()
        for s in range(splits):
            r = (sp == s).nonzero()[:, 0]
            if r.numel():
                want |= {int(r[0]), int(r[-1])}
        assert set(rb.split_ends(T, splits).tolist()) == want
    B, S, H, D, norm, rope, lo, n = rb.HIDDEN_CASES[1][:8]
    f = set(rb.prep_forced(B, S, H, D, norm, lo, n).tolist())
    assert {lo - 1, lo, lo + n - 1, lo + n, S - 1, S, S + lo} <= f       # RoPE range and batch boundary


# ---- sensitivity -------------------------------------------------------------------------------------------------
def changed(a, b, dtype):
    return (rw.round_to(a, dtype).double() != rw.round_to(b, dtype).double()).double().mean().item()


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("N", [32, 64, 128, 256])
def test_formula_mutants_change_dx(N, dtype):
    """A divisor N - 1 moves dx by about 1/N of the m0 x^ term (the shift shrinks with N, yet in bf16 at N = 256 it
    still moves about half the elements); a dropped term moves nearly all."""
    for layer in (False, True):
        g = rb.gamma(N, N)
        c = rb.rows(N, torch.arange(2048), N, g, layer=layer)
        x, dn, ref = c["x"], c["dn"], c["dx"]
        mut = lambda **kw: rb.norm_bwd(x, dn, g, layer=layer, **kw)  # noqa: E731
        assert torch.equal(mut(), ref)
        assert changed(ref, mut(div=N - 1), dtype) > 0.4            # mean(u x^) over N - 1
        assert changed(ref, mut(drop_ux=True), dtype) > 0.9          # no x^ mean(u x^) term
        if layer:
            assert changed(ref, mut(div_u=N - 1), dtype) > 0.2      # mean(u) over N - 1
            assert changed(ref, mut(drop_u=True), dtype) > 0.9      # no mean(u) term


def test_hidden_mutants_change_dx():
    H, D = rw.WAN_H, rw.WAN_D
    HD = H * D
    g = rb.gamma(9, HD)
    c = rb.rows(9, torch.arange(256), HD, g, layer=False)
    x, dn, ref = c["x"], c["dn"], c["dx"]
    for dtype in DTYPES:
        assert changed(ref, rb.norm_bwd(x, dn, g, layer=False, div=HD - 1), dtype) > 5e-3          # m over HD - 1
        assert changed(ref, rb.norm_bwd(x, dn, g, layer=False, div=D), dtype) > 0.5                 # m over D
        assert changed(ref, rb.norm_bwd(x, dn, g, layer=False, rstd=c["rstd"] * H ** -0.5), dtype) > 0.9  # r over D
        assert changed(ref, rb.norm_bwd(x, dn, g[torch.arange(HD) % D], layer=False), dtype) > 0.5  # gamma[c % D]
    # stats of batch 0 read for batch 1 (same token): r and m of another row
    B, S = 2, 128
    rs, m0 = c["rstd"].view(B, S), c["m0"].view(B, S)
    xb, ub = x.double().view(B, S, HD), c["u"].view(B, S, HD)
    wrong = rs[0, :, None] * (ub[1] - xb[1] * rs[0, :, None] * m0[0, :, None])
    assert changed(ref.view(B, S, HD)[1], wrong, torch.bfloat16) > 0.5


def test_dgamma_mutants_change_sums():
    """dgamma summing u x^ instead of dn x^, and the last CTA's (split's) partial dropped or counted twice."""
    n = 128
    m = rb.row_norm_rows(n)[3]                                         # two passes of 592 CTAs
    g = rb.gamma(5, n)
    idx = torch.arange(m)
    c = rb.rows(5, idx, n, g, layer=True, live=rb.row_live(5, idx, m, n))
    t = c["dn"] * c["xh"]
    dg = t.sum(0).float()
    assert (dg != (c["u"] * c["xh"]).sum(0).float()).double().mean() > 0.5
    cta = idx // rb.rpb(n) % rb.row_blocks(m, n)
    last = cta == rb.row_blocks(m, n) - 1
    for part, total in ((t[last].sum(0), dg), (c["dn"][last].sum(0), c["dn"].sum(0).float())):
        assert (total != (total.double() - part).float()).double().mean() > 0.5
        assert (total != (total.double() + part).float()).double().mean() > 0.5
    # the hidden path's last non-empty split
    B, S, H, D = rb.HIDDEN_CASES[1][:4]
    T, splits = B * S, rb.hidden_splits(B, S, H, D)
    per = -(-T // splits)
    tok = torch.arange(T)
    gh = rb.gamma(6, H * D)
    ch = rb.rows(6, tok, H * D, gh, layer=False, live=rb.prep_live(6, B, S, H, D, 3, 17, 981))
    th = ch["dn"] * ch["xh"]
    lastsplit = tok // per == (T - 1) // per
    total = th.sum(0).float()
    assert (total != (total.double() - th[lastsplit].sum(0)).float()).double().mean() > 0.5


@pytest.mark.parametrize("rope", [1, 2])
def test_rope_range_off_by_one_changes_dx(rope):
    """The first and last rotated token treated as text, and the text tokens next to the range rotated: dx of the
    whole head row changes."""
    D, H, n = 128, 3, 20
    g = rb.gamma(7, D)
    c = rb.rows(7, torch.arange((n + 2) * H), D, g, layer=False)
    x, dn, ref = c["x"].view(n + 2, H, D), c["dn"].view(n + 2, H, D), c["dx"].view(n + 2, H, D)
    cos, sin = rb.quarter_tables(7, n, D, rope)
    lo = 1                                                              # tokens 1 .. n rotated, 0 and n + 1 text
    dy = dn.clone()
    dy[lo:lo + n] = rb.rotate(dn[lo:lo + n].transpose(0, 1), cos, sin, rope).transpose(0, 1)
    for t in (lo, lo + n - 1):                                           # rotated token read as text
        got = rb.norm_bwd(x[t], dy[t], g, layer=False)
        assert changed(ref[t], got, torch.bfloat16) > 0.5
    for t, row in ((lo - 1, 0), (lo + n, n - 1)):                        # text token rotated by a neighbour's table
        d = rope_t(dy[t], cos[row:row + 1].expand(H, -1), sin[row:row + 1].expand(H, -1), rope)
        assert changed(ref[t], rb.norm_bwd(x[t], d, g, layer=False), torch.bfloat16) > 0.5
