"""CPU proof that the row-wise census (tests/test_rowwise_census_gpu.py, oracle/rowwise.py) is exact and sees the bugs
it is meant to see, plus the host-side argument checks of the Wan block glue.

  * premises: every row's sums are integers below 2^24 and |x| is exact in bf16; every glue intermediate is exact in
    fp32; every norm output is representable in its 16-bit dtype with a margin that rsqrtf, eps and the fp32
    roundings cannot cross (the smallest margin / error-bound ratio is printed per case);
  * coverage: all ten glue instantiations, every norm width and head dim, every RoPE mode and every qkv_prep
    norm x rope combination; each production-size case crosses the grid cap or the multi-pass threshold it claims to;
  * sensitivity: oracle-level mutants (a gamma column shifted, the modulation batch off by one, a row taking its
    neighbour's or the row a grid ahead's data, the text range off by one, LayerNorm without centring) change many
    expected elements.
"""
import ctypes as C
from pathlib import Path

import pytest
import torch

from oracle import rowwise as rw

ROOT = Path(__file__).resolve().parent.parent
DTYPES = (torch.bfloat16, torch.float16)


def gen(seed=0):
    return torch.Generator().manual_seed(seed)


# ---- premises ----------------------------------------------------------------------------------------------------
def test_blocks_and_rows_are_exact():
    assert rw.BLOCKS.shape[0] >= 32
    assert torch.equal(rw.BLOCKS.sum(1), torch.zeros(rw.BLOCKS.shape[0]))
    assert torch.equal((rw.BLOCKS ** 2).sum(1), torch.full((rw.BLOCKS.shape[0],), 128.0))
    for centred in (False, True):
        x, rstd = rw.row_x(1, 300, 264, centred=centred)
        c = x.double() - (x.double().mean(1, keepdim=True) if centred else 0)
        assert torch.equal((c * c).mean(1), rstd ** -2)                      # var (mean square) = rstd^-2 exactly
        assert x.abs().max() <= rw.XMAX and rw.row_sums_ok(x, centred)
        assert torch.unique(rw.xhat(x, rstd, centred) * 4).numel() == 13     # x^ in {-3/2, ..., 3/2}
        # chunks built from row0 are the same rows (the GPU builds production inputs in chunks)
        x2, r2 = rw.row_x(1, 100, 264, centred=centred, row0=150)
        assert torch.equal(x2, x[150:250]) and torch.equal(r2, rstd[150:250])
    m, j = rw.row_params(1, 10000)
    assert m.unique().numel() == 2 * rw.MMAX + 1 and j.unique().numel() == len(rw.JS)
    assert rw.XMAX <= 256 and 16 * 4 ** min(rw.JS) >= 64                   # exact in bf16; eps 1e-6 absorbed


def test_sums_below_2_24_at_the_widest_rows():
    """The largest row sums of any case: N = 8192 glue rows and 5120-wide hidden RMS rows at the largest j."""
    for N in (8192, 5120):
        lim = 2.0 ** 24
        assert N * rw.XMAX < lim                         # sum |x|
        assert N * 16 * 4 ** max(rw.JS) < lim            # sum x^2 of RMS rows, sum (x - mean)^2: N var, partials below


def glue_premises(rows, N, nb, seed, r0=0, total=None):
    """Every intermediate of the four glue ops exact in fp32, on rows [r0, r0 + rows) of a case of `total` rows in nb
    batches."""
    g = gen(seed)
    x, rstd = rw.row_x(seed, rows, N, centred=True, row0=r0)
    xc, rc = rw.row_x(seed, rows, N, centred=False, row0=r0)
    assert rw.row_sums_ok(x, True) and rw.row_sums_ok(xc, False)
    w, b = rw.gammas((N,), g), rw.shifts((N,), g)
    sc, sh, gt = (f((nb, N), g) for f in (rw.scales, rw.shifts, rw.gammas))
    res = rw.residuals((rows, N), g)
    ms = lambda v: rw.mod_slice(v, total or rows, r0, r0 + rows)  # noqa: E731
    xh = rw.xhat(x, rstd, True)
    o = xh * w.double()
    steps = [xh, o, o + b.double(), 1 + ms(sc), (o + b.double()) * (1 + ms(sc)),
             rw.glue_layernorm(x, rstd, w.to(torch.bfloat16).float(), b.to(torch.bfloat16).float(), ms(sc), ms(sh)),
             rw.glue_rmsnorm(xc, rc, w), x.double() * (1 + ms(sc)), rw.glue_modulate(x, ms(sc), ms(sh)),
             x.double() * ms(gt), rw.glue_gate_residual(res, x, ms(gt))]
    assert rw.fp32_exact(*steps)
    for t in (w, b, res):
        assert rw.exact_in(t, torch.bfloat16) and rw.exact_in(t, torch.float16)
    assert ((1 + sc) > 0).all()


@pytest.mark.parametrize("N", rw.GLUE_NS)
def test_glue_premises(N):
    for rows in rw.GLUE_ROWS:
        glue_premises(rows, N, rw.GLUE_MOD[rows], seed=N + rows)


def test_glue_premises_production():
    """Wan 720p rows, sampled at the start, across the batch boundary and at the end."""
    for r0 in (0, rw.WAN_ROWS // 2 - 64, rw.WAN_ROWS - 128):
        glue_premises(128, rw.WAN_N, 2, seed=r0, r0=r0, total=rw.WAN_ROWS)


def norm_case_margin(m_rows, n, layer, dtype, seed, r0=0):
    g = gen(seed)
    x, rstd = rw.row_x(seed, m_rows, n, centred=layer, row0=r0)
    gm = rw.gammas((n,), g)
    b = rw.betas((n,), g) if layer else None
    assert rw.exact_in(gm, dtype) and (b is None or rw.exact_in(b, dtype)) and rw.exact_in(x, dtype)
    assert rw.row_sums_ok(x, layer)
    v = rw.row_norm(x, rstd, gm, b)
    scale = (rw.xhat(x, rstd, layer) * gm.double()).abs() + (0 if b is None else b.double().abs())
    return rw.norm_margin_ok(v, scale, dtype)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("layer", [False, True])
@pytest.mark.parametrize("n", rw.NORM_NS)
def test_norm_margins(n, layer, dtype, capsys):
    """Standalone norms (n) and per-head norms of qkv_prep (D): v exactly representable, far from a rounding
    boundary.  Rows sampled from the start and from past the multi-pass threshold."""
    for r0 in (0, rw.norm_threshold(n) - 100):
        ok, ratio = norm_case_margin(512, n, layer, dtype, seed=n + layer, r0=r0)
        with capsys.disabled():
            print(f"\n  norm n {n} {'layer' if layer else 'rms'} {dtype}: margin / error bound >= {ratio:.3g}", end="")
        assert ok, (n, layer, dtype, ratio)


def test_norm_margin_catches_unrepresentable_and_cancelled():
    v = torch.tensor([1.0 + 2 ** -9])
    assert not rw.norm_margin_ok(v, v.abs(), torch.bfloat16)[0]             # not a bf16 value
    assert rw.norm_margin_ok(v, v.abs(), torch.float16)[0]
    assert not rw.norm_margin_ok(torch.tensor([0.0]), torch.tensor([3.0]), torch.float16)[0]   # cancelled to 0
    assert rw.norm_margin_ok(torch.tensor([0.0]), torch.tensor([0.0]), torch.float16)[0]       # an exact 0
    assert rw.betas((10000,), gen()).mul(32).remainder(2).eq(1).all()        # beta never cancels x^ g exactly


def test_rope_and_prep_outputs_exact_in_fp32():
    """The rotation of a 16-bit value (the input, or the norm output rounded to 16 bits) by tables from
    {-1, -1/2, 0, 1/2, 1} is exact in fp32, so the kernel's one rounding meets the closed form's."""
    g = gen(3)
    for complex_ in (False, True):
        for dtype in DTYPES:
            x, rstd = rw.row_x(3, 400, 128, centred=True)
            v = rw.round_to(rw.row_norm(x, rstd, rw.gammas((128,), g), rw.betas((128,), g)), dtype).double()
            c, s = rw.census_tables(400, 64 if complex_ else 128, g)
            assert rw.fp32_exact(rw.rope(v, c, s, complex_), rw.rope(x, c, s, complex_))
            q = torch.randint(-100, 101, (400, 128), generator=g).to(dtype)
            assert rw.fp32_exact(rw.rope(q, c, s, complex_))


def test_hidden_rms_is_exact():
    """NORM_RMS_HIDDEN (IEEE sqrtf over H*D = 5120): x^ gamma exact and representable in both 16-bit dtypes."""
    x, rstd = rw.row_x(5, 64, rw.WAN_H * rw.WAN_D, centred=False)
    v = rw.xhat(x, rstd, False) * rw.gammas((rw.WAN_H * rw.WAN_D,), gen()).double()
    for dtype in DTYPES:
        assert rw.exact_in(v, dtype)


# ---- coverage ----------------------------------------------------------------------------------------------------
def test_glue_coverage():
    inst = {rw.glue_instantiation(op, x, r) for op, x, _, r in rw.glue_dtype_cases()}
    assert len(inst) == 10                                       # LN 2 + RMS 2 + modulate 2 + gate_residual 4
    cases = rw.glue_dtype_cases()
    assert {c[2] for c in cases} == {"bf16", "fp16", "fp32"}
    assert {c[3] for c in cases if c[0] == "layernorm"} == {None, "bf16", "fp16", "fp32"}
    assert 8 in rw.GLUE_NS and rw.GLUE_MAX_N in rw.GLUE_NS
    vec = lambda N: -(-(N // 8) // rw.GLUE_THREADS)  # noqa: E731  8-element groups per thread
    assert vec(2048) == 1 and vec(2056) == 2 and vec(rw.GLUE_MAX_N) == rw.GLUE_MAX_VEC
    walks = [r for r in rw.GLUE_ROWS if r > rw.glue_grid(r)]
    assert walks and max(rw.GLUE_ROWS) > 2 * rw.GLUE_GRID        # some CTAs walk three rows
    for rows, nb in rw.GLUE_MOD.items():
        assert rows % nb == 0
        if 1 < nb < rows:
            rpb = rows // nb
            assert rpb % rw.GLUE_GRID and rpb < rows            # batch boundaries fall inside CTA walks
    # the dtype sweep: CTA 0 walks rows 0 and 1184, in different batches
    assert rw.GLUE_DT_B * rw.GLUE_DT_S > rw.GLUE_GRID and rw.GLUE_GRID // rw.GLUE_DT_S != 0
    assert rw.WAN_ROWS // rw.glue_grid(rw.WAN_ROWS) >= 63


def test_norm_coverage():
    assert rw.NORM_NS == (32, 64, 128, 256) and rw.HEAD_DIMS == (64, 128, 256)
    for n, t in zip(rw.NORM_NS, (1212416, 606208, 303104, 151552)):
        assert rw.norm_threshold(n) == t
        below, above = rw.norm_rows(n)
        assert rw.norm_passes(below, n) == 1 and rw.norm_passes(above, n) == 2
        unit = rw.NORM_THREADS // (n // 8) * rw.NORM_UNROLL
        assert below % unit and above % unit
    assert rw.norm_passes(rw.HY_NORM_ROWS, rw.HY_NORM_N) == 10
    assert rw.HY_S * rw.HY_H == rw.HY_NORM_ROWS


# ---- sensitivity -------------------------------------------------------------------------------------------------
def changed(a, b, dtype=torch.float32):
    return (rw.round_to(a, dtype).double() != rw.round_to(b, dtype).double()).double().mean().item()


def test_glue_mutants_change_outputs():
    rows, N, nb = 2 * rw.GLUE_GRID + 4, 264, 4
    g = gen(9)
    x, rstd = rw.row_x(9, rows, N, centred=True)
    w, b = rw.gammas((N,), g), rw.shifts((N,), g)
    sc, sh, gt = (f((nb, N), g) for f in (rw.scales, rw.shifts, rw.gammas))
    ms = lambda v: rw.mod_slice(v, rows, 0, rows)  # noqa: E731
    ref = rw.glue_layernorm(x, rstd, w, b, ms(sc), ms(sh))
    assert changed(ref, rw.glue_layernorm(x, rstd, w.roll(1), b, ms(sc), ms(sh))) > 0.5          # gamma column
    off = lambda v: rw.mod_slice(v.roll(1, 0), rows, 0, rows)  # noqa: E731                      # batch off by one
    assert changed(ref, rw.glue_layernorm(x, rstd, w, b, off(sc), off(sh))) > 0.5
    # the modulation by blockIdx.x / rows_per_batch, not row / rows_per_batch: wrong past each CTA's first row
    blk = torch.arange(rows) % rw.GLUE_GRID // (rows // nb)
    sc_b, sh_b = sc.double()[blk], sh.double()[blk]
    assert changed(ref, rw.glue_layernorm(x, rstd, w, b, sc_b, sh_b)) > 0.4
    assert changed(ref, rw.glue_layernorm(x.roll(1, 0), rstd.roll(1, 0), w, b, ms(sc), ms(sh))) > 0.5   # neighbour
    # a stale prefetch: row r + grid keeps row r's data
    stale = torch.arange(rows)
    stale[rw.GLUE_GRID:] -= rw.GLUE_GRID
    got = rw.glue_layernorm(x[stale], rstd[stale], w, b, ms(sc), ms(sh))
    assert changed(ref[rw.GLUE_GRID:], got[rw.GLUE_GRID:]) > 0.5
    assert changed(ref, rw.glue_layernorm(x, rstd, w, b, ms(sc), ms(sh), centred=False)) > 0.9    # no centring
    res = rw.residuals((rows, N), g)
    ref = rw.glue_gate_residual(res, x, ms(gt))
    assert changed(ref, rw.glue_gate_residual(res, x, rw.mod_slice(gt.roll(1, 0), rows, 0, rows))) > 0.5


@pytest.mark.parametrize("dtype", DTYPES)
def test_norm_mutants_change_outputs(dtype):
    n, rows = 128, 4096
    g = gen(4)
    x, rstd = rw.row_x(4, rows, n, centred=True)
    gm, b = rw.gammas((n,), g), rw.betas((n,), g)
    ref = rw.row_norm(x, rstd, gm, b)
    assert changed(ref, rw.row_norm(x, rstd, gm.roll(1), b), dtype) > 0.5
    assert changed(ref, rw.row_norm(x.roll(16, 0), rstd.roll(16, 0), gm, b), dtype) > 0.5  # a row group ahead
    assert changed(ref, rw.row_norm(x, rstd, gm, None), dtype) > 0.9                        # no beta
    nc = rw.xhat(x, rstd, False) * gm.double() + b.double()                                 # no centring
    assert changed(ref, nc, dtype) > 0.9
    xr, rr = rw.row_x(4, rows, n, centred=False)
    assert changed(rw.row_norm(xr, rr, gm), rw.row_norm(xr.roll(1, 0), rr.roll(1, 0), gm), dtype) > 0.5


@pytest.mark.parametrize("complex_", [False, True])
def test_rope_text_range_off_by_one_changes_outputs(complex_):
    g = gen(5)
    n, D = 64, 128
    q = torch.randint(-100, 101, (3, n + 1, D), generator=g).double()
    c, s = rw.census_tables(n + 1, D // 2 if complex_ else D, g)
    ref = rw.rope(q[:, 1:], c[:n], s[:n], complex_)
    shifted = rw.rope(q[:, 1:], c[1:], s[1:], complex_)          # tables read one row off
    assert changed(ref, shifted) > 0.5
    assert changed(q[:, :1], rw.rope(q[:, :1], c[:1], s[:1], complex_)) > 0.5   # a text row rotated


# ---- host side: the glue's C ABI and the wrappers' checks --------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    import importlib.util

    spec = importlib.util.spec_from_file_location("svgb200_build", ROOT / "sparse-videogen_b200" / "build.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.build_lib()
    from svgb200 import _lib

    return _lib.lib()


def test_glue_abi_argument_errors(lib):
    A = 256  # a 16-byte aligned stand-in address: every call below fails its checks before touching memory
    BF, F32 = 0, 3

    def ln(N=64, x=A, xd=BF, w=A, b=A, wd=F32, sc=A, sh=A, y=A, yd=F32, rows=10):
        return lib.svgb_layernorm_modulate(x, xd, w, b, wd, 1e-6, sc, sh, 0, y, yd, rows, N, None)

    for kw, msg in ((dict(N=60), b"multiple of 8"), (dict(N=8200), b"multiple of 8 and <= 8192"),
                    (dict(N=0), b"multiple of 8"), (dict(x=A + 8), b"16-byte aligned"), (dict(y=A + 4), b"16-byte"),
                    (dict(w=A + 8), b"16-byte"), (dict(sh=A + 8), b"16-byte"), (dict(xd=2), b"dtype"),
                    (dict(yd=4), b"dtype"), (dict(wd=2), b"weight dtype"), (dict(b=None), b"weight and bias"),
                    (dict(w=None), b"weight and bias"), (dict(sh=None), b"scale and shift"), (dict(x=None), b"null"),
                    (dict(rows=-1), b"hidden size")):
        assert ln(**kw) < 0, kw
        assert msg in lib.svgb_last_error(), (kw, lib.svgb_last_error())
    assert lib.svgb_rmsnorm_hidden(A, BF, None, F32, 1e-6, A, BF, 10, 64, None) < 0
    assert b"weight required" in lib.svgb_last_error()
    assert lib.svgb_rmsnorm_hidden(A, BF, A, 2, 1e-6, A, BF, 10, 64, None) < 0
    assert lib.svgb_rmsnorm_hidden(A, BF, A, BF, 1e-6, A, BF, 10, 8200, None) < 0
    assert b"8192" in lib.svgb_last_error()
    assert lib.svgb_modulate_shift(A, BF, A, None, 0, A, F32, 10, 64, None) < 0
    assert lib.svgb_modulate_shift(A, BF, A + 4, A, 0, A, F32, 10, 64, None) < 0
    assert b"16-byte" in lib.svgb_last_error()
    assert lib.svgb_gate_residual(A, 2, A, BF, A, 0, A, F32, 10, 64, None) < 0
    assert lib.svgb_gate_residual(None, BF, A, BF, A, 0, A, F32, 10, 64, None) < 0
    assert lib.svgb_gate_residual(A + 8, BF, A, BF, A, 0, A, F32, 10, 64, None) < 0
    assert b"16-byte" in lib.svgb_last_error()
    assert lib.svgb_gate_residual(A, BF, A, BF, A, 0, A, F32, 10, 12, None) < 0
    # zero rows is not an error, and launches nothing
    assert lib.svgb_gate_residual(A, BF, A, BF, A, 0, A, F32, 0, 64, None) == 0


# The wrappers validate shapes and dtypes before any device work, so these run on CPU tensors.
def test_modulate_shift_checks_the_shift_batch():
    from svgb200 import core
    from svgb200._lib import SvgbError

    x = torch.zeros(2, 5, 64)
    with pytest.raises(SvgbError, match="scale and shift must have the same batch"):
        core.modulate_shift(x, torch.zeros(2, 1, 64), torch.zeros(1, 64))
    with pytest.raises(SvgbError, match="scale and shift must have the same batch"):
        core.modulate_shift(x, torch.zeros(64), torch.zeros(2, 1, 64))


def test_layernorm_bias_must_match_the_weight_dtype():
    from svgb200 import core
    from svgb200._lib import SvgbError

    x = torch.zeros(3, 64)
    with pytest.raises(SvgbError, match="bias dtype"):
        core.layernorm_modulate(x, torch.ones(64, dtype=torch.bfloat16), torch.zeros(64))


def test_glue_norm_weights_must_hold_n_elements():
    from svgb200 import core
    from svgb200._lib import SvgbError

    x = torch.zeros(3, 64)
    with pytest.raises(SvgbError, match="weight must hold the hidden size 64"):
        core.layernorm_modulate(x, torch.ones(32), torch.zeros(64))
    with pytest.raises(SvgbError, match="bias must hold the hidden size 64"):
        core.layernorm_modulate(x, torch.ones(64), torch.zeros(32))
    with pytest.raises(SvgbError, match="weight must hold the hidden size 64"):
        core.rmsnorm_hidden(x, torch.ones(56), 1e-6)


def test_glue_unsupported_out_dtype_raises_svgb_error():
    from svgb200 import core
    from svgb200._lib import SvgbError

    x, v = torch.zeros(3, 64), torch.zeros(64)
    for call in (lambda: core.layernorm_modulate(x, out_dtype=torch.float64),
                 lambda: core.rmsnorm_hidden(x, v, 1e-6, out_dtype=torch.int8),
                 lambda: core.modulate_shift(x, v, v, out_dtype=torch.float64),
                 lambda: core.gate_residual(x, x, v, out_dtype=torch.int32)):
        with pytest.raises(SvgbError, match="unsupported out_dtype"):
            call()
