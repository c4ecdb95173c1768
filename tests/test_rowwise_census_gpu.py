"""Exact census of the row-wise forward kernels on the GPU (oracle/rowwise.py): the Wan block glue, the standalone QK
norms, the in-place RoPE and the fused qkv_prep forward, compared bit for bit (int16 / int32 views) with a closed
form, at the shapes where their grid-stride loops, prefetch buffers and row ranges come into play.  Outputs go into
NaN-filled buffers, so an element that is never written fails."""
import pytest
import torch

from oracle import rowwise as rw

pytestmark = pytest.mark.gpu

CHUNK = 1 << 23   # elements per chunk of the production-size builders and comparisons


def poison(cuda, nbytes=64 << 20):
    """Fill the caching allocator's free blocks with NaN so outputs the kernels never write show up."""
    t = torch.full((nbytes // 2 + 1,), float("nan"), dtype=torch.float16, device=cuda)
    del t


def assert_bits(got, want, what):
    """got == want bit for bit; else the count and the first differing (row, column) of the [-1, last dim] view."""
    assert got.dtype == want.dtype and got.shape == want.shape, f"{what}: {got.dtype} {got.shape} vs {want.dtype} {want.shape}"
    iv = {2: torch.int16, 4: torch.int32}[got.element_size()]
    ne = got.contiguous().view(iv) != want.contiguous().view(iv)
    if bool(ne.any()):
        r, c = (int(i) for i in ne.reshape(-1, got.shape[-1]).nonzero()[0])
        g, w = got.reshape(-1, got.shape[-1])[r, c].item(), want.reshape(-1, want.shape[-1])[r, c].item()
        raise AssertionError(f"{what}: {int(ne.sum())} elements differ; first at row {r}, column {c}: got {g}, want {w}")


def build_x(seed, rows, N, centred, dtype, cuda):
    """oracle rows built on the GPU in chunks, stored in dtype (exact); rstd [rows] float64."""
    x = torch.empty(rows, N, dtype=dtype, device=cuda)
    rstd = torch.empty(rows, dtype=torch.float64, device=cuda)
    step = max(1, CHUNK // N)
    for r0 in range(0, rows, step):
        n = min(step, rows - r0)
        xc, rc = rw.row_x(seed, n, N, centred=centred, row0=r0, device=cuda)
        x[r0:r0 + n], rstd[r0:r0 + n] = xc.to(dtype), rc
    return x, rstd


def compare_rows(y, expect, what):
    """y [..., N] against expect(r0, r1) (float64 rows r0..r1 of the [-1, N] view, exact in fp32), rounded once to
    y's dtype, in row chunks."""
    N = y.shape[-1]
    y = y.reshape(-1, N)
    step = max(1, CHUNK // N)
    for r0 in range(0, y.shape[0], step):
        r1 = min(y.shape[0], r0 + step)
        assert_bits(y[r0:r1], rw.round_to(expect(r0, r1), y.dtype), f"{what}, rows from {r0}")


# ---- 1. Wan block glue -------------------------------------------------------------------------------------------
def run_glue(cuda, op, rows, N, nb, *, seed, x_dt="bf16", y_dt="fp32", w_dt="fp32", res_dt="bf16", mod=True):
    """One glue op on `rows` census rows of N with nb modulation vectors ([nb, rows / nb, N] input), bit for bit."""
    from svgb200 import core

    gen = torch.Generator(device=cuda).manual_seed(seed)
    x, rstd = build_x(seed, rows, N, op != "rmsnorm", rw.DT[x_dt], cuda)
    shape = (nb, rows // nb, N) if nb > 1 else (rows, N)
    mshape = (nb, 1, N) if nb > 1 else (N,)
    Y = rw.DT[y_dt]
    ms = lambda v, r0, r1: rw.mod_slice(v, rows, r0, r1)  # noqa: E731
    what = f"{op} rows {rows} N {N} nb {nb} x {x_dt} y {y_dt} w {w_dt} res {res_dt} mod {mod}"
    if op == "layernorm":
        w = rw.gammas((N,), gen).to(rw.DT[w_dt]) if w_dt else None
        b = rw.shifts((N,), gen).to(rw.DT[w_dt]) if w_dt else None
        sc, sh = (rw.scales(mshape, gen), rw.shifts(mshape, gen)) if mod else (None, None)
        poison(cuda, rows * N * Y.itemsize + (1 << 20))
        y = core.layernorm_modulate(x.view(shape), w, b, rw.GLUE_EPS, sc, sh, out_dtype=Y)
        compare_rows(y, lambda r0, r1: rw.glue_layernorm(x[r0:r1], rstd[r0:r1], w, b, *(
            (ms(sc, r0, r1), ms(sh, r0, r1)) if mod else (None, None))), what)
    elif op == "rmsnorm":
        w = rw.gammas((N,), gen).to(rw.DT[w_dt])
        poison(cuda, rows * N * Y.itemsize + (1 << 20))
        y = core.rmsnorm_hidden(x.view(shape), w, rw.GLUE_EPS, out_dtype=Y)
        compare_rows(y, lambda r0, r1: rw.glue_rmsnorm(x[r0:r1], rstd[r0:r1], w), what)
    elif op == "modulate":
        sc, sh = rw.scales(mshape, gen), rw.shifts(mshape, gen)
        poison(cuda, rows * N * Y.itemsize + (1 << 20))
        y = core.modulate_shift(x.view(shape), sc, sh, out_dtype=Y)
        compare_rows(y, lambda r0, r1: rw.glue_modulate(x[r0:r1], ms(sc, r0, r1), ms(sh, r0, r1)), what)
    else:
        gt = rw.gammas(mshape, gen)
        res = rw.residuals((rows, N), gen).to(rw.DT[res_dt])
        poison(cuda, rows * N * Y.itemsize + (1 << 20))
        y = core.gate_residual(res.view(shape), x.view(shape), gt, out_dtype=Y)
        compare_rows(y, lambda r0, r1: rw.glue_gate_residual(res[r0:r1], x[r0:r1], ms(gt, r0, r1)), what)


@pytest.mark.parametrize("rows", rw.GLUE_ROWS)
@pytest.mark.parametrize("N", rw.GLUE_NS)
def test_glue_census_shapes(cuda, N, rows):
    """Every hidden size (kMaxVec boundaries 2048 / 2056, N = 8 and 8192) at row counts around the grid cap of 1184
    CTAs, where each CTA walks rows 1184 apart with the next row prefetched; modulation by one vector, per batch with
    rows_per_batch not a multiple of the grid, or per row (oracle GLUE_MOD)."""
    nb = rw.GLUE_MOD[rows]
    for i, op in enumerate(("layernorm", "rmsnorm", "modulate", "gate")):
        run_glue(cuda, op, rows, N, nb, seed=N * 10 + rows + i, x_dt="bf16" if N % 16 else "fp16",
                 y_dt="bf16" if op == "modulate" else "fp32")


@pytest.mark.parametrize("op", ["layernorm", "rmsnorm", "modulate", "gate"])
def test_glue_census_dtypes(cuda, op):
    """Every x / y / weight / residual dtype the wrappers pass (all ten kernel instantiations) at 1185 rows of 2056 in
    three batches of 395: CTA 0 walks rows 0 and 1184, in batches 0 and 2."""
    rows = rw.GLUE_DT_B * rw.GLUE_DT_S
    for i, (o, x, y, w) in enumerate(c for c in rw.glue_dtype_cases() if c[0] == op):
        kw = dict(res_dt=w) if op == "gate" else dict(w_dt=w)
        run_glue(cuda, op, rows, rw.GLUE_DT_N, rw.GLUE_DT_B, seed=100 + i, x_dt=x, y_dt=y,
                 mod=not (op == "layernorm" and w is not None and i % 2), **kw)


@pytest.mark.parametrize("op", ["layernorm", "modulate"])
@pytest.mark.parametrize("nb", [1, 4, 2372])
def test_glue_census_modulation(cuda, op, nb):
    """One modulation vector, four batches of 593 rows, and one vector per row, on 2372 rows of 264."""
    run_glue(cuda, op, 2372, 264, nb, seed=nb, y_dt="bf16")
    if op == "modulate":
        run_glue(cuda, "gate", 2372, 264, nb, seed=nb + 1, res_dt="fp32")


@pytest.mark.parametrize("B", [1, 2])
def test_glue_census_wan720p(cuda, B):
    """Wan 720p: 75 600 rows of 5120 (about 64 rows per CTA), B = 1 and B = 2 with [2, 1, N] modulation, including the
    fp32 residual stream."""
    R, N = rw.WAN_ROWS, rw.WAN_N
    run_glue(cuda, "layernorm", R, N, B, seed=B, w_dt=None, y_dt="bf16")
    run_glue(cuda, "gate", R, N, B, seed=B + 2, res_dt="fp32")
    if B == 2:
        run_glue(cuda, "layernorm", R, N, 1, seed=7, w_dt="fp32", mod=False)
        run_glue(cuda, "modulate", R, N, B, seed=8, y_dt="bf16")
        run_glue(cuda, "rmsnorm", R, N, 1, seed=9, w_dt="bf16", y_dt="bf16")


# ---- 2. standalone QK norms --------------------------------------------------------------------------------------
def run_norm(cuda, layer, m, n, dtype, seed):
    from svgb200 import core

    gen = torch.Generator(device=cuda).manual_seed(seed)
    x, rstd = build_x(seed, m, n, layer, dtype, cuda)
    g = rw.gammas((n,), gen).to(dtype)
    b = rw.betas((n,), gen).to(dtype) if layer else None
    xs = x.clone()
    if layer:
        core.layer_norm_(x, g, b)
    else:
        core.rms_norm_(x, g, 1e-6)
    compare_rows(x, lambda r0, r1: rw.row_norm(xs[r0:r1], rstd[r0:r1], g, b),
                 f"{'layer' if layer else 'rms'}_norm m {m} n {n} {dtype}")


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("n", rw.NORM_NS)
@pytest.mark.parametrize("layer", [False, True])
def test_norm_census_multipass(cuda, layer, n, dtype):
    """Row counts just below and just above the row where row_norm_kernel's grid-stride loop takes a second pass."""
    for i, m in enumerate(rw.norm_rows(n)):
        run_norm(cuda, layer, m, n, dtype, seed=n + i)


@pytest.mark.parametrize("layer", [False, True])
def test_norm_census_hunyuan720p(cuda, layer):
    """HunyuanVideo 720p's QK norm: 2 857 344 head rows of 128 (ten passes)."""
    run_norm(cuda, layer, rw.HY_NORM_ROWS, rw.HY_NORM_N, torch.bfloat16, seed=3 + layer)


# ---- 3. RoPE forward, in place -----------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("D", rw.HEAD_DIMS)
def test_rope_census_inplace(cuda, dtype, mode, D):
    """The rotated rows equal the closed form bit for bit; the text rows are untouched (Hq != Hk, B = 2)."""
    from svgb200 import core

    B, Hq, Hk, S, txt = 2, 4, 2, 203, 29
    gen = torch.Generator(device=cuda).manual_seed(mode * 1000 + D)
    cos, sin = rw.census_tables(S - txt, D // 2 if mode == 2 else D, gen)
    q0 = torch.randint(-100, 101, (B, Hq, S, D), generator=gen, device=cuda).to(dtype)
    k0 = torch.randint(-100, 101, (B, Hk, S, D), generator=gen, device=cuda).to(dtype)
    q, k = q0.clone(), k0.clone()
    core.qk_rope_(q, k, cos, sin, txt, mode)
    lo, hi = (0, S - txt) if mode == 1 else (txt, S)
    for got, x, name in ((q, q0, "q"), (k, k0, "k")):
        want = x.clone()
        want[:, :, lo:hi] = rw.round_to(rw.rope(x[:, :, lo:hi], cos, sin, mode == 2), dtype)
        assert_bits(got, want, f"rope {name} mode {mode} D {D} {dtype}")


# ---- 4. fused qkv_prep forward -----------------------------------------------------------------------------------
def prep_inputs(seed, B, S, H, D, norm, dtype, cuda):
    """packed [B, S, 3*H*D] and the rstd of q and k's normalised rows (head rows; NORM_RMS_HIDDEN: hidden rows)."""
    packed = torch.empty(B, S, 3 * H * D, dtype=dtype, device=cuda)
    rstd = []
    for i in range(3):
        if norm == 3 and i < 2:
            x, r = build_x(seed * 3 + i, B * S, H * D, False, dtype, cuda)
        else:
            x, r = build_x(seed * 3 + i, B * S * H, D, norm == 2, dtype, cuda)
        packed[..., i * H * D:(i + 1) * H * D] = x.view(B, S, H * D)
        rstd.append(r)
        del x
    return packed, rstd


def prep_expect(x, rstd, H, D, norm, g, b, rope, cos, sin, lo, n, dtype, t0, t1):
    """Expected q or k output rows [B, H, t1 - t0, D] (float64 of dtype values) for input tokens [t0, t1)."""
    B = x.shape[0]
    xs = x[:, t0:t1]
    if norm == 3:
        rs = rstd.view(B, -1)[:, t0:t1].reshape(-1)
        o = rw.xhat(xs.reshape(-1, H * D), rs, False) * g.double()
        o = rw.round_to(o, dtype).double().view(B, t1 - t0, H, D)
    elif norm:
        rs = rstd.view(B, -1, H)[:, t0:t1].reshape(-1)
        o = rw.row_norm(xs.reshape(-1, D), rs, g, b if norm == 2 else None)
        o = rw.round_to(o, dtype).double().view(B, t1 - t0, H, D)
    else:
        o = xs.double().view(B, t1 - t0, H, D)
    o = o.transpose(1, 2)
    if rope:
        a, e = max(t0, lo), min(t1, lo + n)
        if a < e:
            o = o.clone()
            o[:, :, a - t0:e - t0] = rw.round_to(rw.rope(o[:, :, a - t0:e - t0], cos[a - lo:e - lo], sin[a - lo:e - lo],
                                                         rope == 2), dtype).double()
    return o


def run_prep(cuda, B, S, H, D, norm, rope, lo, n, dtype, seed, r0=0, tail=0):
    from svgb200 import core

    gen = torch.Generator(device=cuda).manual_seed(seed)
    packed, rstd = prep_inputs(seed, B, S, H, D, norm, dtype, cuda)
    qi, ki, vi = (packed[..., i * H * D:(i + 1) * H * D] for i in range(3))
    gw = H * D if norm == 3 else D
    gq, gk = (rw.gammas((gw,), gen).to(dtype) for _ in range(2)) if norm else (None, None)
    bq, bk = (rw.betas((D,), gen).to(dtype) for _ in range(2)) if norm == 2 else (None, None)
    cos, sin = rw.census_tables(n, D // 2 if rope == 2 else D, gen) if rope else (None, None)
    S_out = r0 + S + tail
    out = tuple(torch.full((B, H, S_out, D), float("nan"), dtype=dtype, device=cuda) for _ in range(3))
    core.qkv_prep(qi, ki, vi, H, out=out, out_row0=r0, out_rows=S_out, norm=norm, gamma_q=gq, gamma_k=gk, beta_q=bq,
                  beta_k=bk, eps=1e-6, rope=rope, cos=cos, sin=sin, rope_lo=lo, rope_n=n if rope else None)
    what = f"qkv_prep B {B} S {S} H {H} D {D} norm {norm} rope {rope} lo {lo} {dtype}"
    nan = torch.full((B, H, 1, D), float("nan"), dtype=dtype, device=cuda)
    for i, (x, g, b) in enumerate(((qi, gq, bq), (ki, gk, bk), (vi, None, None))):
        o = out[i]
        assert_bits(o[:, :, :r0], nan.expand(B, H, r0, D), f"{what}: rows before out_row0 of output {i}")
        assert_bits(o[:, :, r0 + S:], nan.expand(B, H, tail, D), f"{what}: rows after the written range of output {i}")
        step = max(1, CHUNK // (B * H * D))
        for t0 in range(0, S, step):
            t1 = min(S, t0 + step)
            want = prep_expect(x, rstd[i], H, D, norm if i < 2 else 0, g, b, rope if i < 2 else 0, cos, sin, lo, n,
                               dtype, t0, t1)
            assert_bits(o[:, :, r0 + t0:r0 + t1], want.to(dtype), f"{what}: output {i}, tokens from {t0}")


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("D", rw.HEAD_DIMS)
@pytest.mark.parametrize("rope, text_first", [(0, False), (1, False), (1, True), (2, True)])
@pytest.mark.parametrize("norm", [0, 1, 2, 3])
def test_qkv_prep_census(cuda, norm, rope, text_first, D, dtype):
    """Norm x RoPE x D x dtype on packed strided inputs, into rows [37, 37 + S) of NaN-filled outputs of 37 + S + 11
    rows: the rows outside stay NaN."""
    B, S, H, txt = 2, 157, 3, 21
    lo = txt if text_first else 0
    run_prep(cuda, B, S, H, D, norm, rope, lo, S - txt, dtype, seed=norm * 100 + rope * 10 + D + text_first, r0=37,
             tail=11)


def test_qkv_prep_census_hunyuan720p(cuda):
    """HunyuanVideo single-stream block: S = 119 056, H = 24, D = 128, per-head RMS, RoPE on all but the last 256."""
    S = rw.HY_S
    run_prep(cuda, 1, S, rw.HY_H, rw.HY_D, 1, 1, 0, S - rw.HY_TXT, torch.bfloat16, seed=11)


def test_qkv_prep_census_wan720p(cuda):
    """Wan 720p: S = 75 600, H = 40, D = 128, RMS over the full hidden row of 5120, complex RoPE on every token."""
    S = rw.WAN_S
    run_prep(cuda, 1, S, rw.WAN_H, rw.WAN_D, 3, 2, 0, S, torch.bfloat16, seed=12)
