"""Exact census of the row-wise forward kernels.  TEST INFRASTRUCTURE ONLY.

The Wan block glue (csrc/glue.cu), the standalone QK norms, the in-place RoPE and the fused qkv_prep forward
(csrc/prep.cu) are fed inputs on which every quantity of the exact computation is representable, so the expected
output is a closed form that does not depend on summation order, on FMA contraction, or on the approximate rsqrtf.

  rows    x = m + d per normalised row (a glue row of N, a head row of D, or a full hidden row of H*D).  d is built
          from blocks of 8 integers in [-6, 6] with sum 0 and sum of squares 128 (a multiset from `BLOCKS`, permuted
          per block), scaled by 2^j.  So sum(d) = 0 and the variance (RMS rows: m = 0, the mean square) is exactly
          16 * 4^j: rstd = 2^-(2+j), x^ = d * rstd is a multiple of 1/4 in [-3/2, 3/2], whatever m and j are.  m and j
          vary per row (m in [-MMAX, MMAX], j in JS), so rows that get mixed up give different outputs.  |x| <= 112:
          an integer exact in bf16, fp16 and fp32; every sum of a row stays below 2^24.
  factors gamma / LayerNorm weight and gate: multiples of 1/4 in [-2, 2]; 1 + scale: multiples of 1/4 in [1/4, 2].
          beta (row norms): odd multiples of 1/32 in (-2, 2), so x^ g + b is never 0 and never a cancelled sum;
          LayerNorm bias, shift: multiples of 1/16 in [-2, 2]; residual: multiples of 1/8 in [-16, 16].
  rope    tables from {-1, -1/2, 0, 1/2, 1}: every product is exact.

Glue (IEEE sqrtf and division, eps = 1e-6 absorbed since var >= 64): every intermediate is exact in fp32, so the
output is the exact value rounded once to the output dtype.  Row norms and the per-head norms of qkv_prep (rsqrtf,
LayerNorm's fixed eps 1e-5): the exact value is representable in the 16-bit dtype, and the CPU test checks element by
element that it sits further from a rounding boundary than the approximate path can move it (`norm_margin_ok`).  The
fused prep rounds the norm output to 16 bits before it rotates; the closed form does the same.

Large inputs are a hash of (seed, row, block) computed with integer torch ops, so they build on any device, in row
chunks, with the same values on the CPU and the GPU.  Expected values are computed in float64 and rounded once.
"""
from __future__ import annotations

import itertools
import math

import torch

GLUE_THREADS, GLUE_MAX_VEC, SMS = 256, 4, 148
GLUE_GRID = SMS * 8                 # glue CTAs: min(rows, GLUE_GRID), each walks rows GLUE_GRID apart
GLUE_MAX_N = GLUE_THREADS * GLUE_MAX_VEC * 8
NORM_THREADS, NORM_UNROLL, NORM_GRID = 256, 4, SMS * 32   # row_norm_kernel: kThreads, kUnrollRows, grid cap
NORM_NS = (32, 64, 128, 256)
HEAD_DIMS = (64, 128, 256)
GLUE_EPS = 1e-6
LN_EPS = 1e-5                       # the standalone / per-head LayerNorm's fixed eps
MMAX = 64
JS = (1, 2, 3)                      # d = block * 2^j: var = 16 * 4^j in {64, 256, 1024}
XMAX = MMAX + 6 * 2 ** max(JS)      # 112
# error bound of the norm paths relative to |x^ g| + |b|: rsqrt.approx (< 2^-22.9), LayerNorm's eps at var >= 64
# (< 2^-23.6) and three fp32 roundings (2^-24 each) add to < 2^-21.3; twice that and more:
ERR_REL = 2.0 ** -20
_P = 2147483647                     # 2^31 - 1: hash arithmetic stays inside int64 on every device

DT = {"bf16": torch.bfloat16, "fp16": torch.float16, "fp32": torch.float32}


def _blocks():
    """Every multiset of 8 integers in [-6, 6] with sum 0 and sum of squares 128, as rows of a [n, 8] table."""
    out = [c for c in itertools.combinations_with_replacement(range(-6, 7), 8)
           if sum(c) == 0 and sum(v * v for v in c) == 128]
    return torch.tensor(out, dtype=torch.float32)


BLOCKS = _blocks()
PERMS = torch.tensor(list(itertools.permutations(range(8))), dtype=torch.int64)  # all 40320


def _hash(*vals):
    """A deterministic int64 hash in [0, 2^31 - 1) of int64 tensors / ints, equal on every device."""
    h = 0
    for v in vals:
        h = (h + v) % _P * 48271 % _P
        h = (h * 16807 + 12345) % _P
    return h


def _rows(rows, row0, device, idx):
    """The int64 row indices [row0, row0 + rows), or idx (any int64 tensor of row indices) when given."""
    if idx is not None:
        return idx.to(device=device, dtype=torch.int64)
    return torch.arange(row0, row0 + rows, dtype=torch.int64, device=device)


def row_params(seed, rows, row0=0, device="cpu", *, js=JS, idx=None):
    """(m, j) of rows [row0, row0 + rows) (or of the rows idx): int64 tensors, j drawn from js."""
    h = _hash(_rows(rows, row0, device, idx), seed + 7)
    return (h >> 4) % (2 * MMAX + 1) - MMAX, torch.tensor(js, device=device)[(h >> 12) % len(js)]


def block_hash(seed, r, nb):
    """The hash h [n, nb], the BLOCKS index [n, nb] and the permutation [n, nb, 8] of each 8-block of rows r."""
    dev = r.device
    h = _hash(r[:, None], torch.arange(nb, dtype=torch.int64, device=dev)[None, :], seed)
    return h, (h >> 3) % BLOCKS.shape[0], PERMS.to(dev)[_hash(h, 3) % PERMS.shape[0]]


def row_x(seed, rows, N, *, centred, row0=0, device="cpu", js=JS, idx=None):
    """x [rows, N] float32 of integers (rows row0..., or the rows idx) and rstd [rows] float64, exact: see the module
    docstring.  js: the exponents j a row may draw (LayerNorm's backward census keeps to var >= 256)."""
    assert N % 8 == 0
    r = _rows(rows, row0, device, idx)
    _, bi, perm = block_hash(seed, r, N // 8)
    d = torch.gather(BLOCKS.to(device)[bi], 2, perm)                       # [rows, nb, 8]
    m, j = row_params(seed, rows, row0, device, js=js, idx=idx)
    if not centred:
        m = torch.zeros_like(m)
    # powers of two from exact tables: torch.pow on CUDA may be an ulp off
    scale = torch.tensor([2.0 ** v for v in range(max(js) + 1)], device=device)[j]
    rstd = torch.tensor([2.0 ** -(2 + v) for v in range(max(js) + 1)], dtype=torch.float64, device=device)[j]
    return d.reshape(r.shape[0], N) * scale[:, None] + m.float()[:, None], rstd


def multiples(shape, step, lo, hi, gen, odd=False):
    """Random multiples of `step` in [lo, hi] (odd multiples only with odd=True), float32, on gen's device."""
    k = torch.randint(int(round(lo / step)), int(round(hi / step)) + 1, shape, generator=gen, device=gen.device)
    if odd:
        k = k - (k % 2 == 0).long() * torch.where(k > 0, 1, -1)
    return (k * step).float()


def gammas(shape, gen):
    return multiples(shape, 0.25, -2, 2, gen)


def betas(shape, gen):
    return multiples(shape, 1 / 32, -63 / 32, 63 / 32, gen, odd=True)


def scales(shape, gen):
    return multiples(shape, 0.25, -0.75, 1.0, gen)


def shifts(shape, gen):
    return multiples(shape, 1 / 16, -2, 2, gen)


def residuals(shape, gen):
    return multiples(shape, 1 / 8, -16, 16, gen)


def census_tables(n, width, gen):
    """cos / sin drawn per element from {-1, -1/2, 0, 1/2, 1}."""
    vals = torch.tensor([-1.0, -0.5, 0.0, 0.5, 1.0], device=gen.device)
    pick = lambda: vals[torch.randint(0, 5, (n, width), generator=gen, device=gen.device)]  # noqa: E731
    return pick(), pick()


# ---- closed forms (float64) --------------------------------------------------------------------------------------
def xhat(x, rstd, centred):
    x = x.double()
    # the integer row sum (below 2^53) over N by one correctly rounded division: exact, unlike a multiply by 1/N
    if centred:
        s = x.sum(-1, keepdim=True)
        mean = s / torch.full_like(s, x.shape[-1])
    else:
        mean = 0.0
    return (x - mean) * rstd[:, None]


def mod_slice(v, rows, r0, r1):
    """Modulation [nb, N] (or [nb, 1, N], [N]) -> float64 [r1 - r0, N]: the vector of each row in [r0, r1) of `rows`
    rows, batch row // (rows // nb)."""
    v = v.reshape(-1, v.shape[-1]).double()
    if v.shape[0] == 1:
        return v.expand(r1 - r0, -1)
    return v[torch.arange(r0, r1, device=v.device) // (rows // v.shape[0])]


# x, rstd: rows of row_x; w, b: [N]; scale, shift, gate: per row (mod_slice)
def glue_layernorm(x, rstd, w=None, b=None, scale=None, shift=None, centred=True):
    o = xhat(x, rstd, centred)
    if w is not None:
        o = o * w.double() + b.double()
    if scale is not None:
        o = o * (1 + scale) + shift
    return o


def glue_rmsnorm(x, rstd, w):
    return xhat(x, rstd, False) * w.double()


def glue_modulate(x, scale, shift):
    return x.double() * (1 + scale) + shift


def glue_gate_residual(res, x, gate):
    return res.double() + x.double() * gate


def row_norm(x, rstd, g, b=None):
    """rms_apply / ln_apply closed form on [rows, n]; b selects LayerNorm."""
    o = xhat(x, rstd, b is not None) * g.double()
    return o if b is None else o + b.double()


def rope(x, c, s, complex_):
    """The forward rotation on [..., n, D] (float64): interleaved pairs with per-element tables [n, D] or complex
    pairs with tables [n, D/2]."""
    x, c, s = x.double(), c.double(), s.double()
    a, b = x[..., 0::2], x[..., 1::2]
    if complex_:
        return torch.stack([a * c - b * s, b * c + a * s], -1).flatten(-2)
    return torch.stack([a * c[..., 0::2] - b * s[..., 0::2], b * c[..., 1::2] + a * s[..., 1::2]], -1).flatten(-2)


def round_to(v, dtype):
    """The exact float64 value v (exact in fp32) rounded once to dtype."""
    return v.float().to(dtype)


# ---- premises ----------------------------------------------------------------------------------------------------
def exact_in(t, dtype):
    t = t.double()
    return bool(torch.equal(t.to(dtype).double(), t))


def norm_margin_ok(v, scale, dtype):
    """Element-wise: v is representable in the 16-bit dtype, and it lies further than ERR_REL * scale (scale = |x^ g|
    + |b|, the size of the terms the approximate path rounds) from the midpoints to its neighbours, so rsqrtf a few
    ulps off, an unabsorbed eps and the fp32 roundings of x^ g + b cannot move its rounding.  Any per-element scale
    works: the backward census (oracle/rowwise_bwd.py) passes r (|u| + |x^ m0|).  Returns (ok, the smallest ratio of the
    margin to the error bound)."""
    v = v.double()
    if not exact_in(v, dtype):
        return False, 0.0
    p = {torch.bfloat16: 8, torch.float16: 11}[dtype]
    mant, e = torch.frexp(v)
    ulp = torch.pow(2.0, (e - p).double())
    below = torch.where(mant.abs() == 0.5, ulp / 2, ulp)     # the spacing below a power of two is half
    gap = torch.where(v == 0, torch.full_like(v, 2.0 ** -133), below / 2)
    err = ERR_REL * scale.double()
    zero_ok = (v != 0) | (err == 0)                           # an exact 0 stays 0 only if nothing is added to it
    ratio = torch.where(err > 0, gap / err.clamp_min(1e-300), torch.full_like(v, math.inf))
    return bool(zero_ok.all() and (ratio > 1).all()), float(ratio.min())


def row_sums_ok(x, centred):
    """The kernels' row sums (sum x, sum (x - mean)^2, sum x^2) are integers below 2^24, so exact in any order."""
    x = x.double()
    lim = 2.0 ** 24
    ok = bool(x.abs().sum(-1).max() < lim) and bool((x * x).sum(-1).max() < lim or centred)
    if centred:
        c = x - x.mean(-1, keepdim=True)
        ok = ok and bool((c * c).sum(-1).max() < lim)
    return ok and exact_in(x, torch.bfloat16)


def fp32_exact(*ts):
    """Every intermediate of the glue is exact in fp32: then contraction or not, the result is the exact value."""
    return all(exact_in(t, torch.float32) for t in ts)


# ---- grid geometry -----------------------------------------------------------------------------------------------
def glue_grid(rows):
    return min(rows, GLUE_GRID)


def norm_blocks(m, n):
    rpb = NORM_THREADS // (n // 8)
    return max(1, min(NORM_GRID, -(-m // (rpb * NORM_UNROLL))))


def norm_threshold(n):
    """Rows above which row_norm_kernel's grid-stride loop makes a second pass."""
    return NORM_GRID * (NORM_THREADS // (n // 8)) * NORM_UNROLL


def norm_passes(m, n):
    rpb = NORM_THREADS // (n // 8)
    return -(-m // (norm_blocks(m, n) * rpb * NORM_UNROLL))


# ---- the GPU test's cases ----------------------------------------------------------------------------------------
GLUE_NS = (8, 264, 2048, 2056, 5120, 8192)
GLUE_ROWS = (1, 1183, 1184, 1185, 2 * 1184 + 3)
# modulation batches per row count: one vector, per batch (rows_per_batch not a multiple of the grid) or per row
GLUE_MOD = {1: 1, 1183: 7, 1184: 2, 1185: 3, 2 * 1184 + 3: 2 * 1184 + 3}
GLUE_DT_N, GLUE_DT_B, GLUE_DT_S = 2056, 3, 395     # the dtype sweep: rows 1185, CTA walks cross a batch boundary
WAN_ROWS, WAN_N = 75600, 5120


def glue_dtype_cases():
    """(op, x, y, w or res) of the dtype sweep: every dtype the wrappers pass, so all ten instantiations run."""
    dts = ("bf16", "fp16", "fp32")
    cases = [("layernorm", x, y, w) for x in dts for y in dts for w in (None,) + dts]
    cases += [("rmsnorm", x, y, w) for x in dts for y in dts for w in dts]
    cases += [("modulate", x, y, None) for x in dts for y in dts]
    cases += [("gate", x, y, r) for x in dts for y in dts for r in dts]
    return cases


def glue_instantiation(op, x, res):
    """The glue_rows_kernel<OP, F32, RF32> a case runs."""
    return (op, x == "fp32", op == "gate" and res == "fp32")


def norm_rows(n):
    """Row counts of the standalone norm sweep: just below and just above the multi-pass threshold (neither a
    multiple of RPB * kUnrollRows)."""
    t = norm_threshold(n)
    return (t - 1, t + 1 + NORM_THREADS // (n // 8))


HY_NORM_ROWS, HY_NORM_N = 2857344, 128
HY_S, HY_H, HY_D, HY_TXT = 119056, 24, 128, 256
WAN_S, WAN_H, WAN_D = 75600, 40, 128
