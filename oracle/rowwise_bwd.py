"""Exact census of the pre-attention backward (csrc/prep.cu, the "backward" section).  TEST INFRASTRUCTURE ONLY.

The norm backwards `rms_bwd` / `ln_bwd` (in row_norm_bwd_kernel and, for the per-head norms, in qkv_prep_bwd_kernel),
the two-pass NORM_RMS_HIDDEN backward (the (r, mean(u x^)) stats pass, then hidden_rms_bwd_kernel over token splits)
and the parameter-gradient reductions (cta_column_sum, per-split partials, column_sum_kernel) are fed inputs whose
exact gradients are short closed forms.

  rows    x: the forward census's rows (oracle/rowwise.py row_x): per 8-block sum(x^) = 0 and sum(x^^2) = 8, so over
          any row of whole blocks (a head row of D, or a hidden row of H*D) mean(x^^2) = 1, r = rstd = 2^-(2+j) exact
          and x^ a multiple of 1/4.  LayerNorm rows keep to j in LN_JS (var 256 / 1024), where the fixed eps 1e-5 is
          absorbed in fp32 (half an ulp of 64 is only 3.8e-6); RMS rows with eps 1e-6 use every j.
  u       u = gamma * dn is chosen per row as  u = m0 x^ + c + e:
            m0  per row, from M0S (nonzero short dyadics);
            c   constant on each 8-block.  RMS rows: an odd multiple of 1/8.  LayerNorm rows: mu +- delta on the two
                blocks of a pair, mu (per row) and delta odd multiples of 1/16, so mean(c) = mu != 0 and c - mu != 0;
            e   a small integer vector orthogonal to 1 and to the block's d (E_VECS, permuted with the block).
          Then mean(u x^) = m0 and mean(u) = mean(c) exactly, and
            RMS:        dx = r (u - x^ mean(u x^))            = r (c + e)
            LayerNorm:  dx = r (u - mean(u) - x^ mean(u x^))  = r (c + e - mu)
          both odd multiples of r/16 or r/8, so never 0, and short enough to be exact in bf16 and fp16.  The kernel
          still has to cancel the m0 x^ part of u against its own x^ * m, so a wrong m, r or x^ shows up.
  gamma   from GAMMAS (nonzero powers of two), so dn = u / gamma is exact and short in 16 bits.
  rope    quarter-turn tables (c, s) in QUARTER (never the identity), equal on both elements of an interleaved pair:
          the rotation is orthogonal, so the census feeds dy = RoPE(dn) and the kernel's transpose returns dn exactly.
  dgamma  sum of dn x^, dbeta sum of dn: fp32 sums of multiples of Q_DG (Q_DB), exact in any order while the sum of
          |terms| stays below 2^24 quanta.  Production-size cases keep dn = 0 on all but a hashed sparse subset of
          rows (one in 2^k) plus every row at a boundary of the grids (`walk_ends`, `split_ends`), text / RoPE and batch
          boundaries.  Rows with dn = 0 give dx = 0 (of either sign).

Exactness of the kernels' arithmetic: every sum the kernels form (sum x^2, sum u x, sum u, the dgamma / dbeta
partials) is a sum of short dyadics below 2^24 quanta, so exact in any order.  The hidden path (IEEE sqrtf and
division) then computes r and m = (r * sum(u x)) / (H*D) exactly.  The per-head and standalone paths compute r with
rsqrtf: dx stays exact if rsqrtf is a few ulps off (`rw.norm_margin_ok` with the error scale r (|u| + |x^ m0|),
checked on the CPU for every element), and x^ = x * r, hence dgamma, is exact when rsqrt.approx.f32 returns 2^-k for
4^k exactly; tests/test_rowwise_bwd_census_gpu.py pins that premise on the census variances.

Inputs are hashes of (seed, row, block) as in oracle/rowwise.py, so they build on any device, in chunks or on any
subset of rows, with the same values.
"""
from __future__ import annotations

import itertools

import torch

from oracle import rowwise as rw
from oracle.rowwise import _hash

THREADS, UNROLL, HIDDEN_THREADS = 256, 4, 128     # kThreads, kUnrollRows, kHiddenThreads
BWD_CTAS = 148 * 4                                # kBwdCtas: the persistent backward grids
RMS_EPS, LN_EPS = 1e-6, rw.LN_EPS
LN_JS = (2, 3)
GAMMAS = (-2.0, -1.0, -0.5, 0.5, 1.0, 2.0)
M0S = (-1.0, -0.5, -0.25, 0.25, 0.5, 1.0)
ODD8 = tuple(k / 8 for k in (-7, -5, -3, -1, 1, 3, 5, 7))
ODD16 = tuple(k / 16 for k in (-7, -5, -3, -1, 1, 3, 5, 7))
QUARTER = ((0.0, 1.0), (-1.0, 0.0), (0.0, -1.0))   # (cos, sin): a quarter, half and three-quarter turn
Q_DB = 2.0 ** -5                                  # dn: u a multiple of 1/16 over |gamma| <= 2
Q_DG = 2.0 ** -7                                  # dn x^: times a multiple of 1/4
SUM_LIMIT = 2.0 ** 24
DENSE = 4096                                      # hashed live units per column sum, about
NE = 8                                            # e vectors per block


def _e_vecs():
    """[len(BLOCKS), NE, 8]: for every block, NE vectors from {-1, 0, 1}^8 orthogonal to 1 and to the block."""
    cand = torch.tensor(list(itertools.product((-1, 0, 1), repeat=8)), dtype=torch.float32)
    cand = cand[(cand.sum(1) == 0) & (cand.abs().sum(1) > 0)]
    out = []
    for b in rw.BLOCKS:
        ok = cand[cand @ b == 0]
        out.append(ok[torch.linspace(0, ok.shape[0] - 1, NE).round().long()])
    return torch.stack(out)


E_VECS = _e_vecs()


def _tab(vals, device):
    return torch.tensor(vals, dtype=torch.float64, device=device)


def gamma(seed, N, device="cpu"):
    """Norm weight [N] (float64) from GAMMAS, a hash of the column."""
    return _tab(GAMMAS, device)[_hash(torch.arange(N, device=device), seed + 17) % len(GAMMAS)]


def rows(seed, idx, N, g, *, layer, live=None):
    """The census on rows idx (int64 [n]) of N-wide normalised rows with weight g [N]: a dict of x [n, N] float32
    (integers), and in float64 rstd [n], xh, u, m0 [n], dn = u / g and the exact dx, both 0 on rows where live [n] is
    False."""
    dev = idx.device
    n, nb = idx.shape[0], N // 8
    x, rstd = rw.row_x(seed, 0, N, centred=layer, device=dev, js=LN_JS if layer else rw.JS, idx=idx)
    h, bi, perm = rw.block_hash(seed, idx, nb)
    e = torch.gather(E_VECS.to(dev)[bi, _hash(h, 5) % NE], 2, perm).double()          # [n, nb, 8]
    hr = _hash(idx, seed + 11)
    m0 = _tab(M0S, dev)[hr % len(M0S)]
    if layer:
        assert nb % 2 == 0
        mu = _tab(ODD16, dev)[(hr >> 4) % len(ODD16)]
        delta = _tab(ODD16, dev)[_hash(h[:, 0::2], 7) % len(ODD16)]                    # one per pair of blocks
        cc = torch.stack([delta, -delta], -1).flatten(1)                                # c - mu
        c = mu[:, None] + cc
    else:
        c = cc = _tab(ODD8, dev)[_hash(h, 7) % len(ODD8)]
    xh = rw.xhat(x, rstd, layer)
    u = m0[:, None] * xh + (c[..., None] + e).reshape(n, N)
    dx = rstd[:, None] * (cc[..., None] + e).reshape(n, N)
    if live is not None:
        keep = live[:, None]
        u, dx = torch.where(keep, u, 0.0), torch.where(keep, dx, 0.0)
    return dict(x=x, rstd=rstd, xh=xh, u=u, m0=m0, dn=u / g.double(), dx=dx)


def quarter_tables(seed, n, D, rope, device="cpu"):
    """float32 cos / sin of RoPE table rows [0, n): a quarter turn from QUARTER per pair; rope 1: [n, D] with both
    elements of a pair equal, rope 2 (complex): [n, D/2]."""
    q = _hash(torch.arange(n, device=device)[:, None], torch.arange(D // 2, device=device)[None, :], seed + 23)
    q = q % len(QUARTER)
    c, s = (_tab([t[k] for t in QUARTER], device)[q] for k in (0, 1))
    if rope == 1:
        c, s = c.repeat_interleave(2, -1), s.repeat_interleave(2, -1)
    return c.float(), s.float()


# ---- which rows carry a gradient -----------------------------------------------------------------------------------
def walk_ends(units, group, grid):
    """First and last unit (row or token) of every CTA of a persistent walk: CTA b takes the groups of `group` units
    b, b + grid, ... (row_norm_bwd_kernel, qkv_prep_bwd_kernel)."""
    first = torch.arange(grid, dtype=torch.int64) * group
    first = first[first < units]
    last_group = first + (units - 1 - first) // (grid * group) * (grid * group)
    return torch.cat([first, torch.clamp(last_group + group - 1, max=units - 1)])


def split_ends(T, splits):
    """First and last token of every non-empty split of hidden_rms_bwd_kernel (ceil(T / splits) tokens each)."""
    per = -(-T // splits)
    lo = torch.arange(splits, dtype=torch.int64) * per
    lo = lo[lo < T]
    return torch.cat([lo, torch.clamp(lo + per, max=T) - 1])


def sparsity(units):
    """k such that about DENSE of `units` rows feeding one column sum are hashed live (one in 2^k)."""
    k = 0
    while units > DENSE << k:
        k += 1
    return k


def live(seed, idx, k, forced):
    """Rows idx live: one in 2^k by hash, and every row in forced (int64 indices)."""
    hashed = _hash(idx, seed + 19) % (1 << k) == 0
    return hashed | torch.isin(idx, forced.to(idx.device))


def prep_forced(B, S, H, D, norm, lo, n):
    """Tokens (b * S + t) of a qkv_prep_bwd case that always carry a gradient: the ends of every CTA walk in every
    batch, the ends of every hidden split, and the tokens on both sides of the RoPE range."""
    ends = walk_ends(S, rpb(D), prep_bwd_blocks(B, S, D))
    edge = torch.tensor([t for t in (lo - 1, lo, lo + n - 1, lo + n) if n and 0 <= t < S], dtype=torch.int64)
    per_b = torch.cat([ends, edge])
    forced = torch.cat([b * S + per_b for b in range(B)])
    if norm == 3:
        forced = torch.cat([forced, split_ends(B * S, hidden_splits(B, S, H, D))])
    return forced.unique()


# ---- grid geometry (prep.cu host side) -----------------------------------------------------------------------------
def rpb(n):
    return THREADS // (n // 8)


def row_blocks(m, n, cap=BWD_CTAS):
    return max(1, min(cap, -(-m // (rpb(n) * UNROLL))))


def row_passes(m, n):
    return -(-m // (row_blocks(m, n) * rpb(n) * UNROLL))


def row_threshold(n):
    """Rows above which row_norm_bwd_kernel's walk takes a second pass."""
    return BWD_CTAS * rpb(n) * UNROLL


def prep_bwd_blocks(B, S, D):
    return min(-(-S // rpb(D)), max(1, BWD_CTAS // B))


def prep_passes(B, S, D):
    return -(-S // (prep_bwd_blocks(B, S, D) * rpb(D)))


def prep_threshold(B, D):
    """Tokens above which qkv_prep_bwd_kernel's walk takes a second pass."""
    return rpb(D) * (BWD_CTAS // B)


def hidden_cols(H, D):
    return -(-(H * (D // 8)) // HIDDEN_THREADS)


def hidden_splits(B, S, H, D):
    return max(1, min(BWD_CTAS // hidden_cols(H, D), B * S))


def row_forced(m, n):
    """Rows of a standalone norm case that always carry a gradient: the ends of every CTA walk."""
    return walk_ends(m, rpb(n), row_blocks(m, n))


# ---- the backward from first principles, and its mutants (float64) -------------------------------------------------
def norm_bwd(x, dn, g, *, layer, div=None, div_u=None, drop_ux=False, drop_u=False, rstd=None):
    """dx of the RMS / LayerNorm backward on rows x [n, N] for the output gradient dn, computed the kernels' way from
    x alone (r from the row's variance; the census's eps is absorbed, which the CPU test checks).  Mutants: div /
    div_u replace N in mean(u x^) / mean(u); drop_ux / drop_u drop the x^ mean(u x^) / mean(u) term; rstd [n]
    replaces r (stats read for another row)."""
    x = x.double()
    N = x.shape[-1]
    xc = x - x.mean(-1, keepdim=True) if layer else x
    r = (xc * xc).mean(-1, keepdim=True).rsqrt() if rstd is None else rstd.double()[:, None]
    xh = xc * r
    u = dn.double() * g.double()
    m = (u * xh).sum(-1, keepdim=True) / (div or N)
    d = u - (0 if drop_ux else xh * m)
    if layer and not drop_u:
        d = d - u.sum(-1, keepdim=True) / (div_u or N)
    return r * d


def margin_scale(c):
    """The error scale of dx on the rsqrtf paths, per element: r (|u| + |x^ m0|) of a census dict."""
    return c["rstd"][:, None] * (c["u"].abs() + (c["xh"] * c["m0"][:, None]).abs())


def rotate(dn, c, s, rope):
    """dy = RoPE(dn) on [..., n, D] with tables of n rows (float64): what the forward's rotation makes of dn."""
    return rw.rope(dn, c, s, rope == 2)


def row_live(seed, idx, m, n):
    """Live rows idx of a standalone case of m rows of n."""
    return live(seed, idx, sparsity(m), row_forced(m, n))


def prep_live(seed, B, S, H, D, norm, lo, n):
    """Live tokens (b * S + t, all B * S of them) of a qkv_prep_bwd case; a live token is live in every head."""
    tok = torch.arange(B * S, dtype=torch.int64)
    return live(seed, tok, sparsity(B * S * (1 if norm == 3 else H)), prep_forced(B, S, H, D, norm, lo, n))


# ---- the GPU test's cases ------------------------------------------------------------------------------------------
def row_norm_rows(n):
    """m = 1, m below RPB (one CTA partly dead), and just below / above the second-pass threshold (neither a multiple
    of RPB * kUnrollRows)."""
    t = row_threshold(n)
    return (1, rpb(n) - 3, t - 1, t + 1 + rpb(n))


# (layer, n, dtype, m, seed)
ROW_CASES = [(layer, n, dt, m, 10 * n + i + 100 * layer + 1000 * (dt == "fp16"))
             for layer in (False, True) for n in rw.NORM_NS for dt in ("bf16", "fp16")
             for i, m in enumerate(row_norm_rows(n))]
ROW_CASES_HY = [(layer, rw.HY_NORM_N, "bf16", rw.HY_NORM_ROWS, 7 + layer) for layer in (False, True)]


def prep_rows(B, D):
    """S_in just below and just above the persistent walk's second-pass threshold, neither a multiple of RPB."""
    t = prep_threshold(B, D)
    return (t - 3, t + rpb(D) + 5)


# (B, S, H, D, norm, rope, lo, n, dtype, seed, r0, tail); n = 0 without RoPE
PREP_CASES = [(2, 157, 3, D, norm, rope, 21 if tf else 0, 136, dt, norm * 100 + rope * 10 + D + tf, 37, 11)
              for norm in (1, 2) for rope, tf in ((0, 0), (1, 0), (1, 1), (2, 1)) for D in rw.HEAD_DIMS
              for dt in ("bf16", "fp16")]
PREP_CASES = [c[:7] + ((c[7] if c[5] else 0),) + c[8:] for c in PREP_CASES]
PREP_CASES_THRESHOLD = [(2, S, 2, D, norm, 1, 13, S - 40, ("bf16", "fp16")[i], 1000 + D + 7 * norm + i, 5, 3)
                        for norm in (1, 2) for D in rw.HEAD_DIMS for i, S in enumerate(prep_rows(2, D))]
HIDDEN_CASES = [  # NORM_RMS_HIDDEN: (cols, splits, tokens per split) in the comments
    (2, 200, 5, 128, 3, 2, 0, 200, "bf16", 31, 7, 2),     # 80 live threads of 128; 400 splits of one token
    (2, 1001, 5, 128, 3, 1, 17, 981, "fp16", 32, 7, 2),   # 592 splits of 4: split 250 crosses the batch boundary
    (2, 500, 20, 128, 3, 2, 0, 500, "fp16", 33, 0, 0),    # 3 column blocks (320 live threads); 197 splits of 6
    (1, 300, 13, 64, 3, 0, 0, 0, "bf16", 34, 3, 1),       # D = 64: 104 live threads; 300 splits of one token
    (2, 334, 6, 256, 3, 1, 0, 331, "bf16", 35, 1, 4),     # D = 256: 2 column blocks; 296 splits of 3, one crossing
]
PREP_CASES_FULL = [
    (1, rw.WAN_S, rw.WAN_H, rw.WAN_D, 3, 2, 0, rw.WAN_S, "bf16", 21, 0, 0),                  # Wan 2.1 720p
    (1, rw.HY_S, rw.HY_H, rw.HY_D, 1, 1, 0, rw.HY_S - rw.HY_TXT, "bf16", 22, 0, 0),         # HunyuanVideo 720p
]
# the autograd wiring tests' censuses: (B, S, H, D, norm, rope, lo, n, dtype, seed)
AUTOGRAD_PREP_CASES = [
    (2, 150, 3, 64, 2, 1, 19, 131, "fp16", 41),           # core.qkv_prep, LayerNorm, RoPE text first
    (1, 203, 40, 128, 3, 2, 0, 203, "bf16", 42),          # prep.wan_qkv
    (2, 301, 3, 128, 1, 1, 0, 301, "bf16", 43),           # HunyuanVideo double block: video stream
    (2, 37, 3, 128, 1, 0, 0, 0, "bf16", 44),              #                           prompt stream
]
AUTOGRAD_ROW_CASES = [(False, 64, "bf16", 42, 31), (True, 64, "bf16", 42, 32)]   # (layer, n, dtype, m, seed)
