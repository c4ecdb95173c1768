"""Closed form of sample_mse (svgb_sample_mse, csrc/sample_mse.cu).  TEST INFRASTRUCTURE ONLY.

The inputs make every row's softmax a closed form, so the two MSEs per head are known exactly from the oracle's
profiling masks (oracle.attention.profiling_mask_rows / profiling_mask_rows_cog), never from the engine.

Key census (hot=False): q = 0, so every allowed key gets p = 1 and a row's output under pass X (full, spatial,
temporal) is cnt_X / n_X: n_X the keys the row sees, cnt_X[d] those of them with code d.  V is one-hot by a key code
of oracle/census.py, code_0(j) = j mod D or code_1(j) = (j div D) mod D (head h uses encoding h mod 2, on j shifted by
a per-head offset so that the heads differ).  code_1 is what makes an aligned 128-key chunk visible: with j mod D
alone, dropping one leaves the output unchanged.  A row that sees no key gives 0 (the kernel's convention; svgb200.h).

Per-row classes (hot=True): sampled position p gets q[p, c(p)] = HOT_Q, key j of class kcls(j) gets
k[j, kcls(j)] = HOT_K, every other entry of q and k is 0.  A hot score is HOT_Q * HOT_K = 2048, any other score 0.  The
kernel forms p = ex2(s * c - m * c) with m * c rounded to fp32 and s * c fused; 2048 is a power of two, so m * c is
exact and every hot key gets p = 1 exactly (127 * 16 = 2032 would leave a residual of up to 2^-16 in the exponent, a
1e-5 error common to every row).  For D in {64, 128} and c = log2(e) / sqrt(D) the hot level is 2048 c >= 261 in
log2 units, so a cold key next to a hot one gets ex2(-261) = 0 exactly, in a chunk and in the split merge.  A row's
output is the mean of V over its visible keys of its own class, or over all its visible keys when it sees none of
them.  make_case places each position's class keys where a mask can be off by one: at the edges of its spatial and
temporal bands, at frame and 128-key chunk boundaries, the first-frame sink, the text block and the last partial
chunk, a few keys per position.  One key kept or dropped then moves a small tier.

MSE_X = mean over rows r < n_rows and d < D of (out_X - out_full)^2, computed in fp64.

Rounding bound (bound()).  Everything above is exact in the kernel except:
  * the epilogue: o = cnt * fl(1 / l) in fp32, l an exact integer: relative error <= 2u (u = 2^-24);
  * the LSE of a split, fp32 ((m c + log2f(l)) * ln2): log2f within 1 ulp, two roundings;
  * the merge: w_s = __expf(lse_s - max) (ex2.approx on x * log2(e) rounded), then num / den over nsplit terms.
    A split below the row's top level (a cold split next to a hot one) gets w = 0 exactly, as does an empty split
    (lse = -inf).  A row whose top-level keys lie in one split gets w = __expf(0) = 1 there and 0 elsewhere: its
    output is the split's o, exact up to the epilogue.  Otherwise each weight carries a relative error eps_w, which
    moves out by at most eps_w * max_s |o_s - out| (spread), plus (2 nsplit + 2) u for num, den and the division;
  * the fp32 squares and sums: per term one subtraction and one square (2u), and a sum chain of at most
    ceil(16 * D / 256) + 5 + 8 + kCombineParts + 1 = 30 additions of nonnegative terms (thread, warp shuffle, warps,
    parts, division): 33u relative overall; bound() uses 40u.
With per-element output errors e = E_X + E_full (E = rel * |out| + eps_w * spread),
    |MSE_kernel - MSE| <= (1 + 40u) / (n D) * sum (2 |out_X - out_full| e + e^2) + 40u * MSE.
The bound is computed per head and per mask from the closed form and the split partials of simulate() at the
call's split count.  On the suite's cases it is 4e-6 to 7e-4 of the MSE; it is largest where a row's top level spans
several splits, since the weights carry most of the error.

simulate() runs the sample_mse.cu flow in fp64 (gather, split partition, split partials, merge, row reduction) and can
apply one MUTATION, a plausible bug of that flow; the CPU suite shows that each one moves some GPU case by at least
10x the bound.  layout() mirrors smse_layout: the split count, chunks per split and the workspace bytes.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np
import torch

from oracle import attention as oa

CHUNK = 128
MAX_SPLITS = 32
COMBINE_PARTS = 8
HOT_Q, HOT_K = 128.0, 16.0
LAYOUTS = {"hy": 0, "wan": 1, "cog": 2}
U = 2.0 ** -24

MUTATIONS = (
    "split_end_plus1",     # split 0 runs one chunk past its range (a chunk counted twice)
    "split_end_minus1",    # the last non-empty split stops one chunk early (its last chunk dropped)
    "empty_split_nan",     # an empty split's partial read as NaN with lse 0
    "empty_split_lse0",    # an empty split's partial read as 0 with lse 0 instead of -inf
    "qindex_gathered",     # the mask sees the gathered row s * 128 + r instead of rows[r]
    "qindex_minus1",       # the mask sees rows[r] - 1
    "qindex_plus1",        # the mask sees rows[r] + 1
    "qindex_plus_P",       # the mask sees rows[r] + P
    "q_neighbour",         # q gathered from rows[r] + 1
    "padding_summed",      # padding rows n_rows .. 127 summed too
    "last_row_dropped",    # row n_rows - 1 left out of the sum
    "heads_swapped",       # heads 0 and 1 exchanged
    "divide_128D",         # the sum divided by 128 D instead of n_rows D
    "thres_rounded",       # band threshold rounded instead of floored
    "passes_swapped",      # spatial and temporal results exchanged
)


# --------------------------------------------------------------------------------------------
# smse_layout mirror
# --------------------------------------------------------------------------------------------
def _al(b):
    return (b + 255) // 256 * 256


def layout(BH, S, D, n_sms):
    """(nsplit, chunks per split, n_chunks, workspace bytes) as smse_layout computes them."""
    n_chunks = (S + CHUNK - 1) // CHUNK
    nsplit = max(1, min(n_sms // BH, MAX_SPLITS, n_chunks))
    cps = (n_chunks + nsplit - 1) // nsplit
    rows = nsplit * 128
    parts = [2 * BH * rows * D, 4 * rows, 256, 32 * nsplit, 8 * n_chunks, 8 * n_chunks, 12 * BH * rows * D,
             12 * BH * rows, 4 * 2 * BH * COMBINE_PARTS]
    return nsplit, cps, n_chunks, sum(_al(b) for b in parts)


def split_ranges(S, nsplit):
    """[(k0, k1)] key range of each split (smse_plan_kernel), empty ones included."""
    n_chunks = (S + CHUNK - 1) // CHUNK
    cps = (n_chunks + nsplit - 1) // nsplit
    out = []
    for s in range(nsplit):
        c0 = min(n_chunks, s * cps)
        c1 = min(n_chunks, c0 + cps)
        out.append((c0 * CHUNK, min(S, c1 * CHUNK)))
    return out


def thres_of(lay, P, rounded=False):
    x = (2 * P if lay == "wan" else 1.5 * P) / 128.0
    return int(math.floor(x + 0.5)) if rounded else int(x)


# --------------------------------------------------------------------------------------------
# cases
# --------------------------------------------------------------------------------------------
@dataclass
class Case:
    lay: str
    ctx: int
    F: int
    P: int
    D: int
    BH: int
    rows: torch.Tensor        # int64 [n_rows] (cpu), duplicates allowed
    hot: bool
    codes: torch.Tensor       # int64 [BH, S]: V[h, j, codes[h, j]] = 1
    kcls: torch.Tensor        # int64 [BH, S]: class of key j, -1 = none
    pos_cls: list             # per head {position: class} of the sampled positions (hot=True)

    @property
    def S(self):
        return self.ctx + self.F * self.P

    @property
    def n(self):
        return int(self.rows.numel())


def mask_rows(lay, name, positions, ctx, F, P, thres=None):
    """bool [len(positions), S] rows of the profiling mask `name` ("spatial" / "temporal"; "full" = all ones)."""
    S = ctx + F * P
    pos = torch.as_tensor(positions, dtype=torch.long).view(-1)
    if name == "full":
        return torch.ones(len(pos), S, dtype=torch.bool)
    if lay == "cog":
        return oa.profiling_mask_rows_cog(name, pos, ctx, F, P, thres=thres)
    return oa.profiling_mask_rows(name, pos, lay, ctx, F, P, thres=thres)


def _edges(m):
    """keys on both sides of every change of a bool row"""
    t = torch.nonzero(m[1:] != m[:-1]).view(-1) + 1
    return torch.cat([t - 1, t])


def make_case(lay, ctx, F, P, D, BH, rows, hot=True, seed=0, keys_per_pos=(1, 4)):
    """Case with per-head codes and (hot) per-head classes; head h depends on (seed, h) only, so the same head
    comes out the same in calls with different BH."""
    S = ctx + F * P
    rows = torch.as_tensor(rows, dtype=torch.long).view(-1)
    uniq = torch.unique(rows)
    j = torch.arange(S)
    V = F * P
    structural = torch.tensor([0, 1, P - 1, P, P + 1, ctx - 1, ctx, V - 1, V, S - 2, S - 1,
                               (S - 1) // CHUNK * CHUNK - 1, (S - 1) // CHUNK * CHUNK])
    cand = {}
    if hot:
        ms = mask_rows(lay, "spatial", uniq, ctx, F, P)
        mt = mask_rows(lay, "temporal", uniq, ctx, F, P)
        for i, p in enumerate(uniq.tolist()):
            near = torch.tensor([p - 1, p, p + 1, p // P * P, p // P * P + P - 1, p // CHUNK * CHUNK,
                                 p // CHUNK * CHUNK + CHUNK - 1])
            cand[p] = (_edges(ms[i]), _edges(mt[i]), torch.cat([structural, near]))
    codes = torch.empty(BH, S, dtype=torch.long)
    kcls = torch.full((BH, S), -1, dtype=torch.long)
    pos_cls = []
    for h in range(BH):
        g = torch.Generator().manual_seed(seed * 100003 + h)
        shift = int(torch.randint(0, S, (1,), generator=g))
        codes[h] = (j + shift) % D if h % 2 == 0 else ((j + shift) // D) % D
        pc = {}
        if hot:
            order = uniq[torch.randperm(len(uniq), generator=g)].tolist()
            c0 = int(torch.randint(0, D, (1,), generator=g))
            for i, p in enumerate(order):
                c = (c0 + i) % D
                pc[p] = c
                lo, hi = keys_per_pos
                want = int(torch.randint(lo, hi + 1, (1,), generator=g))
                es, et, st = cand[p]
                pools = [x[(x >= 0) & (x < S)] for x in (es, et, st)]
                placed = 0
                for t in range(4 * want):  # spatial edge, temporal edge, structural place, in turn
                    if placed >= want:
                        break
                    pool = pools[t % 3]
                    if len(pool) == 0:
                        continue
                    key = int(pool[int(torch.randint(0, len(pool), (1,), generator=g))])
                    if kcls[h, key] < 0:
                        kcls[h, key] = c
                        placed += 1
        pos_cls.append(pc)
    return Case(lay, ctx, F, P, D, BH, rows, hot, codes, kcls, pos_cls)


def tensors(case, dtype, device):
    """q, k, v [BH, S, D] of the case, exact in bf16 and fp16."""
    BH, S, D = case.BH, case.S, case.D
    q = torch.zeros(BH, S, D, dtype=dtype, device=device)
    k = torch.zeros(BH, S, D, dtype=dtype, device=device)
    v = torch.zeros(BH, S, D, dtype=dtype, device=device)
    hi = torch.arange(BH, device=device).view(BH, 1).expand(BH, S)
    ji = torch.arange(S, device=device).view(1, S).expand(BH, S)
    v[hi, ji, case.codes.to(device)] = 1
    if case.hot:
        for h in range(BH):
            for p, c in case.pos_cls[h].items():
                q[h, p, c] = HOT_Q
        kc = case.kcls.to(device)
        sel = kc >= 0
        k[hi[sel], ji[sel], kc[sel]] = HOT_K
    return q, k, v


# --------------------------------------------------------------------------------------------
# the sample_mse flow in fp64
# --------------------------------------------------------------------------------------------
def _split_partials(M, cls, kcls_h, E_h, ranges):
    """per split: (level [R] 1 hot / 0 cold / -1 empty, n [R], hist [R, D]) of rows with masks M [R, S] (bool) and
    classes cls [R] (-2 = none) over the key ranges"""
    res = []
    for k0, k1 in ranges:
        if k1 <= k0:
            R = M.shape[0]
            res.append((torch.full((R,), -1, dtype=torch.long, device=M.device),
                        torch.zeros(R, dtype=torch.float64, device=M.device),
                        torch.zeros(R, E_h.shape[1], dtype=torch.float64, device=M.device)))
            continue
        m = M[:, k0:k1]
        hot = m & (kcls_h[k0:k1].view(1, -1) == cls.view(-1, 1))
        nh = hot.sum(1).double()
        nv = m.sum(1).double()
        Ek = E_h[k0:k1]
        hh = hot.double() @ Ek
        hv = m.double() @ Ek
        lvl = torch.where(nh > 0, 1, torch.where(nv > 0, 0, -1))
        n = torch.where(nh > 0, nh, nv)
        hist = torch.where((nh > 0).view(-1, 1), hh, hv)
        res.append((lvl, n, hist))
    return res


def _merge(parts, mutation=None, empty_ids=()):
    """(out [R, D], top level [R], spread [R, D], n_top [R]) of the merged split partials"""
    lvl = torch.stack([p[0] for p in parts])       # [ns, R]
    n = torch.stack([p[1] for p in parts])         # [ns, R]
    hist = torch.stack([p[2] for p in parts])      # [ns, R, D]
    top = lvl.max(0).values
    w = ((lvl == top.view(1, -1)) & (top.view(1, -1) >= 0)).double()
    num = (w.unsqueeze(-1) * hist).sum(0)
    den = (w * n).sum(0)
    out = torch.where(den.view(-1, 1) > 0, num / den.clamp(min=1).view(-1, 1), torch.zeros_like(num))
    o_s = hist / n.clamp(min=1).unsqueeze(-1)
    spread = ((o_s - out.unsqueeze(0)).abs() * w.unsqueeze(-1)).amax(0)
    if mutation in ("empty_split_nan", "empty_split_lse0") and len(empty_ids):
        # the empty split's partial gets weight exp(0 - lse_max) against the top-level splits
        hot_ln = HOT_Q * HOT_K * math.log2(math.e) / math.sqrt(hist.shape[-1]) * math.log(2.0)
        lse_top = torch.where(den > 0, top.double() * hot_ln + torch.log(den.clamp(min=1)), torch.zeros_like(den))
        we = torch.exp(-lse_top.clamp(min=0)) * len(empty_ids)
        if mutation == "empty_split_nan":
            out = torch.where((we > 0).view(-1, 1), torch.full_like(out, float("nan")), out)
        else:
            out = out * (1.0 / (1.0 + we)).view(-1, 1)
    return out, top, spread, n


def simulate(case, nsplit, mutation=None, device="cpu", details=False):
    """fp64 sample_mse [2, BH] of the case at split count nsplit, optionally with one MUTATION.
    details=True also returns (out [3, BH, R, D], top level [3, BH, R], spread [3, BH, R, D]) of the unmutated flow."""
    assert mutation is None or mutation in MUTATIONS, mutation
    lay, ctx, F, P, S, D, BH = case.lay, case.ctx, case.F, case.P, case.S, case.D, case.BH
    dev = torch.device(device)
    rows = case.rows.tolist()
    n_rows = len(rows)
    R = 128 if mutation == "padding_summed" else n_rows
    ranges = split_ranges(S, nsplit)
    if mutation == "split_end_plus1":
        k0, k1 = ranges[0]
        ranges[0] = (k0, min(S, k1 + CHUNK))
    if mutation == "split_end_minus1":
        i = max(s for s, (a, b) in enumerate(ranges) if b > a)
        k0, k1 = ranges[i]
        ranges[i] = (k0, max(k0, (k1 - 1) // CHUNK * CHUNK))
    empty_ids = [s for s, (a, b) in enumerate(ranges) if b <= a]
    thres = thres_of(lay, P, rounded=True) if mutation == "thres_rounded" else None

    def mpos(s):
        """mask position of each row in split s (padding rows: 0, like the kernel's q_index)"""
        step = {"qindex_minus1": -1, "qindex_plus1": 1}.get(mutation, 0)
        out = []
        for r in range(R):
            if r >= n_rows:
                out.append(0)
            elif mutation == "qindex_gathered":
                out.append(s * 128 + r)
            elif mutation == "qindex_plus_P":
                out.append((rows[r] + P) % S)
            else:
                out.append(min(max(rows[r] + step, 0), S - 1))
        return out

    src = [((rows[r] + 1) % S if mutation == "q_neighbour" else rows[r]) if r < n_rows else None for r in range(R)]
    names = ["full", "spatial", "temporal"]
    per_split_pos = mutation == "qindex_gathered"
    masks = {}
    for X in names[1:]:
        if per_split_pos:
            masks[X] = [mask_rows(lay, X, [min(p, S - 1) for p in mpos(s)], ctx, F, P, thres).to(dev)
                        for s in range(nsplit)]
        else:
            masks[X] = mask_rows(lay, X, mpos(0), ctx, F, P, thres).to(dev)
    full = torch.ones(R, S, dtype=torch.bool, device=dev)
    j = torch.arange(S, device=dev)
    outs = torch.zeros(3, BH, R, D, dtype=torch.float64)
    tops = torch.zeros(3, BH, R, dtype=torch.long)
    spreads = torch.zeros(3, BH, R, D, dtype=torch.float64)
    for h in range(BH):
        E = torch.zeros(S, D, dtype=torch.float64, device=dev)
        E[j, case.codes[h].to(dev)] = 1
        kc = case.kcls[h].to(dev)
        pc = case.pos_cls[h]
        cls = torch.tensor([pc.get(p, -2) if (case.hot and p is not None) else -2 for p in src], device=dev)
        for x, X in enumerate(names):
            if X == "full":
                parts = _split_partials(full, cls, kc, E, ranges)
            elif per_split_pos:
                parts = [_split_partials(masks[X][s], cls, kc, E, [ranges[s]])[0] for s in range(nsplit)]
            else:
                parts = _split_partials(masks[X], cls, kc, E, ranges)
            o, t, sp, _ = _merge(parts, mutation, empty_ids)
            outs[x, h], tops[x, h], spreads[x, h] = o.cpu(), t.cpu(), sp.cpu()
    if mutation == "passes_swapped":
        outs = outs[[0, 2, 1]]
    if mutation == "last_row_dropped":
        outs[:, :, n_rows - 1] = outs[0:1, :, n_rows - 1]  # difference 0: the row adds nothing
    div = (128 if mutation == "divide_128D" else n_rows) * D
    mse = torch.stack([((outs[1] - outs[0]) ** 2).sum((1, 2)), ((outs[2] - outs[0]) ** 2).sum((1, 2))]) / div
    if mutation == "heads_swapped":
        mse = mse[:, [1, 0] + list(range(2, BH))]
    return (mse, (outs, tops, spreads)) if details else mse


def closed_form(case, device="cpu"):
    """fp64 [2, BH]: the MSEs straight from the masks and classes, without splits (cnt_X / n_X per row)."""
    return simulate(case, 1, device=device)


def _sp32(x):
    return float(np.spacing(np.float32(abs(x))))


def eps_w(level, D, S):
    """relative error of one merge weight __expf(lse_s - lse_max) between two splits of one level"""
    M = level * HOT_Q * HOT_K * math.log2(math.e) / math.sqrt(D)  # exact in fp32 (power-of-two score)
    L = math.log2(max(S, 2))
    V = M + L
    lse = V * math.log(2.0)
    d_lse = math.log(2.0) * (_sp32(L) + _sp32(V) / 2) + lse * 2.0 ** -25 + _sp32(lse) / 2
    x = math.log(max(S, 2))  # |lse_s - lse_max| <= ln(n) within one level
    return 2 * d_lse + _sp32(lse) / 2 + x * math.log2(math.e) * 1.5 * U * math.log(2.0) + 2.0 ** -21


def bound(case, nsplit, device="cpu"):
    """(closed form [2, BH], per-head bound [2, BH]) on |kernel - closed form| at split count nsplit"""
    mse, (out, top, spread) = simulate(case, nsplit, device=device, details=True)
    D, S, n = case.D, case.S, case.n
    rel = (2 + 2 * nsplit + 2 + 4) * U
    ew = torch.where(top > 0, eps_w(1, D, S), eps_w(0, D, S)).double().unsqueeze(-1)
    E = rel * out.abs() + 1.01 * ew * spread  # [3, BH, R, D]
    b = []
    for x in (1, 2):
        e = E[x] + E[0]
        t = (2 * (out[x] - out[0]).abs() * e + e * e).sum((1, 2)) / (n * D)
        b.append((1 + 40 * U) * t + 40 * U * mse[x - 1])
    return mse, torch.stack(b)
