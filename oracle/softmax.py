"""Exact census of the attention kernel's online softmax.  TEST INFRASTRUCTURE ONLY.

The inputs are chosen so that no operation of the kernel rounds before the epilogue; the expected output is then a
closed-form function of the inputs and the mask, whatever the order of chunks, accumulations and rescales.

  scale   The kernel works in log2 units: c = fp32(sm_scale) * fp32(log2 e) (times fp32(q_scale * k_scale) for e4m3).
          `scale_for` finds the fp32 sm_scale that makes c exactly 1/2, 1 or 2.
  scores  Q and K hold small integers (exact in bf16, fp16 and e4m3).  Key position p (in the plan's key order) has a
          class kcls(p) and a level t(p) in 0..R; row r has a class rcls(r) (D - 1: none).  With
              q[r, rcls(r)] = a,  q[r, D-1] = b,   k[p, kcls(p)] = 16,  k[p, D-1] = t(p)
          the score is s = 16a [rcls(r) == kcls(p)] + b t(p), an integer, and c s = GAP [hot] + e t(p) with
          16 a c = GAP = 160 and e = b c in {1, 2}.  Hot keys (class match) and cold keys are >= GAP - e R >= 150
          apart after c, so ex2.approx.ftz gives a cold key seen after a hot one p = 0, and the alpha at a row's first
          hot key, 2^(<= -150), wipes its cold history to exactly 0.  Inside a tier every p and every alpha is a power
          of two in [2^-eR, 1].
  values  V holds integers in [-4, 4].  Every partial sum of P V and of l is a multiple of 2^(s_min - m) c of
          magnitude below `budget` (checked per row, < 2^22), so fp32 holds it exactly in any order.

So the kernel's O and l are exactly O_r = sum_j 2^(c s_j - c M) v_j and l_r = sum_j 2^(c s_j - c M) over the row's
live tier (its hot keys, or all its keys if it has none), M the row max, and

    out = round16(fp32(O) * fp32(fp32(1 / l) * v_scale)),  lse = (M c + log2f(l)) * fp32(ln 2)

The output is compared bit for bit; the lse within log2f's one-ulp error (`lse_bounds`).

The tables are exact integer sums (fp32 matmuls, TF32 off on the GPU: every sum is an integer below 2^24).  `visit` restates the kernel's visit order (band plans: 128-column chunks in ascending key order;
variable-block plans: runs of adjacent selected key blocks cut into 128-column chunks; gather plans: the selected
keys in map order, 128 per chunk) and `simulate` runs the chunk loop on one row in fp64, with optional mutations.
Both serve the coverage and sensitivity claims of the CPU tests only; the GPU tests compare with the closed form.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import numpy as np
import torch

LOG2E = np.float32(1.4426950408889634)   # the kernel's fp32 log2(e)
LN2 = np.float32(0.6931471805599453)     # the kernel's fp32 ln(2)
GAP = 160          # hot - cold distance after c, at equal t
MIN_GAP = 150      # required hot / cold separation: 2^-150 is below every fp32 (ftz: below 2^-126)
BUDGET = 1 << 22   # per-row bound of every partial sum, in units of the tier's smallest term
VMAX = 4           # |v| <= VMAX
EX2_MIN = -126     # ex2.approx.ftz: 2^x for x >= -126, 0 below (subnormal results flush)
CHUNK = 128


# --------------------------------------------------------------------------------------------
# scale
# --------------------------------------------------------------------------------------------
def kernel_c(sm_scale: float, qk_scale: float | None = None) -> float:
    """The kernel's c: fp32(sm_scale) * fp32(log2 e) (attn_fwd.cu), times fp32(q_scale * k_scale) for e4m3."""
    c = np.float32(np.float32(sm_scale) * LOG2E)
    if qk_scale is not None:
        c = np.float32(c * np.float32(qk_scale))
    return float(c)


def scale_for(c: float) -> float:
    """The fp32 sm_scale (as a Python float) for which kernel_c(sm_scale) == c exactly."""
    x = np.float32(np.float32(c) / LOG2E)
    for _ in range(8):
        got = kernel_c(float(x))
        if got == c:
            return float(x)
        x = np.nextafter(x, np.float32(np.inf if got < c else -np.inf))
    raise AssertionError(f"no fp32 sm_scale gives c = {c}")


def qk_ints(c: float):
    """(a, b) of the Q encoding for an effective c: 16 a c = GAP and e = b c an integer >= 1."""
    a = GAP / (16 * c)
    b = max(1.0, 1.0 / c)
    assert a == int(a) and b == int(b) and b * c == int(b * c), c
    return int(a), int(b)


# --------------------------------------------------------------------------------------------
# cases: one problem per head, everything in plan order (plan row r, plan key position p)
# --------------------------------------------------------------------------------------------
@dataclass
class Case:
    name: str
    S: int                   # plan rows (queries)
    D: int
    H: int
    R: int
    c: list                  # effective c per head (fp32-exact powers of two)
    kcls: torch.Tensor       # [H, Skv] key class per plan key position
    kt: torch.Tensor         # [H, Skv] key level t per plan key position
    rcls: torch.Tensor       # [H, S] row class per plan row (D - 1, which no key has: a cold-only row)
    v: torch.Tensor          # [H, Skv, D] int8, per plan key position
    vs: list                 # v_scale per head (1.0 for 16-bit inputs)
    band: tuple | None = None            # (mode, m0, m1, m2) of plan_band
    mod: object = None                   # mask predicate of the band plan
    bm: torch.Tensor | None = None       # [H, QC, KC] block map (variable-block / gather plans)
    rows: torch.Tensor | None = None     # [H, QC]
    cols: torch.Tensor | None = None     # [H, KC]
    gather: bool = False
    q_rows: torch.Tensor | None = None   # [H, S] gather: source row of plan row r
    kv_rows: torch.Tensor | None = None  # [H, S] gather: source row of plan key position p
    o_rows: torch.Tensor | None = None   # [H, S] output row of plan row r
    notes: dict = field(default_factory=dict)
    Skv: int | None = None               # plan key positions (None: S); gather cases are square

    @property
    def Sk(self) -> int:
        return self.S if self.Skv is None else self.Skv

    def qk_plan(self, dtype=torch.float32):
        """Q [H, S, D] and K [H, Skv, D] in plan order (integers, exact in every input format)."""
        q = torch.zeros(self.H, self.S, self.D)
        k = torch.zeros(self.H, self.Sk, self.D)
        C = self.D - 1
        for h in range(self.H):
            a, b = qk_ints(self.c[h])
            r = torch.arange(self.S)
            live = self.rcls[h] < C
            q[h, r[live], self.rcls[h][live].long()] = float(a)
            q[h, :, C] = float(b)
            k[h, torch.arange(self.Sk), self.kcls[h].long()] = 16.0
            k[h, :, C] = self.kt[h].float()
        return q.to(dtype), k.to(dtype)

    def tensors(self, dtype=torch.float32):
        """Q [H, S, D], K, V [H, Skv, D] as the kernel reads them: plan order, or scattered to source rows for gather
        plans."""
        q, k = self.qk_plan(dtype)
        v = self.v.to(dtype)
        if self.gather:
            q2, k2, v2 = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
            for h in range(self.H):
                q2[h, self.q_rows[h].long()] = q[h]
                k2[h, self.kv_rows[h].long()] = k[h]
                v2[h, self.kv_rows[h].long()] = v[h]
            return q2, k2, v2
        return q, k, v


def region_keys(S, L, C, R, offset=0):
    """Key classes and levels by position: regions of L keys take classes 0, 1, .., C-1 in turn and t rises
    0 .. R across each region, so a row whose class is one region's sees that region's keys in rising t."""
    p = torch.arange(S) + offset
    return (p // L) % C, ((p % L) * (R + 1)) // L


def with_cold_rows(rcls, D, every=13, at=7):
    """Rows r with r % every == at get class D - 1, which no key has: they only ever see the cold tier."""
    rcls = rcls.clone()
    rcls[..., at::every] = D - 1
    return rcls


def int_values(H, S, D, gen):
    return torch.randint(-VMAX, VMAX + 1, (H, S, D), generator=gen, dtype=torch.int8)


# --------------------------------------------------------------------------------------------
# visit order (plan order positions and chunk ids of one row)
# --------------------------------------------------------------------------------------------
def _block_runs(bm_row, cols):
    """Selected non-empty key blocks of one q-block -> runs (start, end) of adjacent key positions."""
    starts = torch.cat([torch.zeros(1, dtype=torch.long), cols.long().cumsum(0)])
    runs = []
    for j in torch.nonzero(bm_row & (cols > 0)).flatten().tolist():
        s, e = int(starts[j]), int(starts[j + 1])
        if runs and runs[-1][1] == s:
            runs[-1][1] = e
        else:
            runs.append([s, e])
    return runs


def visit(case: Case, h: int, r: int):
    """(key positions, chunk ids) of plan row r of head h, in the kernel's visit order."""
    if case.mod is not None:
        pos = torch.nonzero(case.mod(torch.tensor([[r]]), torch.arange(case.Sk).view(1, -1))[0]).flatten()
        return pos.numpy(), (pos // CHUNK).numpy()
    qb = int(torch.searchsorted(case.rows[h].long().cumsum(0), torch.tensor(r), right=True))
    runs = _block_runs(case.bm[h, qb], case.cols[h])
    pos, ch, n = [], [], 0
    for s, e in runs:
        pos.append(np.arange(s, e))
        ch.append(n + (pos[-1] - s) // CHUNK)
        n += -(-(e - s) // CHUNK)
    if not pos:
        return np.zeros(0, dtype=np.int64), np.zeros(0, dtype=np.int64)
    pos = np.concatenate(pos)
    # gather plans cut the concatenated selected keys into 128-key chunks, across run boundaries
    return pos, (np.arange(len(pos)) // CHUNK if case.gather else np.concatenate(ch))


def exponents(case: Case, h: int, r: int, pos):
    """c s of plan row r against key positions pos (integers, exact)."""
    a, b = qk_ints(case.c[h])
    hot = (case.kcls[h][pos] == case.rcls[h][r]).numpy()
    return (GAP * hot + b * case.c[h] * case.kt[h][pos].numpy()).astype(np.float64), hot


def _ex2(x):
    return np.where(x >= EX2_MIN, np.exp2(np.maximum(x, EX2_MIN)), 0.0)


def simulate(case: Case, h: int, r: int, mutant: str | None = None):
    """The chunk loop of the kernel on plan row r of head h, in fp64 (exact here).  Returns (O [D], l, m, stats)
    where m is the row max of c s and stats = dict(wipe, partial, last_partial): the chunks whose alpha is 0 with
    O != 0, the chunks after the last wipe whose alpha is in (0, 1) with O != 0, and the index of the last chunk whose
    alpha is in (0, 1) with l > 0.
    mutant: None, "prev_alpha" (O is scaled by the previous chunk's alpha), "l_once" (l is not rescaled at the
    row's last partial rescale), "drop_hot" (the row's first hot key in visit order is skipped)."""
    pos, ch = visit(case, h, r)
    x, hot = exponents(case, h, r, pos)
    v = case.v[h][pos].double().numpy()
    if mutant == "drop_hot" and hot.any():
        keep = np.ones(len(pos), dtype=bool)
        keep[np.argmax(hot)] = False
        x, v, ch = x[keep], v[keep], ch[keep]
    skip_at = simulate(case, h, r)[3]["last_partial"] if mutant == "l_once" else -1
    O = np.zeros(case.D)
    l, m, prev_alpha = 0.0, -np.inf, 1.0
    wipe = partial = 0
    last_partial = -1
    bounds = np.flatnonzero(np.diff(ch)) + 1
    for n, seg in enumerate(np.split(np.arange(len(x)), bounds)):
        if seg.size == 0:
            continue
        m_new = max(m, float(x[seg].max()))
        alpha = 0.0 if m == -np.inf else float(_ex2(np.float64(m - m_new)))
        p = _ex2(x[seg] - m_new)
        nonzero = bool(np.any(O != 0))
        if alpha == 0.0 and nonzero:
            wipe += 1
            partial = 0
        elif 0.0 < alpha < 1.0 and nonzero:
            partial += 1
        if 0.0 < alpha < 1.0 and l > 0:
            last_partial = n
        a_o = prev_alpha if mutant == "prev_alpha" else alpha
        a_l = 1.0 if n == skip_at else alpha
        O = O * a_o + p @ v[seg]
        l = l * a_l + float(p.sum())
        m, prev_alpha = m_new, alpha
    return O, l, m, dict(wipe=wipe, partial=partial, last_partial=last_partial)


# --------------------------------------------------------------------------------------------
# closed form: per-row tables of (tier, level) sums
# --------------------------------------------------------------------------------------------
def _features(case: Case, h: int, device, dtype):
    """[Skv, (R+1)(D+1)]: key p contributes [v_p, 1] in the column group of its level t(p)."""
    R1, D1 = case.R + 1, case.D + 1
    f = torch.zeros(case.Sk, R1, D1, dtype=dtype, device=device)
    idx = torch.arange(case.Sk, device=device)
    t = case.kt[h].long().to(device)
    f[idx, t, : case.D] = case.v[h].to(device=device, dtype=dtype)
    f[idx, t, case.D] = 1
    return f.view(case.Sk, R1 * D1)


def _reduce(case: Case, h: int, hot, allt):
    """Tables [n, R+1, D+1] (hot tier, all keys) -> O [n, D] fp64, l [n], m_raw [n] (raw max score, -inf when the
    row has no key), budget [n] (largest tier sum of 2^(c s - c s_min) * VMAX)."""
    a, b = qk_ints(case.c[h])
    e = b * case.c[h]
    hot, allt = hot.double(), allt.double()
    cold = allt - hot
    D = case.D
    lv = torch.arange(case.R + 1, dtype=torch.float64, device=hot.device)

    def tier(tab):
        cnt = tab[..., D]
        live = cnt > 0
        tmax = torch.where(live, lv, torch.full_like(lv, -1)).max(1).values
        tmin = torch.where(live, lv, torch.full_like(lv, 1e9)).min(1).values
        w = torch.where(live, torch.exp2(e * (lv[None] - tmax[:, None])), torch.zeros_like(cnt))
        bud = (torch.where(live, torch.exp2(e * (lv[None] - tmin[:, None])), torch.zeros_like(cnt)) * cnt).sum(1)
        return (w[..., None] * tab[..., :D]).sum(1), (w * cnt).sum(1), tmax, bud * VMAX

    Oh, lh, th, bh = tier(hot)
    Oc, lc, tc, bc = tier(cold)
    has_hot = lh > 0
    O = torch.where(has_hot[:, None], Oh, Oc)
    l = torch.where(has_hot, lh, lc)
    m_raw = torch.where(has_hot, 16.0 * a + b * th, b * tc)
    m_raw = torch.where(l > 0, m_raw, torch.full_like(m_raw, -math.inf))
    return O, l, m_raw, torch.maximum(bh, bc)


def expected(case: Case, h: int, device="cpu", row_chunk: int = 1024, row_ids=None):
    """Closed form of head h in PLAN row order: O [S, D] fp64, l [S], m_raw [S], budget [S].  Band cases may
    restrict it to the plan rows `row_ids` (the tables then follow their order)."""
    dev = torch.device(device)
    dtype = torch.float32
    old_tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        feat = _features(case, h, dev, dtype)
        kcls = case.kcls[h].to(dev)
        rcls = case.rcls[h].to(dev)
        classes = sorted(set(case.rcls[h].tolist()))
        by_class = {k: torch.nonzero(kcls == k).flatten() for k in classes}
        R1, D1 = case.R + 1, case.D + 1
        outs = []
        if case.mod is not None:
            kv = torch.arange(case.Sk, device=dev).view(1, -1)
            ids = torch.arange(case.S, device=dev) if row_ids is None else torch.as_tensor(row_ids, device=dev)
            for r0 in range(0, ids.numel(), row_chunk):
                rr = ids[r0:r0 + row_chunk]
                A = case.mod(rr.view(-1, 1), kv).to(dtype)
                allt = A @ feat
                hot = torch.zeros_like(allt)
                rc = rcls[rr]
                for k in classes:
                    sel = torch.nonzero(rc == k).flatten()
                    if sel.numel() and by_class[k].numel():
                        hot[sel] = A[sel][:, by_class[k]] @ feat[by_class[k]]
                outs.append(_reduce(case, h, hot.view(-1, R1, D1), allt.view(-1, R1, D1)))
        else:
            cols = case.cols[h].long().to(dev)
            kb = torch.repeat_interleave(torch.arange(cols.numel(), device=dev), cols)
            bm = case.bm[h].to(device=dev, dtype=dtype)
            qb = torch.repeat_interleave(torch.arange(case.rows[h].numel(), device=dev), case.rows[h].long().to(dev))
            allt = (bm @ torch.zeros(cols.numel(), feat.shape[1], dtype=dtype, device=dev).index_add_(0, kb, feat))[qb]
            hot = torch.zeros_like(allt)
            for k in classes:
                sel = torch.nonzero(rcls == k).flatten()
                fk = torch.zeros_like(feat)
                fk[by_class[k]] = feat[by_class[k]]
                pb = torch.zeros(cols.numel(), feat.shape[1], dtype=dtype, device=dev).index_add_(0, kb, fk)
                hot[sel] = (bm @ pb)[qb[sel]]
            outs.append(_reduce(case, h, hot.view(-1, R1, D1), allt.view(-1, R1, D1)))
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old_tf32
    return tuple(torch.cat([o[i] for o in outs]).cpu() for i in range(4))


def to_output_rows(case: Case, h: int, *tabs):
    """Plan-row tables -> output-row tables (output row o_rows[r] holds plan row r)."""
    if case.o_rows is None:
        return tabs
    idx = case.o_rows[h].long()
    out = []
    for t in tabs:
        t2 = torch.empty_like(t)
        t2[idx] = t
        out.append(t2)
    return tuple(out)


def expected_output(O, l, vs: float, out_dtype):
    """round16(fp32(O) * fp32(fp32(1 / l) * vs)); rows without keys give 0 (IEEE division, as the kernel)."""
    lf = l.to(torch.float32)
    inv = torch.where(lf > 0, torch.reciprocal(lf), torch.zeros_like(lf)) * torch.tensor(vs, dtype=torch.float32)
    assert torch.equal(O.to(torch.float32).double(), O), "O is not an fp32 value"
    return (O.to(torch.float32) * inv[:, None]).to(out_dtype)


def lse_bounds(m_raw, l, c: float):
    """[lo, hi] of the kernel's fp32 lse = (m c + log2f(l)) * fp32(ln 2) when log2f is within one ulp; -inf for
    rows without keys.  m c is exact (an integer), the sum and the product round once each (fp32, numpy)."""
    mr = m_raw.numpy()
    live = l.numpy() > 0
    lv = np.where(live, l.numpy(), 1.0)
    mc = np.where(live, mr, 0.0).astype(np.float32) * np.float32(c)
    L = np.log2(lv).astype(np.float32)
    cands = []
    for Lc in (np.nextafter(L, np.float32(-np.inf)), L, np.nextafter(L, np.float32(np.inf))):
        cands.append(((mc + Lc).astype(np.float32) * LN2).astype(np.float32))
    lo = np.where(live, np.minimum.reduce(cands), -np.inf)
    hi = np.where(live, np.maximum.reduce(cands), -np.inf)
    return torch.from_numpy(lo), torch.from_numpy(hi)


def exact_lse(m_raw, l, c: float):
    """(m c + log2 l) ln 2 in fp64 (the kernel result is compared against lse_bounds)."""
    return torch.where(l > 0, (m_raw * c + torch.log2(l.clamp(min=1e-300))) * math.log(2), torch.full_like(l, -math.inf))


# --------------------------------------------------------------------------------------------
# the cases of tests/test_softmax_census_gpu.py (built on the CPU; the CPU tests check budget and coverage)
# --------------------------------------------------------------------------------------------
HY720 = dict(ctx=256, F=33, P=3600, plen=71)

# name -> (mask kind, band_args / generic parameters, S, L, R, C): small band plans, S not a multiple of 128
BAND = {
    "hy": ("hy", (6, 200, 48, 20, 4.0), 48 + 6 * 200, 512, 3, 8),
    "wan": ("wan", (7, 180, 0, 0, 3.0), 7 * 180, 512, 3, 8),
    "cog": ("cog", (4, 260, 40, 40, 2.5), 40 + 4 * 260, 512, 3, 8),
    "cog_sink": ("cog_sink", (4, 260, 40, 40, 2.5), 40 + 4 * 260, 512, 3, 8),
    "generic_254": ("generic", (2, 50, 0, 254), 1100, 384, 2, 8),
    "generic_255": ("generic", (1, 1800, 1900, 255), 1993, 384, 2, 8),
    "none": ("generic", (0, 0, 0, 0), 1000, 384, 2, 8),
}


def band_case(name, D=128, H=2, c=None, vs=None, seed=0):
    from oracle import attention as oa
    from oracle import census as oc

    if name == "hy720":
        h = HY720
        S, L, R, C = h["ctx"] + h["F"] * h["P"], 4096, 3, 8
        mul = oa.sparsity_to_width(0.3, h["ctx"], h["F"], h["P"])
        band, mod = oc.band_args("hy", h["F"], h["P"], h["ctx"], h["plen"], mul)
    else:
        kind, args, S, L, R, C = BAND[name]
        if kind == "generic":
            band, mod = args, oa.generic_mask_fn(*args)
        else:
            band, mod = oc.band_args(kind, *args, attn_sink=kind == "cog_sink")
    g = torch.Generator().manual_seed(seed)
    kcls, kt = region_keys(S, L, C, R)
    # a row takes the class of its own region (region 1 for rows of region 0): the band reaches it after the cold
    # keys before the region, and sees the region's t rise
    rcls = with_cold_rows((torch.clamp(torch.arange(S), min=L) // L) % C, D)
    c = c or [1.0] * H
    return Case(name, S, D, H, R, list(c), kcls.expand(H, S).clone(), kt.expand(H, S).clone(),
                rcls.expand(H, S).clone(), int_values(H, S, D, g), list(vs or [1.0] * H), band=band, mod=mod)


def _anchor_classes(case: Case, L, C, frac, offset=0):
    """Row classes of a block-map case: the class of the region holding the key at `frac` of the row's visit order,
    so the row meets cold keys first and that region's rising t later (regions as region_keys(..., offset))."""
    rcls = torch.full((case.H, case.S), case.D - 1, dtype=torch.long)
    for h in range(case.H):
        ends = case.rows[h].long().cumsum(0)
        for qb in range(case.rows[h].numel()):
            n = int(case.rows[h][qb])
            if n == 0:
                continue
            pos, _ = visit(case, h, int(ends[qb]) - n)
            if len(pos):
                rcls[h, int(ends[qb]) - n: int(ends[qb])] = ((int(pos[int(frac * len(pos))]) + offset) // L) % C
    return with_cold_rows(rcls, case.D)


def _finish_blocks(case: Case, L, R, C, frac, offset=0):
    kcls, kt = region_keys(case.Sk, L, C, R, offset)
    case.kcls, case.kt = kcls.expand(case.H, case.Sk).clone(), kt.expand(case.H, case.Sk).clone()
    case.rcls = _anchor_classes(case, L, C, frac, offset)
    return case


def varblock_case(D=128, c=None, vs=None, seed=1):
    """Two heads, S = 6000, 24 q-blocks of q_sizes (every r % 256 class, empty q-blocks, odd tail count), 60 key
    blocks: head 0 the "joined" map (runs across empty key blocks, an all-selected and an all-empty q-block),
    head 1 a random map of density 0.4.  Output through a random o_rows."""
    from oracle import census as oc

    g = torch.Generator().manual_seed(seed)
    H, S, QC, KC = 2, 6000, 24, 60
    rows = torch.stack([oc.q_sizes(S, QC, g) for _ in range(H)]).int()
    bm0, col0 = oc.varblock_head("joined", QC, KC, S, g)
    col1 = oc.partition(S, KC, g)
    bm1 = torch.rand(QC, KC, generator=g) < 0.4
    bm, cols = torch.stack([bm0, bm1]), torch.stack([col0, col1]).int()
    o_rows = torch.stack([torch.randperm(S, generator=g) for _ in range(H)]).int()
    z = torch.zeros(H, S, dtype=torch.long)
    case = Case("varblock", S, D, H, 3, list(c or [1.0] * H), z, z, z, int_values(H, S, D, g), list(vs or [1.0] * H),
                bm=bm, rows=rows, cols=cols, o_rows=o_rows)
    return _finish_blocks(case, 2048, 3, 4, 0.5)


def gather_case(D=128, c=None, vs=None, seed=2):
    """Two heads, S = 6000, 37 query and 101 key clusters from random labels; plan rows and keys in cluster order
    (stable argsort), read through q_rows / kv_rows, written through o_rows.  Head 0 has an empty query cluster, a
    query cluster that selects nothing and one that selects everything; head 1 an empty key cluster."""
    g = torch.Generator().manual_seed(seed)
    H, S, QC, KC = 2, 6000, 37, 101
    ql = torch.randint(0, QC, (H, S), generator=g)
    kl = torch.randint(0, KC, (H, S), generator=g)
    ql[0][ql[0] == 5] = 6
    kl[1][kl[1] == 3] = 4
    bm = torch.rand(H, QC, KC, generator=g) < 0.4
    bm[0, 7, :] = False
    bm[0, 8, :] = True
    qperm = torch.sort(ql, dim=1, stable=True).indices.int()
    kperm = torch.sort(kl, dim=1, stable=True).indices.int()
    rows = torch.stack([torch.bincount(ql[h], minlength=QC) for h in range(H)]).int()
    cols = torch.stack([torch.bincount(kl[h], minlength=KC) for h in range(H)]).int()
    z = torch.zeros(H, S, dtype=torch.long)
    case = Case("gather", S, D, H, 3, list(c or [1.0] * H), z, z, z, int_values(H, S, D, g), list(vs or [1.0] * H),
                bm=bm, rows=rows, cols=cols, gather=True, q_rows=qperm, kv_rows=kperm, o_rows=qperm)
    return _finish_blocks(case, 2048, 3, 4, 0.5)


def rect_blockmap_case(name, bm, rows, cols, D=128, c=None, vs=None, seed=5, L=512, R=3, C=4, frac=0.5, offset=0):
    """A variable-block case of Sq = sum(rows) queries and Skv = sum(cols) keys: bm [H, QC, KC], rows [H, QC],
    cols [H, KC].  Key classes and levels over the Skv keys (region_keys with `offset`), every q-block's class from its
    own visit order (_anchor_classes), so its rows meet cold keys first, are wiped by their first hot chunk and rescale
    afterwards."""
    H = bm.shape[0]
    Sq, Skv = int(rows[0].sum()), int(cols[0].sum())
    g = torch.Generator().manual_seed(seed)
    zq, zk = torch.zeros(H, Sq, dtype=torch.long), torch.zeros(H, Skv, dtype=torch.long)
    case = Case(name, Sq, D, H, R, list(c or [1.0] * H), zk, zk, zq, int_values(H, Skv, D, g), list(vs or [1.0] * H),
                bm=bm, rows=rows.int(), cols=cols.int(), Skv=Skv)
    return _finish_blocks(case, L, R, C, frac, offset)


def row_anchor_classes(mod, S, Skv, L, C, D, frac=0.5, device="cpu", row_chunk=512):
    """Row classes [S] of a mask-predicate case over S x Skv: the class of the region holding the key at `frac` of each
    row's own visit order (ascending keys), as _anchor_classes takes it per q-block; D - 1 for rows without keys."""
    dev = torch.device(device)
    rcls = torch.full((S,), D - 1, dtype=torch.long)
    kv = torch.arange(Skv, device=dev).view(1, -1)
    for r0 in range(0, S, row_chunk):
        r1 = min(S, r0 + row_chunk)
        m = mod(torch.arange(r0, r1, device=dev).view(-1, 1), kv)
        n = m.sum(1)
        idx = torch.floor(frac * n.double()).long()
        pos = (m.long().cumsum(1) <= idx[:, None]).sum(1)  # the idx-th allowed key (0-based) of every row
        rcls[r0:r1] = torch.where(n > 0, (pos // L) % C, torch.full_like(pos, D - 1)).cpu()
    return rcls


def mask_case(name, mod, S, Skv, D=128, H=2, L=384, R=3, C=8, c=None, vs=None, seed=6, frac=0.5, device="cpu"):
    """A case of any mask predicate mod(q_idx, kv_idx) over S queries and Skv keys, in the visit order of band and
    segment plans (128-key chunks in ascending key order): key regions of L keys over the Skv keys, each row's class
    from its own visit order (row_anchor_classes), every 13th row cold-only."""
    g = torch.Generator().manual_seed(seed)
    kcls, kt = region_keys(Skv, L, C, R)
    rcls = with_cold_rows(row_anchor_classes(mod, S, Skv, L, C, D, frac, device), D)
    return Case(name, S, D, H, R, list(c or [1.0] * H), kcls.expand(H, Skv).clone(), kt.expand(H, Skv).clone(),
                rcls.expand(H, S).clone(), int_values(H, Skv, D, g), list(vs or [1.0] * H), mod=mod, Skv=Skv)


def bsr_case(D=128, seed=3):
    """The reference's temporal BSR blocks (F = 8, P = 300, blocks of 30) behind a 40-row all-to-all text prefix,
    one plan for both heads (items_stride = 0)."""
    from oracle import attention as oa

    H, F, P, text = 2, 8, 300, 40
    blocks, (Rb, _) = oa.ref_gen_temporal_mask(F, P, 1.5)
    keep = torch.from_numpy(blocks >= 0)
    MB = keep.shape[0]
    bm = torch.ones(MB + 1, MB + 1, dtype=torch.bool)
    bm[1:, 1:] = keep
    sz = torch.tensor([text] + [Rb] * MB, dtype=torch.int32)
    S = text + F * P
    g = torch.Generator().manual_seed(seed)
    z = torch.zeros(H, S, dtype=torch.long)
    case = Case("bsr", S, D, H, 3, [1.0] * H, z, z, z, int_values(H, S, D, g), [1.0] * H,
                bm=bm.expand(H, -1, -1).contiguous(), rows=sz.expand(H, -1).contiguous(),
                cols=sz.expand(H, -1).contiguous())
    case.notes["indptr"] = torch.cat([torch.zeros(1, dtype=torch.long), keep.sum(1).cumsum(0)])
    case.notes["indices"] = keep.nonzero()[:, 1]
    case.notes["bsr"] = (F, P, text, Rb)
    return _finish_blocks(case, 512, 3, 8, 0.5)


# e4m3: per-head q_scale, k_scale (product 2 on head 0, 1/2 on head 1, c = 1 from sm_scale) and v_scale
FP8_QS, FP8_KS, FP8_VS = [4.0, 0.25], [0.5, 2.0], [0.5, 2.0]
FP8_C = [kernel_c(scale_for(1.0), float(np.float32(q) * np.float32(k))) for q, k in zip(FP8_QS, FP8_KS)]


def premise_case(which, D=128):
    """The smallest cases of the three premises the design rests on (mode NONE, one chunk, one item):
    ex2     : every row has four hot keys with t = 0..3 (p = 1/8 .. 1, each in its own V column: V is the identity)
              and 124 cold keys 160 below (p = 0);
    accum   : every key hot with t = 0 (p = 1) and random integer V: the P V wgmma sums 128 integer products;
    e4m3_qk : S = 100, exactly one hot key per row (key r for row r, random t), so O = v_r, l = 1 and the lse is
              M c ln 2 itself (both heads of FP8_C)."""
    g = torch.Generator().manual_seed(4)
    if which == "e4m3_qk":
        H, S = 2, 100
        kcls = torch.arange(S).expand(H, S).clone()
        kt = torch.randint(0, 4, (H, S), generator=g)
        rcls = kcls.clone()
        v, c, vs = int_values(H, S, D, g), FP8_C, FP8_VS
    else:
        H, S = 1, 128
        c, vs = [1.0], [1.0]
        if which == "ex2":
            kcls = (torch.arange(S) % 32)[None]
            kt = (torch.arange(S) // 32)[None]
            rcls = kcls.clone()
            v = torch.eye(S, D, dtype=torch.int8)[None]
        else:
            kcls = torch.zeros(1, S, dtype=torch.long)
            kt = torch.zeros(1, S, dtype=torch.long)
            rcls = kcls.clone()
            v = int_values(1, S, D, g)
    from oracle import attention as oa

    return Case(f"premise_{which}", S, D, H, 3, list(c), kcls, kt, rcls, v, list(vs), band=(0, 0, 0, 0),
                mod=oa.generic_mask_fn(0, 0, 0, 0))


def coverage(case: Case, stride: int = 1):
    """Visit-order statistics over plan rows r = 0, stride, 2 stride, ... of every head: rows with keys, rows that
    see a wipe and then at least two partial rescales, cold-only rows with keys, rows without keys, and rows of a
    second 128-row stream (band plans: rows 128..255 of each 256-row item) with keys.  Also checks that the
    chunk-loop simulation reproduces the closed form on every visited row."""
    st = dict(rows=0, keyed=0, covered=0, wipes=0, cold_only=0, keyless=0, stream1=0)
    rows = list(range(0, case.S, stride))
    for h in range(case.H):
        if case.mod is not None:
            O, l, m_raw, _ = expected(case, h, row_ids=rows)
        else:
            O, l, m_raw, _ = (t[rows] for t in expected(case, h))
        for i, r in enumerate(rows):
            Os, ls, ms, s = simulate(case, h, r)
            assert np.array_equal(Os, O[i].numpy()) and ls == float(l[i]), (case.name, h, r)
            assert ms == (float(m_raw[i]) * case.c[h] if ls > 0 else -np.inf), (case.name, h, r)
            st["rows"] += 1
            if ls == 0:
                st["keyless"] += 1
                continue
            st["keyed"] += 1
            st["covered"] += int(s["wipe"] > 0 and s["partial"] >= 2)
            st["wipes"] += int(s["wipe"] > 0)
            st["cold_only"] += int(int(case.rcls[h, r]) == case.D - 1)
            st["stream1"] += int(case.mod is not None and r % 256 >= 128)
    return st
