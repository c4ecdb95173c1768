"""Closed form of split KV-cache attention (svgb_attn_fwd_kvcache_split, plan_kvcache(num_splits=)).  TEST
INFRASTRUCTURE ONLY.

The split forward runs in two launches: one attention pass per split writes fp32 partials o_s [n, R, Hq, D] and
lse_s [n, Hq, R] (the split_items epilogue of csrc/attn_kernel.cuh), then kv_split_merge_kernel (csrc/attn_fwd.cu)
combines them.  This module predicts both from the mask alone.

Split rule (mirror of kv_lists_kernel, csrc/kvcache.cu).  Item k of stream b (rows r0 = 256 k .., at logical positions
p = L_b - Sq + r) visits its sink chunks [0, ns) first, then the window chunks [jlo, jhi] of its first and last
positions (block-causal: rounded to their block ends).  These nvis chunks are cut into pieces of ceil(nvis / n) in
that order; split s keeps the chunks of its piece that hold an allowed key of some row of the item.  Under the token
rule and the block rule the window of an item is the union of its rows' windows, one interval, and every sink is
allowed to every row, so no visited chunk is empty: cutting the kept list would give the same pieces here.  The CPU
suite checks that premise on every case.

Key census (q = 0; V one-hot by key code, kv head hk encodes logical key j as code_{hk mod 2}(j + 101 hk), the codes of
oracle/census.py).  Every allowed score is 0, so p = 1, and on the keys K_s(r) = allowed(r) ∩ chunks(s, item(r)):
    o_s[r, d] = fp32(cnt_s[r, d]) * fp32(1 / n_s[r])   bit for bit,  cnt_s = #{j in K_s : code(j) = d}, n_s = |K_s|
    lse_s[r]  = fp32(fp32(log2f(n_s)) * fp32(ln 2))    inside oracle.softmax.lse_bounds(m_raw = 0, l = n_s, c)
and a row that split s does not reach has o_s = 0, lse_s = -inf.  The merged lse identifies N = sum_s n_s, the
single-pass count of the mask, as long as the merge error stays far below ln((N + 1) / N) (lse_count_margin).

Merge bound (bound()).  From partials (x_s, lambda_s) the kernel computes, over the splits in order,
    m = max lambda_s  (exact),  d_s = fl(lambda_s - m),  w_s = expf(d_s)  (0 for lambda_s = -inf),
    acc = fmaf(w_s, x_s, acc),  den = den + w_s,  o = round16(fl(acc * fl(1 / den))),  lse = fl(m + logf(den)).
-O3 without --use_fast_math keeps expf and logf the accurate functions: the CUDA C Programming Guide gives expf a
maximum error of 2 ulp and logf 1 ulp.  With W_s = e^(lambda_s - m) in exact arithmetic and y = sum W x / sum W:
  * weights: fl(lambda_s - m) is off by at most u |d_s| (u = 2^-24), and 2 ulp of expf is at most 4u relative, so
    w_s = W_s (1 + rho_s), |rho_s| <= r_s = e^(u |d_s| + sigma_s + sigma_m) (1 + 4u) - 1, where sigma_s bounds an
    uncertainty of lambda_s itself (0 for the kernel's own partials; the lse_bounds width for closed-form partials).
    Where W_s falls below 2^-125 (a split more than ~87 nats under the top one, as a cold split beside a hot one in
    the softmax census) expf's result is subnormal or 0 and its 2 ulp are absolute: w_s lies in
    [0, W_s + 2 * 2^-149], so r_s = 1 + 2^-148 / W_s there and the lower sums take max(1 - r_s, 0).
    Then y' = sum w x / sum w differs from y by sum W rho (x - y') / sum w, so
        e1 = sum W r |x - y| / sum W max(1 - r, 0)      (to first order; the factor 1.01 below covers the rest);
  * two sums of n terms with one rounding per term (fmaf, add): gamma_n = n u / (1 - n u) relative to the sums of
    |terms|, so the ratio acc / den is off from y' by at most
        e2 = gamma_n (sum W (1 + r) |x| + (|y| + e1) sum W (1 + r)) / (sum W (1 - r) (1 - gamma_n));
  * the reciprocal and the product: 2u relative, e3 = 2.01 u (|y| + e1 + e2).
  * subnormal sums and products round to an absolute 2^-150, not a relative u: n + 1 roundings, each scaled by at
    most 1 / den <= 1 (the top split's weight is expf(0) = 1).
    beta = 1.01 (e1 + e2 + e3 + (n + 1) 2^-150), and the kernel's 16-bit o must be round16(x) for some x in [y - beta, y + beta]: the
    two (at most) 16-bit values round16(y - beta) .. round16(y + beta).
  * lse: den = sum W (1 + eta), |eta| <= eta_max = r_w + gamma_n (1 + r_w) with r_w = sum W r / sum W, ln den is off by
    eta' = -ln(1 - eta_max), logf by 1 ulp <= 2u |ln den|, and the sum rounds once (u |lse|):
        beta_l = 1.01 (eta' + 2u (|ln sum W| + eta') + u (|m + ln sum W| + eta') + sigma_m),
    around m + ln sum W = ln sum_s e^lambda_s.
merge_fp32() emulates the merge in fp32 with every expf and logf result moved by up to its ulp error, and the CPU suite
checks that it never leaves the bound.

Softmax census (softmax_partials()).  The key census has q = 0, so every lse_s is ln(n_s) <= 10.4 and the merge never
meets a wide range.  oracle/softmax.py's census, on one stream whose Sq = L queries are its keys, gives each split the
Case whose mod is the KV mask restricted to the split's chunks; oracle.softmax.expected then yields O, l, m_raw per
split, the partial is expected_output(O, l, vs, float32) bit for bit and lse_s lies inside lse_bounds.  A split that
holds a row's hot keys has lse_s >= GAP ln 2 ~ 111; one that holds only cold keys for it lies more than 100 nats
lower, so a merge without the max (expf(111) overflows fp32) or with m from another split than the top one fails.
The premise of the census (every partial sum below BUDGET) is rechecked per split, since a split without a row's hot
keys makes its cold tier live.

simulate() runs the flow on the CPU (split rule, per-split closed forms, the epilogue's partial offsets, the merge)
with one MUTATION, a plausible bug of that flow; the CPU suite shows that each one either changes a bit-exact partial
or moves a merged output of some GPU case by at least 10x its bound.
"""
from __future__ import annotations

import dataclasses
import math
from dataclasses import dataclass, field

import numpy as np

CHUNK, ITEM_ROWS = 128, 256
U = 2.0 ** -24
EXPF_ULP, LOGF_ULP = 2, 1   # CUDA C Programming Guide, maximum ulp error of expf and logf
LN2 = np.float32(0.6931471805599453)
BIG = 1 << 40               # an unbounded window

MUTATIONS = (
    "piece_floor",          # piece = floor(nvis / n) instead of ceil
    "piece_over_kept",      # the pieces cut over the kept chunks instead of the visited ones
    "piece_end_plus1",      # every piece ends one chunk late: a chunk in two splits
    "piece_end_minus1",     # every piece ends one chunk early: a chunk dropped
    "sinks_last",           # the visit order puts the window first and the sinks last
    "slot_plus1",           # the epilogue writes split s at slot min(s + 1, n - 1)
    "slot_minus1",          # the epilogue writes split s at slot max(s - 1, 0)
    "lse_head_stride",      # the epilogue's lse offset of split s is s S, not s Hq S
    "equal_weights",        # every live split weighs 1
    "exp2_weights",         # w_s = exp2(lse_s - m)
    "m_split0",             # m = lse_0 instead of the max
    "m_first_live",         # m = the first finite lse_s instead of the max
    "no_max",               # no max subtracted: w_s = expf(lse_s), lse = logf(den)
    "ninf_weight1",         # a -inf split counted with w = 1
    "lse_without_m",        # lse = log(den)
    "neighbour_head",       # the merge reads head h + 1's partials
    "neighbour_row",        # the merge reads row r + 1's partials
    "nokey_nan",            # a row without keys gets o = acc / 0 = NaN
)


# --------------------------------------------------------------------------------------------
# masks and cases
# --------------------------------------------------------------------------------------------
@dataclass
class Mask:
    """Token rule (block = 0): p sees kv < sink or p - left <= kv <= p + right.  Block rule (block = C > 0): p sees
    kv < sink or e(p) - window <= kv < e(p), e(p) the end of p's block (the first ends at first_block)."""
    sink: int = 0
    left: int = BIG
    right: int = 0
    block: int = 0
    first_block: int = 0
    window: int = -1

    def plan_kwargs(self):
        """keyword arguments of core.plan_kvcache"""
        if self.block:
            return dict(window_size=(self.window, -1), sink=self.sink, block=self.block, first_block=self.first_block)
        if self.right == 0:
            return dict(causal=True, window_size=(-1 if self.left >= BIG else self.left, 0), sink=self.sink)
        return dict(window_size=(-1 if self.left >= BIG else self.left, self.right), sink=self.sink)

    def ends(self, p):
        """e(p) of the block rule (numpy int array)"""
        k = np.maximum((p - self.first_block) // self.block + 1, 0)
        return self.first_block + k * self.block

    def row_sets(self, p, L):
        """allowed keys of positions p (int64 array) in a stream of L keys: [0, a1) and [b0, b1), disjoint"""
        a1 = np.full_like(p, min(self.sink, L))
        if self.block:
            e = self.ends(p)
            b0 = np.zeros_like(p) if self.window == -1 else np.maximum(e - self.window, 0)
            b1 = np.minimum(e, L)
        else:
            b0 = np.maximum(p - self.left, 0)
            b1 = np.minimum(p + self.right + 1, L)
        b0 = np.maximum(b0, a1)
        return a1, b0, np.maximum(b1, b0)

    def allowed(self, p, kv):
        """the predicate on one pair (for checks against tests/kvcache_mask.py and tests/block_causal_mask.py)"""
        if kv < self.sink:
            return True
        if self.block:
            e = int(self.ends(np.int64(p)))
            return kv < e and (self.window == -1 or kv >= e - self.window)
        return p - kv <= self.left and kv - p <= self.right

    def kernel_window(self):
        """(left, right) the planner's visit rule works with (block rule: W - 1 and 0 on rounded positions)"""
        if self.block:
            return (BIG if self.window == -1 else self.window - 1), 0
        return self.left, self.right

    def first_last(self, p0, p1):
        if self.block:
            return int(self.ends(np.int64(p0))) - 1, int(self.ends(np.int64(p1))) - 1
        return p0, p1


@dataclass
class Case:
    name: str
    Ls: list                 # keys per stream (the lengths the plan sees)
    Sq: int
    Hkv: int
    G: int
    D: int
    fmt: str                 # "bf16", "fp16", "e4m3" (per-head scales), "e4m3_rows" (per-row scales)
    layout: str              # "contig", "paged", "batch_idx"
    mask: Mask
    n: int                   # splits; 0: the automatic count
    page: int = 256
    seed: int = 0
    notes: dict = field(default_factory=dict)

    @property
    def B(self):
        return len(self.Ls)

    @property
    def Hq(self):
        return self.G * self.Hkv

    @property
    def R(self):
        return self.B * self.Sq

    @property
    def items_per_stream(self):
        return -(-self.Sq // ITEM_ROWS)


# --------------------------------------------------------------------------------------------
# the split rule
# --------------------------------------------------------------------------------------------
def _visit(L, Sq, k, mask):
    """(visited chunks in visit order, ns) of item k of a stream of L keys (kv_lists_kernel)"""
    r0 = k * ITEM_ROWS
    nr = min(ITEM_ROWS, Sq - r0)
    p0 = L - Sq + r0
    e0, e1 = mask.first_last(p0, p0 + nr - 1)
    left, right = mask.kernel_window()
    nch = -(-L // CHUNK)
    ns = -(-min(mask.sink, L) // CHUNK)
    lo, hi = max(e0 - left, 0), min(e1 + right, L - 1)
    jlo = max(ns, lo // CHUNK)
    jhi = -1 if hi < lo else min(nch - 1, hi // CHUNK)
    return list(range(ns)) + list(range(jlo, jhi + 1)), ns


def chunk_kinds(L, Sq, k, mask, chunks):
    """per chunk j: (any row of item k sees a key of it, some row misses one of its valid keys)"""
    r0 = k * ITEM_ROWS
    nr = min(ITEM_ROWS, Sq - r0)
    p = np.arange(r0, r0 + nr, dtype=np.int64) + (L - Sq)
    a1, b0, b1 = mask.row_sets(p, L)
    out = []
    for j in chunks:
        c0, c1 = j * CHUNK, min(j * CHUNK + CHUNK, L)
        cnt = _ov(0, a1, c0, c1) + _ov(b0, b1, c0, c1)
        out.append((bool((cnt > 0).any()), bool((cnt < c1 - c0).any())))
    return out


def _ov(a, b, c0, c1):
    return np.maximum(np.minimum(b, c1) - np.maximum(a, c0), 0)


def split_lists(L, Sq, k, mask, n, mutation=None):
    """[n lists of (chunk j, elem)]: the chunks split s of item k keeps, in visit order"""
    vis, ns = _visit(L, Sq, k, mask)
    if mutation == "sinks_last":
        vis = vis[ns:] + vis[:ns]
    kinds = chunk_kinds(L, Sq, k, mask, vis)
    if mutation == "piece_over_kept":
        pairs = [(j, e) for j, (live, e) in zip(vis, kinds) if live]
        vis, kinds = [j for j, _ in pairs], [(True, e) for _, e in pairs]
    nvis = len(vis)
    piece = nvis // n if mutation == "piece_floor" else -(-nvis // n)
    out = []
    for s in range(n):
        v_lo = min(nvis, s * piece)
        end = v_lo + piece + {"piece_end_plus1": 1, "piece_end_minus1": -1}.get(mutation, 0)
        v_hi = max(v_lo, min(nvis, end))
        out.append([(vis[i], kinds[i][1]) for i in range(v_lo, v_hi) if kinds[i][0]])
    return out


def visited_all_live(case):
    """True when no visited chunk of any item is empty (the premise under which cutting the kept list is the rule)"""
    for L in case.Ls:
        for k in range(case.items_per_stream):
            vis, _ = _visit(L, case.Sq, k, case.mask)
            if not all(live for live, _ in chunk_kinds(L, case.Sq, k, case.mask, vis)):
                return False
    return True


def plan_lists(case, n, mutation=None):
    """per plan item it = s B I + b I + k: (first packed row, rows, [(chunk j, elem)]) as kv_lists_kernel writes them"""
    I = case.items_per_stream
    per = {}
    for b, L in enumerate(case.Ls):
        for k in range(I):
            per[b, k] = split_lists(L, case.Sq, k, case.mask, n, mutation)
    out = []
    for s in range(n):
        for b in range(case.B):
            for k in range(I):
                out.append((b * case.Sq + k * ITEM_ROWS, min(ITEM_ROWS, case.Sq - k * ITEM_ROWS), per[b, k][s]))
    return out


# --------------------------------------------------------------------------------------------
# key census per split
# --------------------------------------------------------------------------------------------
def code_shift(hk):
    return 101 * hk


def key_codes(S, D, hk):
    """code of logical keys 0 .. S-1 under kv head hk"""
    t = np.arange(S, dtype=np.int64) + code_shift(hk)
    return t % D if hk % 2 == 0 else (t // D) % D


def _code_prefix(x, D, enc):
    """#{t in [0, x) : code_enc(t) = d} for x [R] -> [R, D]"""
    d = np.arange(D, dtype=np.int64)[None]
    x = x[:, None]
    if enc == 0:
        return np.maximum((x - d + D - 1) // D, 0)
    full, rem = x // (D * D), x % (D * D)
    return full * D + np.clip(rem - d * D, 0, D)


def _runs(js):
    """sorted chunk list -> maximal runs [(j0, j1)) (duplicates kept as separate runs)"""
    runs = []
    for j in js:
        if runs and runs[-1][1] == j:
            runs[-1][1] = j + 1
        else:
            runs.append([j, j + 1])
    return runs


def key_census(case, n, mutation=None):
    """(n_s [n, R] int64, cnt_s [n, R, Hkv, D] int64) of every split and packed row, and the full count N [R]"""
    R, D, I = case.R, case.D, case.items_per_stream
    ns_ = np.zeros((n, R), dtype=np.int64)
    cnt = np.zeros((n, R, case.Hkv, D), dtype=np.int64)
    N = np.zeros(R, dtype=np.int64)
    for b, L in enumerate(case.Ls):
        for k in range(I):
            r0 = k * ITEM_ROWS
            nr = min(ITEM_ROWS, case.Sq - r0)
            rows = slice(b * case.Sq + r0, b * case.Sq + r0 + nr)
            p = np.arange(r0, r0 + nr, dtype=np.int64) + (L - case.Sq)
            a1, b0, b1 = case.mask.row_sets(p, L)
            N[rows] = a1 + (b1 - b0)
            for s, lst in enumerate(split_lists(L, case.Sq, k, case.mask, n, mutation)):
                for j0, j1 in _runs(sorted(j for j, _ in lst)):
                    c0, c1 = j0 * CHUNK, min(j1 * CHUNK, L)
                    for lo, hi in ((np.zeros_like(a1), a1), (b0, b1)):
                        x0 = np.clip(lo, c0, c1)
                        x1 = np.clip(hi, c0, c1)
                        x1 = np.maximum(x1, x0)
                        ns_[s, rows] += x1 - x0
                        for hk in range(case.Hkv):
                            sh = code_shift(hk)
                            cnt[s, rows, hk] += _code_prefix(x1 + sh, D, hk % 2) - _code_prefix(x0 + sh, D, hk % 2)
    return ns_, cnt, N


def partials_fp32(ns_, cnt, G):
    """the kernel's partials of the key census: o [n, R, Hq, D] fp32, lse [n, Hq, R] fp32"""
    nf = ns_.astype(np.float32)
    with np.errstate(divide="ignore"):
        inv = np.where(nf > 0, np.float32(1) / np.where(nf > 0, nf, 1), np.float32(0)).astype(np.float32)
        l2 = np.log2(np.where(nf > 0, nf, 1)).astype(np.float32)
    o = (cnt.astype(np.float32) * inv[:, :, None, None]).astype(np.float32)
    o = np.repeat(o, G, axis=2)
    lse = np.where(nf > 0, (l2 * LN2).astype(np.float32), np.float32(-np.inf)).astype(np.float32)
    lse = np.repeat(lse[:, None, :], cnt.shape[2] * G, axis=1)
    return o, lse


def lse_partial_bounds(ns_, Hq):
    """[lo, hi] of every partial lse [n, Hq, R] of the key census (oracle.softmax.lse_bounds at m_raw = 0, c = 1)"""
    import torch

    from oracle import softmax as sm

    l = torch.from_numpy(ns_.reshape(-1).astype(np.float64))
    lo, hi = sm.lse_bounds(torch.zeros_like(l), l, 1.0)
    shape = ns_.shape
    lo, hi = lo.numpy().reshape(shape), hi.numpy().reshape(shape)
    return np.repeat(lo[:, None], Hq, axis=1), np.repeat(hi[:, None], Hq, axis=1)


# --------------------------------------------------------------------------------------------
# the merge: exact value, bound, fp32 emulation
# --------------------------------------------------------------------------------------------
def _lse_rows(lse):
    """[n, Hq, R] -> [n, R, Hq, 1] to broadcast against o"""
    return np.transpose(lse, (0, 2, 1))[..., None].astype(np.float64)


def bound(o_part, lse_part, sigma=None):
    """(y [R, Hq, D], beta [R, Hq, D], lse [Hq, R], beta_l [Hq, R]) of the merge of partials o_part [n, R, Hq, D],
    lse_part [n, Hq, R]; sigma [n, Hq, R] (optional) bounds an uncertainty of each lse_part.  Rows without a live
    split give y = 0, beta = 0 and lse = -inf."""
    x = o_part.astype(np.float64)
    lam = _lse_rows(lse_part)
    sg = np.zeros_like(lam) if sigma is None else _lse_rows(sigma)
    n = x.shape[0]
    live = np.isfinite(lam)
    any_live = live.any(0)
    m = np.where(any_live, np.where(live, lam, -np.inf).max(0), 0.0)
    d = np.where(live, lam - m, -np.inf)
    W = np.where(live, np.exp(d), 0.0)
    sg_m = np.where(live, sg, 0).max(0)
    r = np.where(live, np.exp(U * np.abs(np.where(live, d, 0)) + sg + sg_m) * (1 + EXPF_ULP * 2 * U) - 1, 0.0)
    # below the smallest normal expf's ulp error is absolute: w_s anywhere in [0, W_s (1 + r_s)] with
    # W_s r_s = W_s + EXPF_ULP 2^-149
    tiny = live & (W * np.exp(sg + sg_m) < 2.0 ** -125)
    r = np.where(tiny, 1 + EXPF_ULP * 2.0 ** -149 / np.where(tiny, W, 1), r)
    Ws = np.where(any_live, W.sum(0), 1.0)
    xw = np.where(live, x, 0.0)
    y = (W * xw).sum(0) / Ws
    Wlo = (W * np.maximum(1 - r, 0)).sum(0)
    Wlo = np.where(any_live, Wlo, 1.0)
    e1 = (W * r * np.abs(xw - y)).sum(0) / Wlo
    g = n * U / (1 - n * U)
    Whi = (W * (1 + r)).sum(0)
    e2 = g * ((W * (1 + r) * np.abs(xw)).sum(0) + (np.abs(y) + e1) * Whi) / (Wlo * (1 - g))
    e3 = 2.01 * U * (np.abs(y) + e1 + e2)
    beta = np.where(any_live, 1.01 * (e1 + e2 + e3 + (n + 1) * 2.0 ** -150), 0.0)
    y = np.where(any_live, y, 0.0)
    # lse, per (row, head): take column 0 of the broadcast axes
    rw = (W * r).sum(0) / Ws  # the weights' relative error on den
    eta = (rw + g * (1 + rw))[..., 0]
    etap = -np.log1p(-eta)
    lnW = np.log(Ws[..., 0])
    mm = m[..., 0]
    lse = np.where(any_live[..., 0], mm + lnW, -np.inf)
    beta_l = 1.01 * (etap + 2 * LOGF_ULP * U * (np.abs(lnW) + etap) + U * (np.abs(mm + lnW) + etap) + sg_m[..., 0])
    beta_l = np.where(any_live[..., 0], beta_l, 0.0)
    return y, beta, lse.T, beta_l.T


def _ulps(x, k):
    """x (fp32 array) moved by k ulps (k integer array of the same shape)"""
    out = x.copy()
    for step in range(int(np.abs(k).max(initial=0))):
        up = k > step
        dn = -k > step
        out = np.where(up, np.nextafter(out, np.float32(np.inf)), out)
        out = np.where(dn, np.nextafter(out, np.float32(-np.inf)), out)
    return out.astype(np.float32)


def merge_fp32(o_part, lse_part, rng=None, mutation=None, Hq=None):
    """The merge of kv_split_merge_kernel in fp32 (o unrounded [R, Hq, D] fp32, lse [Hq, R] fp32), for checking the
    bound: it is not bit-exact.  Each fmaf is an exact fp64 product plus an fp64 add, then a round to fp32, so it may
    round twice (a further 2^-53 relative, inside the bound's factor 1.01), and expf / logf are numpy's.  rng: move
    every expf result by up to EXPF_ULP ulps and every logf result by up to LOGF_ULP, at random.  mutation: one of
    the merge MUTATIONS."""
    n = o_part.shape[0]
    lam = np.transpose(lse_part, (0, 2, 1)).astype(np.float32)  # [n, R, Hq]
    x = o_part.astype(np.float32)
    if mutation == "neighbour_head":
        lam, x = np.roll(lam, -1, axis=2), np.roll(x, -1, axis=2)
    if mutation == "neighbour_row":
        lam, x = np.roll(lam, -1, axis=1), np.roll(x, -1, axis=1)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        m = lam.max(0) if mutation != "m_split0" else lam[0].copy()
        if mutation == "m_split0":
            m = np.where(np.isfinite(lam).any(0) & (lam[0] == -np.inf), np.float32(-np.inf), m)
        if mutation == "m_first_live":
            first = np.isfinite(lam).argmax(0)
            m = np.take_along_axis(lam, first[None], 0)[0]
        if mutation == "no_max":
            m = np.where(np.isfinite(lam).any(0), np.float32(0), np.float32(-np.inf))
        acc = np.zeros(x.shape[1:], dtype=np.float32)
        den = np.zeros(lam.shape[1:], dtype=np.float32)
        for s in range(n):
            l = lam[s]
            dd = (l - m).astype(np.float32)
            if mutation == "exp2_weights":
                w = np.exp2(dd.astype(np.float64)).astype(np.float32)
            else:
                w = np.exp(dd.astype(np.float64)).astype(np.float32)
            if rng is not None:
                w = np.maximum(_ulps(w, rng.integers(-EXPF_ULP, EXPF_ULP + 1, size=w.shape)), np.float32(0))
            if mutation == "equal_weights":
                w = np.ones_like(w)
            dead = l == -np.inf
            if mutation == "ninf_weight1":
                w = np.where(dead, np.float32(1), w)
                xs = np.where(dead[..., None], np.float32(0), x[s])
            else:
                w = np.where(dead, np.float32(0), w)
                xs = x[s]
            acc = (w[..., None].astype(np.float64) * xs + acc).astype(np.float32)
            den = (den + w).astype(np.float32)
        if mutation == "nokey_nan":
            inv = (np.float32(1) / den).astype(np.float32)
        else:
            inv = np.where(den > 0, (np.float32(1) / np.where(den > 0, den, 1)).astype(np.float32), np.float32(0))
        o = (acc * inv[..., None]).astype(np.float32)
        lg = np.log(np.where(den > 0, den, 1).astype(np.float64)).astype(np.float32)
        if rng is not None:
            lg = _ulps(lg, rng.integers(-LOGF_ULP, LOGF_ULP + 1, size=lg.shape))
        base = np.float32(0) if mutation in ("lse_without_m", "no_max") else m
        lse = np.where(den > 0, (base + lg).astype(np.float32), np.float32(-np.inf))
    return o, lse.T.astype(np.float32)


def round16(x, dtype):
    """x (float array) rounded to the 16-bit output format, as float64 values"""
    import torch

    return torch.from_numpy(np.asarray(x, dtype=np.float32)).to(dtype).double().numpy()


def admissible(o16, y, beta, dtype):
    """o16 (the kernel's 16-bit o as float64) is round16(x) for some x in [y - beta, y + beta]"""
    lo, hi = round16(y - beta, dtype), round16(y + beta, dtype)
    return (o16 >= lo) & (o16 <= hi)


def lse_count_margin(N_max):
    """ln((N + 1) / N) at N = N_max: the lse step between two neighbouring counts"""
    return math.log1p(1.0 / N_max)


# --------------------------------------------------------------------------------------------
# the flow with one mutation
# --------------------------------------------------------------------------------------------
EPILOGUE = ("slot_plus1", "slot_minus1", "lse_head_stride")
RULE = ("piece_floor", "piece_over_kept", "piece_end_plus1", "piece_end_minus1", "sinks_last")


def simulate(case, n, mutation=None):
    """(lists, o_part [n, R, Hq, D], lse_part [n, Hq, R], o [R, Hq, D] fp32 before the 16-bit rounding, lse [Hq, R])
    of the key census of `case` at n splits, with one MUTATION.  Partials a mutated epilogue leaves unwritten are NaN
    (the tests fill the workspace with NaN)."""
    assert mutation is None or mutation in MUTATIONS, mutation
    rule = mutation if mutation in RULE else None
    lists = plan_lists(case, n, rule)
    ns_, cnt, _ = key_census(case, n, rule)
    o_p, l_p = partials_fp32(ns_, cnt, case.G)
    if mutation in ("slot_plus1", "slot_minus1"):
        wo, wl = np.full_like(o_p, np.nan), np.full_like(l_p, np.nan)
        for s in range(n):
            t = min(s + 1, n - 1) if mutation == "slot_plus1" else max(s - 1, 0)
            wo[t], wl[t] = o_p[s], l_p[s]
        o_p, l_p = wo, wl
    if mutation == "lse_head_stride":
        Hq, R = l_p.shape[1:]
        buf = np.full((n * Hq + Hq) * R, np.nan, dtype=np.float32)
        for s in range(n):
            for h in range(Hq):
                buf[(s + h) * R:(s + h + 1) * R] = l_p[s, h]
        l_p = buf[:n * Hq * R].reshape(n, Hq, R)
    merge_mut = mutation if mutation not in RULE + EPILOGUE else None
    o, lse = merge_fp32(o_p, l_p, mutation=merge_mut)
    return lists, o_p, l_p, o, lse


# --------------------------------------------------------------------------------------------
# softmax census per split (one stream, Sq = L = S: plan rows and keys in logical order)
# --------------------------------------------------------------------------------------------
def split_owner(S, mask, n, mutation=None):
    """[items, chunks] int: the split that holds chunk j for item k of a stream of S queries over its S keys, -1 none"""
    items, nch = -(-S // ITEM_ROWS), -(-S // CHUNK)
    owner = np.full((items, nch), -1, dtype=np.int64)
    for k in range(items):
        for s, lst in enumerate(split_lists(S, S, k, mask, n, mutation)):
            for j, _ in lst:
                owner[k, j] = s
    return owner


def split_softmax_cases(base, mask, n):
    """per split s: base (an oracle.softmax Case in logical order) whose mod is `mask` restricted to split s's chunks"""
    import torch

    S = base.S
    owner = split_owner(S, mask, n)

    def mod_for(s):
        def mod(q_idx, kv_idx):
            p = q_idx.cpu().numpy().reshape(-1).astype(np.int64)
            kv = kv_idx.cpu().numpy().reshape(-1).astype(np.int64)
            a1, b0, b1 = mask.row_sets(p, S)
            m = (kv[None] < a1[:, None]) | ((kv[None] >= b0[:, None]) & (kv[None] < b1[:, None]))
            m &= owner[p // ITEM_ROWS][:, kv // CHUNK] == s
            return torch.from_numpy(m).to(q_idx.device)
        return mod

    return [dataclasses.replace(base, name=f"{base.name}_s{s}", mod=mod_for(s)) for s in range(n)]


def softmax_partials(base, mask, n):
    """Closed form of the split partials of the softmax census: (o [n, S, H, D] fp32 bit for bit, lse lo / hi
    [n, H, S] (lse_bounds), lse [n, H, S] fp32 with a correctly rounded log2f, largest per-split budget)"""
    import torch

    from oracle import softmax as sm

    S, H, D = base.S, base.H, base.D
    o = np.zeros((n, S, H, D), dtype=np.float32)
    lo, hi, lse = (np.zeros((n, H, S)) for _ in range(3))
    budget = 0.0
    for s, cs in enumerate(split_softmax_cases(base, mask, n)):
        for h in range(H):
            O, l, m_raw, bud = sm.expected(cs, h)
            budget = max(budget, float(bud.max()))
            o[s, :, h] = sm.expected_output(O, l, cs.vs[h], torch.float32).numpy()
            a, b = sm.lse_bounds(m_raw, l, cs.c[h])
            lo[s, h], hi[s, h] = a.numpy(), b.numpy()
            live = l.numpy() > 0
            mc = np.where(live, m_raw.numpy(), 0).astype(np.float32) * np.float32(cs.c[h])
            L2 = np.log2(np.where(live, l.numpy(), 1.0)).astype(np.float32)
            lse[s, h] = np.where(live, ((mc + L2).astype(np.float32) * LN2).astype(np.float32), -np.inf)
    return o, lo, hi, lse.astype(np.float32), budget
