"""Exact censuses of the attention backward (svgb_attn_bwd).  TEST INFRASTRUCTURE ONLY.

attn_bwd reads lse, o and do as inputs and forms P = exp2(s c - lse log2 e) and delta = rowsum(dO O) from them, so a
census chooses those inputs directly instead of taking them from a forward run.  Two censuses:

KEY CENSUS (which (query, key) pairs each gradient sums).  D' = D / 2 and code(i) a key-identity code over D' values
(oracle.census, encodings i mod D' and (i div D') mod D').  With
    Q_i = e_code(i) on [0, D'),  K_j = e_(D' + code(j)) on [D', D)   (disjoint supports: every score is exactly 0)
    V = 1,  dO_i = e_code(i)   (dP = 1),   O_i = delta(code(i)) e_code(i)   (delta_i = delta(code(i)) in {0, 2})
    lse_i = L(code(i)) ln 2 as the fp32 value whose fp32(lse * fp32(log2 e)) is exactly L = code mod 2 (-inf: no key)
    sm_scale = 1/2
every P is 2^-L and every dS is +-2^-L, so with cnt the forward census table (allowed keys of row i with code d) and
cnt_t the transposed one (rows i that reach key j with code(i) = d)
    dQ_i[D' + d] = 1/2 2^-L_i (1 - delta_i) cnt[i, d]        dQ_i[:D'] = 0
    dK_j[d]      = 1/2 2^-L(d) (1 - delta(d)) cnt_t[j, d]    dK_j[D':] = 0
    dV_j[d]      = 2^-L(d) cnt_t[j, d]                       dV_j[D':] = 0
(every row feeding column d of dK / dV has code d).  All of these are integers times powers of two; while they are
representable in the output format (`key_counts_representable`), one key wrongly kept or dropped changes stored bits.

GRADIENT CENSUS (the arithmetic on real scores and values).  Small integers with every intermediate exact:
    Q_i = b e_(D-1) + sparse integers on a column set A,  K_j = t_j e_(D-1) + sparse integers on the complement B of A
    in [0, D-1) (A and B swap between heads), so c s_ij = e t_j with e = b c an integer (oracle.softmax.qk_ints);
    lse_i = L_i ln 2 with L_i in {2, 3} per row and e t_j in [0, 2], so every exponent e t_j - L_i is in [-3, 0], the
    range where ex2.approx is exact (the softmax census's premise (a)) and P in {1/8, .., 1};
    V in [-2, 2]; dO_i = +-1 and O_i in [-2, 2] on the same two columns, so |dP - delta| <= 8 and dS is exact in bf16.
Every gradient element is then a sum of multiples of 1/8 whose absolute sum stays below 2^24 granules (`budget`), so
the fp32 accumulators are exact in any order and the stored values are round16(fp32(acc) * fp32(sm_scale)) for dQ
and dK and round16(acc) for dV.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import numpy as np
import torch

from oracle import census as oc
from oracle import softmax as osm

KEY_SCALE = 0.5          # sm_scale of the key census (exact power of two)
GRANULE = 8              # dS and P are multiples of 1/8 in the gradient census
BUDGET = 1 << 24
MAX_COUNT = {torch.float16: 2047, torch.bfloat16: 256}  # counts c with c * 2^k exact for every factor of the census


def lse_for(L: int) -> float:
    """The fp32 lse (as a Python float) whose fp32(lse * fp32(log2 e)) is exactly L (the kernel's bwd_lse2)."""
    x = np.float32(L * math.log(2))
    for _ in range(16):
        got = np.float32(x * osm.LOG2E)
        if got == np.float32(L):
            return float(x)
        x = np.nextafter(x, np.float32(np.inf if got < L else -np.inf))
    raise AssertionError(f"no fp32 lse gives log2 = {L}")


# --------------------------------------------------------------------------------------------
# key census
# --------------------------------------------------------------------------------------------
def code_L(code):
    return code % 2


def code_delta(code):
    return 2 * ((code >> 1) & 1)


def key_inputs(S: int, D: int, enc: int, n_rows: torch.Tensor):
    """Q, K, V, O, dO [BH, S, D] (float32, exact in bf16 / fp16) and lse [BH, S] of the key census, encoding enc;
    n_rows [BH, S]: allowed keys per query row (rows without keys get lse = -inf)."""
    Dh = D // 2
    BH = n_rows.shape[0]
    code = oc.key_codes(S, Dh, enc)
    r = torch.arange(S)
    q = torch.zeros(S, D)
    q[r, code] = 1
    k = torch.zeros(S, D)
    k[r, Dh + code] = 1
    o = torch.zeros(S, D)
    o[r, code] = code_delta(code).float()
    lse_l = torch.tensor([lse_for(0), lse_for(1)], dtype=torch.float32)[code_L(code)]
    lse = torch.where(n_rows.cpu() > 0, lse_l.expand(BH, S), torch.tensor(-math.inf))
    ex = lambda t: t.expand(BH, S, D)  # noqa: E731
    return ex(q), ex(k), ex(torch.ones(S, D)), ex(o), ex(q), lse.contiguous()


def key_expected(cnt: torch.Tensor, cnt_t: torch.Tensor, S: int, D: int, enc: int, *, Skv: int | None = None):
    """Closed form of one head (fp64): cnt [S, D'] forward table and cnt_t [Skv, D'] transposed table of encoding enc
    (Skv None: S) -> dq [S, D], dk, dv [Skv, D]."""
    Dh = D // 2
    K = S if Skv is None else Skv
    code = oc.key_codes(S, Dh, enc)
    d = torch.arange(Dh)
    f_row = 0.5 * torch.exp2(-code_L(code).double()) * (1 - code_delta(code)).double()
    f_k = 0.5 * torch.exp2(-code_L(d).double()) * (1 - code_delta(d)).double()
    f_v = torch.exp2(-code_L(d).double())
    dq = torch.zeros(S, D, dtype=torch.float64)
    dk, dv = (torch.zeros(K, D, dtype=torch.float64) for _ in range(2))
    dq[:, Dh:] = f_row[:, None] * cnt.cpu().double()
    dk[:, :Dh] = f_k[None] * cnt_t.cpu().double()
    dv[:, :Dh] = f_v[None] * cnt_t.cpu().double()
    return dq, dk, dv


def key_counts_representable(max_count: int, dtype) -> bool:
    """Every value the closed form can take for counts 0..max_count (count times 1/4, 1/2 or 1, either sign) is exact
    in dtype."""
    c = torch.arange(max_count + 1, dtype=torch.float64)
    vals = torch.cat([c * f for f in (0.25, -0.25, 0.5, -0.5, 1.0)])
    return bool((vals.to(dtype).double() == vals).all())


def band_tables(mod, S: int, D: int, device, *, Skv: int | None = None):
    """(cnt [2, S, D'], n [S], cnt_t [2, Skv, D']) of a band predicate mod(q_idx, kv_idx) over S queries and Skv keys
    (None: S), D' = D / 2.  The transposed table has a row per key and counts the queries by their codes over S."""
    K = S if Skv is None else Skv
    cnt, n = oc.band_census(mod, S, D // 2, device, Skv=K)
    cnt_t, _ = oc.band_census(lambda kk, qq: mod(qq, kk), K, D // 2, device, Skv=S)
    return cnt.cpu(), n.cpu(), cnt_t.cpu()


def blockmap_tables(bm, rows, cols, D: int, *, Skv: int | None = None):
    """The same tables of one head's block map: the transposed table is the census of the transposed map.  Skv: the
    column sizes sum to Skv and the row sizes to the query length (None: a square map)."""
    Sq = None if Skv is None else int(rows.cpu().long().sum())
    cnt, n = oc.blockmap_census(bm, rows, cols, D // 2, Skv=Skv)
    cnt_t, _ = oc.blockmap_census(bm.T, cols, rows, D // 2, Skv=Sq)
    return cnt, n, cnt_t


HY720 = dict(ctx=256, F=33, P=3600, plen=71)
WAN720 = dict(F=21, P=3600)
COG = dict(ctx=226, F=13, P=1350)


def key_band_case(kind, density=None):
    """((mode, m0, m1, m2), mask predicate, S) of the key census's band cases: the forward census's full-size list
    ("hy" 0.1 / 0.3 / "dense", "wan" 0.2 / 0.45, "wan_generic" W, "cog" / "cog_sink" 0.25) and its small list
    (a tuple as in test_census_band_small)."""
    from oracle import attention as oa

    if isinstance(kind, tuple):
        k = kind[0]
        if k.startswith("generic") or k == "none":
            mode = {"generic_hy": 1, "generic_wan": 2, "generic_cog": 3, "none": 0}[k]
            _, m0, m1, m2, S = kind
            return (mode, m0, m1, m2), oa.generic_mask_fn(mode, m0, m1, m2), S
        _, F, P, ctx, plen, mul = kind
        args, mod = oc.band_args(k, F, P, ctx, plen, mul)
        return args, mod, ctx + F * P
    if kind == "wan_generic":
        S, P = WAN720["F"] * WAN720["P"], WAN720["P"]
        return (2, P, 0, density), oa.generic_mask_fn(2, P, 0, density), S
    if kind == "hy":
        c = HY720
        mul = 40.0 if density == "dense" else oa.sparsity_to_width(density, c["ctx"], c["F"], c["P"])
        args, mod = oc.band_args("hy", c["F"], c["P"], c["ctx"], c["plen"], mul)
        return args, mod, c["ctx"] + c["F"] * c["P"]
    if kind == "wan":
        c = WAN720
        args, mod = oc.band_args("wan", c["F"], c["P"], 0, 0, oa.sparsity_to_width(density, 0, c["F"], c["P"]))
        return args, mod, c["F"] * c["P"]
    c = COG
    mul = oa.sparsity_to_width(density, c["ctx"], c["F"], c["P"])
    args, mod = oc.band_args("cog", c["F"], c["P"], c["ctx"], c["ctx"], mul, attn_sink=kind == "cog_sink")
    return args, mod, c["ctx"] + c["F"] * c["P"]


KEY_BAND_FULL = [("hy", 0.1), ("hy", 0.3), ("hy", "dense"), ("wan", 0.2), ("wan", 0.45), ("wan_generic", 4990),
                 ("cog", 0.25), ("cog_sink", 0.25)]
KEY_BAND_SMALL = [
    ("hy", 6, 200, 48, 20, 1.4), ("hy", 5, 333, 64, 64, 0.9), ("wan", 7, 180, 0, 0, 1.2), ("cog", 4, 260, 40, 40, 1.1),
    ("generic_wan", 50, 0, 77, 1100), ("generic_hy", 900, 1000, 1, 1093), ("generic_cog", 3, 130, 129, 1031),
    ("generic_wan", 50, 0, 254, 1100), ("generic_hy", 900, 1000, 255, 1093), ("generic_cog", 3, 130, 255, 1031),
    ("none", 0, 0, 0, 1000)]


def varblock_fullsize(shape: str):
    """The maps of the forward census's full-size variable-block cases ("hunyuan": 3 heads, QC = 400 + 2, KC = 1000 + 2
    with the prompt / padding blocks; "wan": 2 heads, QC = 300, KC = 1000), with the column sizes drawn by q_sizes as
    well, so that the key-major plan (whose rows are the key blocks) meets every r % 256 class, empty blocks and tail
    pairing too.  Column 5 is selected by every q-block and column 6 by none.  -> (bm [H, QC, KC], rows, cols, S)."""
    g = torch.Generator().manual_seed(17 if shape == "hunyuan" else 18)
    if shape == "hunyuan":
        ctx, plen, V, QC, KC = HY720["ctx"], HY720["plen"], HY720["F"] * HY720["P"], 400, 1000
        kinds = ["alternating", "joined", "random"]
    else:
        ctx, plen, V, QC, KC = 0, 0, WAN720["F"] * WAN720["P"], 300, 1000
        kinds = ["alternating", "joined"]
    bms, rows, cols = [], [], []
    for kind in kinds:
        bm, _ = oc.varblock_head(kind, QC, KC, V, g)
        extra = (plen, ctx - plen) if ctx else ()
        row = oc.q_sizes(V, QC, g, extra)
        col = oc.q_sizes(V, KC, g, extra)
        if ctx:
            bm = torch.nn.functional.pad(bm, (0, 2, 0, 2), value=False)
            bm[-2, :-1] = True
            bm[:-1, -2] = True
            bm[-1, -1] = True
            if kind == "joined":
                bm[4, :] = False  # the all-empty row stays empty
        if kind == "alternating":  # "joined" has the all-selected and all-empty rows
            bm[:, 5] = True
            bm[:, 6] = False
        bms.append(bm)
        rows.append(row)
        cols.append(col)
    return torch.stack(bms), torch.stack(rows).int(), torch.stack(cols).int(), V + ctx


# --------------------------------------------------------------------------------------------
# plans read back from their workspace
# --------------------------------------------------------------------------------------------
def read_plan(plan, BH: int):
    """Per head: items int32 [n, 2, 4] (the stream descriptors {row0, nrows, list_off, list_len}) and the chunk store
    int32 [m, 2] (attn_common.cuh)."""
    d = plan.desc
    ws = plan.ws.cpu()

    def i32(off, n):
        return ws[off: off + 4 * n].clone().view(torch.int32)

    shared = d.items_stride == 0
    counts = i32(d.counts_off, 1 if shared else d.BH)
    slots = d.max_items if shared else d.items_stride * d.BH
    items = i32(d.items_off, 8 * slots).view(-1, 2, 4)
    chunks = i32(d.chunks_off, 2 * ((ws.numel() - d.chunks_off) // 8)).view(-1, 2)
    out = []
    for h in range(BH):
        if shared:
            out.append(items[: int(counts[0])])
        else:
            out.append(items[h * d.items_stride: h * d.items_stride + int(counts[h])])
    return out, chunks


def plan_stats(items: torch.Tensor) -> dict:
    """What an item list exercises: two-stream and one-stream items, an empty list beside a non-empty one in one
    item, and stream-0 lists of odd and of even length followed by a stream 1 (the barrier-phase bookkeeping)."""
    two = items[:, 1, 1] > 0
    l0, l1 = items[:, 0, 3], items[:, 1, 3]
    return dict(two=bool(two.any()), one=bool((~two).any()),
                empty_next=bool((two & ((l0 == 0) != (l1 == 0))).any()),
                odd=bool((two & (l0 % 2 == 1)).any()), even=bool((two & (l0 > 0) & (l0 % 2 == 0)).any()))


def band_t_lists(items: torch.Tensor, mod, S: int, device):
    """Per item of a key-major band plan, the list the mask predicate calls for: (query chunk ids, ELEM flags), the
    128-query chunks where one of the item's keys has an allowed query, ELEM where not every such pair is allowed."""
    nch = (S + 127) // 128
    pad = nch * 128 - S
    q = torch.arange(S, device=device, dtype=torch.int32).view(1, S)
    out = []
    for it in range(items.shape[0]):
        r0, n0 = items[it, 0, :2].tolist()
        keys = torch.arange(r0, r0 + n0 + int(items[it, 1, 1]), device=device, dtype=torch.int32).view(-1, 1)
        a = mod(q, keys)  # [keys, queries]: allowed(query, key)
        a_any = torch.nn.functional.pad(a.any(0), (0, pad), value=False).view(nch, 128).any(1)
        a_all = torch.nn.functional.pad(a.all(0), (0, pad), value=True).view(nch, 128).all(1)
        want = a_any.nonzero().flatten()
        out.append((want.cpu(), (~a_all[want]).cpu()))
    return out


def check_band_t_structure(items: torch.Tensor, chunks: torch.Tensor, mod, S: int, device):
    """A key-major band plan against the mask predicate: every key lies in exactly one stream; each item's list is
    exactly the 128-query chunks with an allowed (query, key) pair for one of the item's keys, ascending, with the
    right valid counts; ELEM is set exactly on the chunks where not every pair is allowed.  Returns a message for the
    first violation, or None."""
    cov = torch.zeros(S, dtype=torch.int32)
    for st in range(2):
        for r0, nr in items[:, st, :2].tolist():
            cov[r0: r0 + nr] += 1
    if not bool((cov == 1).all()):
        j = int((cov != 1).nonzero()[0])
        return f"key {j} lies in {int(cov[j])} streams"
    for it, (want, want_elem) in enumerate(band_t_lists(items, mod, S, device)):
        r0, n0, off, ln = items[it, 0].tolist()
        lst = chunks[off: off + ln]
        if ln != want.numel() or not torch.equal(lst[:, 0].long(), want * 128):
            return f"item {it} (keys from {r0}): list {lst[:, 0].tolist()[:8]}.. of {ln} chunks, expected " \
                   f"{(want * 128).tolist()[:8]}.. of {want.numel()}"
        elem = (lst[:, 1] & 256) != 0
        valid = ((lst[:, 1] & 255) + 1).long()
        want_valid = torch.clamp(S - want * 128, max=128)
        if not torch.equal(elem, want_elem) or not torch.equal(valid, want_valid):
            c = int(((elem != want_elem) | (valid != want_valid)).nonzero()[0])
            return f"item {it}: chunk {int(lst[c, 0])} ELEM {bool(elem[c])} valid {int(valid[c])}, expected ELEM " \
                   f"{bool(want_elem[c])} valid {int(want_valid[c])}"
    return None


def band_items(mode: int, m0: int, m1: int, S: int, transposed: bool):
    """(row0, nrows) of every item of a band plan in launch order, restated from the planner's segment rules: items
    never straddle a row-region boundary (HunyuanVideo: video | prompt | padding, text segments first; CogVideoX: the
    text prefix, key-major the first columns m0; Wan key-major: the sink keys)."""
    cuts = []
    if mode == 1:
        cuts = [m0, m1]
    elif mode == 3:
        cuts = [m0 if transposed else m1]
    elif mode == 2 and transposed:
        cuts = [m0]
    b = [0]
    for c in cuts:
        if 0 < c < S and b[-1] < c:
            b.append(c)
    b.append(S)
    segs = [(b[i], b[i + 1]) for i in range(len(b) - 1)]
    if mode == 1:
        segs = segs[::-1]
    return [(r, min(256, e - r)) for s, e in segs for r in range(s, e, 256)]


# --------------------------------------------------------------------------------------------
# gradient census
# --------------------------------------------------------------------------------------------
@dataclass
class GradCase:
    name: str
    S: int
    D: int
    H: int                       # heads (B * H of the call)
    c: float                     # c = fp32(sm_scale) * fp32(log2 e), an exact power of two
    q: torch.Tensor              # [H, S, D] float32 integers
    k: torch.Tensor              # [H, Skv, D]
    v: torch.Tensor              # [H, Skv, D]
    o: torch.Tensor              # [H, S, D]
    do: torch.Tensor             # [H, S, D]
    L: torch.Tensor              # [H, S] int, log2 of the lse of every row
    band: tuple | None = None    # (mode, m0, m1, m2)
    mod: object = None
    bm: torch.Tensor | None = None   # [H, QC, KC]
    rows: torch.Tensor | None = None
    cols: torch.Tensor | None = None
    notes: dict = field(default_factory=dict)
    Skv: int | None = None       # keys (None: S)

    @property
    def Sk(self) -> int:
        return self.S if self.Skv is None else self.Skv

    @property
    def sm_scale(self) -> float:
        return osm.scale_for(self.c)

    def mask(self, h: int, device="cpu") -> torch.Tensor:
        """bool [S, Skv] element mask of head h."""
        if self.mod is not None:
            return self.mod(torch.arange(self.S, device=device).view(-1, 1),
                            torch.arange(self.Sk, device=device).view(1, -1))
        from oracle.attention import block_mask_to_element_mask

        return block_mask_to_element_mask(self.bm[h], self.rows[h], self.cols[h]).to(device)

    def lse(self, device="cpu") -> torch.Tensor:
        """fp32 [H, S]: L ln 2 (exact in the kernel's log2 domain), -inf for rows without keys."""
        tab = torch.tensor([lse_for(2), lse_for(3)], dtype=torch.float32)
        out = tab[(self.L - 2).long()]
        for h in range(self.H):
            out[h][~self.mask(h).any(1)] = -math.inf
        return out.to(device)


def _grad_inputs(H, S, D, c, gen, *, Skv: int | None = None):
    """q, k, v, o, do, L of the gradient census: q, o, do, L over S rows, k, v over Skv (None: S)."""
    K = S if Skv is None else Skv
    a, b = osm.qk_ints(c)
    e = int(b * c)
    T = 2 // e                          # e t <= 2
    cols = torch.arange(D - 1)
    q = torch.zeros(H, S, D)
    k = torch.zeros(H, K, D)
    for h in range(H):
        A = cols[(cols % 2) == h % 2]
        B = cols[(cols % 2) != h % 2]
        mag = torch.randint(1, 3, (S, D), generator=gen) * (torch.randint(0, 2, (S, D), generator=gen) * 2 - 1)
        keep = torch.rand(S, D, generator=gen) < 0.25
        q[h][:, A] = (mag * keep)[:, A].float()
        mag = torch.randint(1, 3, (K, D), generator=gen) * (torch.randint(0, 2, (K, D), generator=gen) * 2 - 1)
        keep = torch.rand(K, D, generator=gen) < 0.25
        k[h][:, B] = (mag * keep)[:, B].float()
    q[:, :, D - 1] = float(b)
    k[:, :, D - 1] = torch.randint(0, T + 1, (H, K), generator=gen).float()
    v = torch.randint(-2, 3, (H, K, D), generator=gen).float()
    do = torch.zeros(H, S, D)
    o = torch.zeros(H, S, D)
    two = torch.stack([torch.randperm(D, generator=gen)[:2] for _ in range(H * S)]).view(H, S, 2)
    sign = (torch.randint(0, 2, (H, S, 2), generator=gen) * 2 - 1).float()
    do.scatter_(2, two, sign)
    o.scatter_(2, two, torch.randint(-2, 3, (H, S, 2), generator=gen).float())
    L = torch.randint(2, 4, (H, S), generator=gen)
    return q, k, v, o, do, L


# name -> (mask kind, parameters, S): S = 1, 64, 65 and 127 mod 128, so the last query chunk of a key-major list has
# valid = 1, 64 (one half), 65 (a one-column second half) and 127 columns
GRAD_BAND = {
    "hy": ("hy", (5, 200, 25, 20, 1.4), 25 + 5 * 200),          # 1025 = 8 * 128 + 1
    "wan": ("wan", (6, 160, 0, 0, 1.2), 6 * 160),               # 960 = 7 * 128 + 64
    "cog": ("cog", (4, 250, 89, 89, 1.1), 89 + 4 * 250),        # 1089 = 8 * 128 + 65
    "none": ("generic", (0, 0, 0, 0), 1151),                    # 1151 = 8 * 128 + 127
}


def grad_band_case(name, D=128, H=2, c=1.0, seed=0):
    from oracle import attention as oa

    kind, args, S = GRAD_BAND[name]
    if kind == "generic":
        band, mod = args, oa.generic_mask_fn(*args)
    else:
        band, mod = oc.band_args(kind, *args)
    g = torch.Generator().manual_seed(seed)
    return GradCase(f"band {name}", S, D, H, c, *_grad_inputs(H, S, D, c, g), band=band, mod=mod)


def grad_varblock_case(D=128, H=2, seed=1):
    """S = 6000, 24 q-blocks and 60 key blocks, both sized by q_sizes (every r % 256 class, empty blocks, an odd tail
    count); head 0 the "joined" map, other heads random maps of density 0.4.  Per head, the first non-empty q-block
    selects nothing (keyless rows), key block 9 is selected by every q-block, and one or two tail-sized key blocks by
    none (unreached keys; head 0's key-major plan then pairs an empty list with a non-empty one)."""
    g = torch.Generator().manual_seed(seed)
    S, QC, KC = 6000, 24, 60
    rows = torch.stack([oc.q_sizes(S, QC, g) for _ in range(H)]).int()
    cols = torch.stack([oc.q_sizes(S, KC, g) for _ in range(H)]).int()
    bms = []
    for h in range(H):
        if h == 0:
            bm, _ = oc.varblock_head("joined", QC, KC, S, g)
        else:
            bm = torch.rand(QC, KC, generator=g) < 0.4
        bm[:, 9] = True
        bm[int((rows[h] > 0).nonzero()[0]), :] = False
        # key blocks whose key-major list is empty: the first tail-sized one, and one more when that leaves an even
        # number of tails with a list, so that the pairing puts an empty list beside a non-empty one
        tails = [j for j in range(KC) if 0 < int(cols[h, j]) % 256 <= 128]
        bm[:, [j for j in tails if j != 9][0]] = False
        live = [j for j in tails if bool((bm[:, j] & (rows[h] > 0)).any())]
        if len(live) % 2 == 0:
            bm[:, [j for j in live if j != 9][-1]] = False
        bms.append(bm)
    return GradCase("varblock", S, D, H, 1.0, *_grad_inputs(H, S, D, 1.0, g), bm=torch.stack(bms), rows=rows,
                    cols=cols)


def grad_bsr_case(D=128, seed=3):
    """The reference's temporal BSR blocks (F = 8, P = 300) behind a 40-row text prefix, one plan for both heads."""
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
    case = GradCase("bsr", S, D, H, 1.0, *_grad_inputs(H, S, D, 1.0, g), bm=bm.expand(H, -1, -1).contiguous(),
                    rows=sz.expand(H, -1).contiguous(), cols=sz.expand(H, -1).contiguous())
    case.notes["indptr"] = torch.cat([torch.zeros(1, dtype=torch.long), keep.sum(1).cumsum(0)])
    case.notes["indices"] = keep.nonzero()[:, 1]
    case.notes["bsr"] = (F, P, text, Rb)
    return case


def grad_rect_case(name, S, Skv, D=128, H=2, c=1.0, seed=7, **mask):
    """A gradient-census case of S queries and Skv keys; `mask` holds mod= (a predicate over S x Skv, with band= its
    plan parameters) or bm=, rows=, cols= (a rectangular block map)."""
    g = torch.Generator().manual_seed(seed)
    return GradCase(name, S, D, H, c, *_grad_inputs(H, S, D, c, g, Skv=Skv), Skv=Skv, **mask)


MUTANTS = ("lse_next", "delta_next", "delta_64", "dk_no_scale", "dv_scale", "drop_pair")


def grad_exact(case: GradCase, h: int, device="cpu", mutant: str | None = None):
    """Exact fp64 accumulators acc_q [S, D], (acc_k, acc_v) [Skv, D] of head h before the epilogue, their budgets (largest
    sum of |terms| over an element, in granules of 1/8) and statistics.  mutant: one of MUTANTS (an oracle restating
    a wrong kernel) or None."""
    dev = torch.device(device)
    q, k, v, o, do = (t[h].to(dev, torch.float64) for t in (case.q, case.k, case.v, case.o, case.do))
    L = case.L[h].to(dev, torch.float64)
    A = case.mask(h, dev)
    if mutant == "drop_pair":  # the first allowed key of every row
        first = A.float().argmax(1)
        A = A.clone()
        A[torch.arange(case.S, device=dev), first] = False
    _, b = osm.qk_ints(case.c)
    e = b * case.c
    t = k[:, case.D - 1]
    if mutant == "lse_next":
        L = torch.cat([L[1:], L[-1:]])
    P = torch.where(A, torch.exp2(e * t[None, :] - L[:, None]), torch.zeros((), dtype=torch.float64, device=dev))
    prod = do * o
    delta = (prod[:, :64] if mutant == "delta_64" else prod).sum(1)
    if mutant == "delta_next":
        delta = torch.cat([delta[1:], delta[-1:]])
    dP = do @ v.T
    dS = P * (dP - delta[:, None])
    acc = (dS @ k, dS.T @ q, P.T @ do)
    budget = tuple(float(x.max()) * GRANULE for x in (dS.abs() @ k.abs(), dS.abs().T @ q.abs(), P.T @ do.abs()))
    stats = dict(allowed=int(A.sum()), ds_nonzero=int((dS != 0).sum()), keyless=int((~A.any(1)).sum()),
                 unreached=int((~A.any(0)).sum()), ds_max=float(dS.abs().max()),
                 ds_exact=bool((dS * GRANULE == (dS * GRANULE).round()).all()))
    return acc, budget, stats


def grad_expected(case: GradCase, h: int, dtype, device="cpu", mutant: str | None = None):
    """The stored gradients dq [S, D], (dk, dv) [Skv, D] in dtype: round16(fp32(acc) * fp32(sm_scale)) for dQ and dK,
    round16(acc) for dV (RNE at both roundings, as the kernel's fp32 multiply and cvt.rn)."""
    (aq, ak, av), _, _ = grad_exact(case, h, device, mutant)
    s = torch.tensor(case.sm_scale, dtype=torch.float32, device=aq.device)
    one = torch.ones((), dtype=torch.float32, device=aq.device)
    sk = one if mutant == "dk_no_scale" else s
    sv = s if mutant == "dv_scale" else one
    return tuple((a.to(torch.float32) * f).to(dtype) for a, f in ((aq, s), (ak, sk), (av, sv)))
