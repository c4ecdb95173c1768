"""Exact census of the key set an attention kernel executes.  TEST INFRASTRUCTURE ONLY.

With q = 0 every allowed score is exactly 0 and every masked one is -inf, so every allowed key gets p = 1 and

    l_i      = n_i = number of keys row i may see            ->  lse_i = ln(n_i)
    o[i, d]  = round16(fp32(cnt_{i,d}) * fp32(1 / n_i))

when V is a one-hot KEY-IDENTITY ENCODING, V[j, d] = [code(j) == d], and cnt_{i,d} counts the allowed keys of row
i whose code is d.  Every term is an integer (p = 1, V in {0, 1}), so the accumulation is exact and the output can be
compared bit for bit.  Two encodings are used, code_0(j) = j mod D and code_1(j) = (j div D) mod D: a key wrongly
kept or dropped moves n_i and one count of each encoding by one, and two keys can only be swapped unnoticed when they
agree modulo D^2.

The expected tables come from the oracle's mask definitions (oracle.attention), never from the engine:
  band masks : the *_mask_mod predicates, evaluated in row chunks (any torch device; integer-exact),
  block maps : cnt[i, d] = sum_j map[qb(i), j] * C[j, d], C[j, d] = keys of key block j with code d.

How far apart the counts stay after rounding is a property of the output format and of n alone; see
`distinguishable_limit`.
"""
from __future__ import annotations

import math

import numpy as np
import torch

ENCODINGS = (0, 1)
# largest sequence length the census runs at (HunyuanVideo 720p) and, per output format, the first count c for which
# round(c / n) == round((c + 1) / n) at some n <= N_MAX (distinguishable_limit; checked on the CPU)
N_MAX = 119056
COUNT_LIMIT = {torch.float16: 1032, torch.bfloat16: 129}


def key_codes(S: int, D: int, enc: int, device=None) -> torch.Tensor:
    """code_enc(j) for j < S (int64)."""
    j = torch.arange(S, device=device)
    return j % D if enc == 0 else (j // D) % D


def column_bound(S: int, D: int, enc: int) -> int:
    """Largest number of keys j < S that share one code: no count of the table can exceed it, whatever the mask."""
    return int(torch.bincount(key_codes(S, D, enc), minlength=D).max())


def identity_values(S: int, D: int, enc: int, H: int, dtype, device, codes: torch.Tensor | None = None):
    """[1, H, S, D] one-hot V with V[0, h, j, code(j)] = 1; `codes` overrides the per-row codes ([S] or [H, S])."""
    c = key_codes(S, D, enc, device) if codes is None else codes.to(device)
    c = c.expand(H, S)
    v = torch.zeros(H, S, D, dtype=torch.float32, device=device)
    v.scatter_(2, c[:, :, None], 1.0)
    return v.to(dtype)[None]


def _onehot_both(codes0: torch.Tensor, codes1: torch.Tensor, D: int, dtype) -> torch.Tensor:
    S = codes0.shape[0]
    e = torch.zeros(S, 2 * D, dtype=dtype, device=codes0.device)
    e[torch.arange(S, device=codes0.device), codes0] = 1
    e[torch.arange(S, device=codes0.device), D + codes1] = 1
    return e


def band_census(mod, S: int, D: int, device, row_chunk: int = 1024, *, Skv: int | None = None):
    """Census tables of an element mask predicate mod(q_idx [R,1], kv_idx [1,Skv]) -> bool [R,Skv] over rows 0..S-1
    and keys 0..Skv-1 (Skv None: S), the key codes taken over the Skv keys.
    Returns cnt int32 [2, S, D] (both encodings, row order) and n int64 [S] on `device`.

    The counts are formed by a 0/1 matmul; every partial sum is an integer no larger than the final count, which
    `column_bound` keeps below 2^11, so fp16 (GPU) or fp32 (CPU) arithmetic is exact."""
    dev = torch.device(device)
    K = S if Skv is None else Skv
    mm_dtype = torch.float16 if dev.type == "cuda" else torch.float32
    for enc in ENCODINGS:
        assert column_bound(K, D, enc) < 2048
    e = _onehot_both(key_codes(K, D, 0, dev), key_codes(K, D, 1, dev), D, mm_dtype)
    kv = torch.arange(K, device=dev, dtype=torch.int32).view(1, K)
    cnt = torch.empty(2, S, D, dtype=torch.int32, device=dev)
    n = torch.empty(S, dtype=torch.int64, device=dev)
    for r0 in range(0, S, row_chunk):
        r1 = min(S, r0 + row_chunk)
        m = mod(torch.arange(r0, r1, device=dev, dtype=torch.int32).view(-1, 1), kv)
        n[r0:r1] = m.sum(1)
        c = (m.to(mm_dtype) @ e).to(torch.int32)
        cnt[0, r0:r1] = c[:, :D]
        cnt[1, r0:r1] = c[:, D:]
    return cnt, n


def blockmap_census(block_map: torch.Tensor, row_sz: torch.Tensor, col_sz: torch.Tensor, D: int,
                    key_ids: torch.Tensor | None = None, *, Skv: int | None = None):
    """Census tables of a variable-block map (dynamic_block_sparse_fwd semantics, one head) in PLAN row order.
    block_map [QC, KC], row_sz [QC], col_sz [KC]; key_ids [Skv] (optional): the key identity (the row of V) read at
    each plan key position, e.g. the kv_rows gather or the k-cluster argsort.  Runs in fp64 on the CPU.
    Skv None: a square map, the row and column sizes both sum to S; otherwise the row sizes sum to Sq and the column
    sizes to Skv, and the key codes are taken over the Skv keys.
    Returns cnt int64 [2, Sq, D], n int64 [Sq]."""
    bm = block_map.cpu().to(torch.float64)
    rs, cs = row_sz.cpu().long(), col_sz.cpu().long()
    S = int(cs.sum())
    assert int(rs.sum()) == S if Skv is None else S == Skv
    ids = torch.arange(S) if key_ids is None else key_ids.cpu().long()
    e = _onehot_both(key_codes(S, D, 0)[ids], key_codes(S, D, 1)[ids], D, torch.float64)
    kb = torch.repeat_interleave(torch.arange(cs.numel()), cs)
    per_block = torch.zeros(cs.numel(), 2 * D, dtype=torch.float64).index_add_(0, kb, e)
    cnt_qb = (bm @ per_block).round().long()
    n_qb = (bm @ cs.double()).round().long()
    qb = torch.repeat_interleave(torch.arange(rs.numel()), rs)
    c = cnt_qb[qb]
    return torch.stack([c[:, :D], c[:, D:]]), n_qb[qb]


def rect_census(bm: torch.Tensor, rows: torch.Tensor, cols: torch.Tensor, D: int):
    """blockmap_census of a rectangular map: cnt int64 [2, Sq, D] (keys of each query row with each code, both
    encodings) and n int64 [Sq] of one head's map [QC, KC], row sizes [QC] (sum Sq), column sizes [KC] (sum Skv)."""
    return blockmap_census(bm, rows, cols, D, Skv=int(cols.cpu().long().sum()))


def scatter_rows(cnt: torch.Tensor, n: torch.Tensor, o_rows: torch.Tensor | None):
    """Plan-row tables -> output-row tables under the fused row scatter (output row o_rows[r] holds plan row r)."""
    if o_rows is None:
        return cnt, n
    idx = o_rows.cpu().long()
    c2, n2 = torch.empty_like(cnt), torch.empty_like(n)
    c2[:, idx] = cnt.cpu()
    n2[idx] = n.cpu()
    return c2, n2


def expected_output(cnt: torch.Tensor, n: torch.Tensor, out_dtype) -> torch.Tensor:
    """round16(fp32(cnt) * fp32(1/n)), 0 for rows without keys: the kernel's epilogue O * (1/l) with O = cnt, l = n.
    cnt [S, D] (one encoding), n [S]; computed on the CPU (IEEE division)."""
    nf = n.cpu().to(torch.float32)
    inv = torch.where(nf > 0, torch.reciprocal(nf), torch.zeros_like(nf))
    return (cnt.cpu().to(torch.float32) * inv[:, None]).to(out_dtype)


def distinguishable_limit(n_max: int, out_dtype, c_max: int = 4096) -> int:
    """Largest C such that for every n <= n_max and every count c < C with c + 1 <= n,
    round(c / n) != round((c + 1) / n) in `out_dtype` (with the kernel's fp32 reciprocal-and-multiply): a table
    whose counts stay <= C - 1 shows every count move of +-1."""
    ns = np.arange(1, n_max + 1, dtype=np.float32)
    inv = torch.from_numpy((np.float32(1) / ns).astype(np.float32))
    prev = (torch.zeros_like(inv)).to(out_dtype)
    for c in range(0, c_max):
        nxt = (inv * np.float32(c + 1)).to(out_dtype)
        live = torch.from_numpy(ns >= c + 1)
        if bool(((prev == nxt) & live).any()):
            return c
        prev = nxt
    return c_max


# --------------------------------------------------------------------------------------------
# plan shapes that hit the edges of the plan builders (shared by the census and the softmax census)
# --------------------------------------------------------------------------------------------
def band_args(kind, F, P, ctx, plen, mul, attn_sink=False):
    """((mask_mode, m0, m1, m2) of svgb200.core.plan_band, oracle mask predicate) of an SVG1 band mask:
    "hy" HunyuanVideo (text last), "wan" (first-frame sink), otherwise CogVideoX (text first, optional sink)."""
    from oracle import attention as oa

    if kind == "hy":
        return (1, F * P, F * P + plen, oa.hy_band_width(mul, P)), oa.hy_mask_mod(ctx, plen, F, P, mul)
    if kind == "wan":
        return (2, P, 0, oa.wan_band_width(mul, P)), oa.wan_mask_mod(F, P, mul)
    first = plen + P if attn_sink else plen
    return (3, first, plen, oa.hy_band_width(mul, P)), oa.cog_mask_mod(plen, F, P, mul, attn_sink)


def partition(total, n, gen):
    """n positive sizes summing to total (random cuts)"""
    cuts = torch.sort(torch.randperm(total - 1, generator=gen)[: n - 1] + 1)[0]
    return torch.diff(torch.cat([torch.tensor([0]), cuts, torch.tensor([total])]))


def _tails(sizes):
    return sum(1 for r in sizes.tolist() if 0 < r % 256 <= 128)


def q_sizes(total, n, gen, extra=()):
    """q-block sizes that hit every class of r % 256 (0, 1..128, 129..255), empty q-blocks, and an odd number of
    tails (one dual item then runs a single tail) counting the `extra` blocks appended after them"""
    special = torch.tensor([0, 0, 1, 17, 128, 129, 200, 255, 256, 257, 384, 385, 511, 512, 513, 640, 767, 768])
    for _ in range(64):
        s = torch.cat([special, partition(total - int(special.sum()), n - special.numel(), gen)])
        s = torch.cat([s[torch.randperm(n, generator=gen)], torch.tensor(extra, dtype=s.dtype)])
        if _tails(s) % 2 == 1:
            return s
    raise AssertionError("no odd tail count")


def varblock_head(kind, QC, KC, total, gen):
    """(map [QC, KC], col sizes [KC]) built to hit one edge of the plan builder"""
    if kind == "alternating":
        # every other key block selected: the most runs per row; selected blocks of 129 keys end in a 1-column
        # chunk, so the chunk count approaches the list capacity S/128 + (KC+1)/2 + 2
        col = torch.empty(KC, dtype=torch.long)
        col[0::2] = 129
        col[1::2] = partition(total - 129 * ((KC + 1) // 2), KC // 2, gen)
        bm = torch.zeros(QC, KC, dtype=torch.bool)
        bm[:, 0::2] = True
        return bm, col
    if kind == "joined":
        # every third key block is empty: selected blocks on both sides of an empty one form one run
        col = torch.zeros(KC, dtype=torch.long)
        live = torch.arange(KC) % 3 != 1
        col[live] = partition(total, int(live.sum()), gen)
        bm = torch.rand(QC, KC, generator=gen) < 0.6
        bm[:, ::3] = True
        bm[3, :] = True    # all selected
        bm[4, :] = False   # none selected
        return bm, col
    # random map, density 0.3, some empty key clusters
    col = partition(total, KC, gen)
    empty = torch.randperm(KC, generator=gen)[: KC // 20]
    col[empty[1:]] = 0
    col[empty[0]] += total - int(col.sum())
    bm = torch.rand(QC, KC, generator=gen) < 0.3
    return bm, col


def lse_count_error(n_max: int) -> float:
    """Worst |exp(lse) - n| over n <= n_max when the kernel's lse = fp32(fp32(log2 n) * fp32(ln 2)) and its log2 is
    off by one ulp either way (fp64 exp).  Below 0.5, the lse identifies n exactly."""
    n = np.arange(1, n_max + 1, dtype=np.float64)
    l2 = np.log2(n).astype(np.float32)
    worst = 0.0
    for l2e in (np.nextafter(l2, np.float32(-np.inf)), l2, np.nextafter(l2, np.float32(np.inf))):
        lse = (l2e.astype(np.float32) * np.float32(math.log(2))).astype(np.float32)
        worst = max(worst, float(np.abs(np.exp(lse.astype(np.float64)) - n).max()))
    return worst
