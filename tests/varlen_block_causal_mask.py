"""The block-causal mask inside packed variable-length segments (svgb_attn_plan_block_varlen) restated on the host for
the tests: the predicate from the definition (blocks anchored at each segment's key 0, queries bottom-right aligned),
the items of both plans from a brute-force vote over that predicate, and the planners' interval forms written out
independently (query-major: rounded first and last rows on the local band; key-major: the interval of positions that
reach each key), so that each can be checked against the vote.  TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import torch

import block_causal_mask as bm

ITEM, CHUNK = 256, 128
NEG = -(1 << 62)  # "no lower bound"


def mask_fn(cu_q, cu_k, sink: int, block: int, first_block: int, window: int):
    """allowed(q, kv) on index tensors, for sanitised bounds: same segment, and kj < sink or e(p) - W <= kj < e(p) with
    p = qi + Lk_i - Lq_i and e the first block end F, F + C, ... past p, counted from the segment's key 0; window -1 is
    unbounded."""
    cq, ck = torch.tensor(cu_q), torch.tensor(cu_k)

    def mod(q_idx, kv_idx):
        q_idx, kv_idx = torch.as_tensor(q_idx).long(), torch.as_tensor(kv_idx).long()
        bq, bk = cq.to(q_idx.device), ck.to(q_idx.device)
        sq = torch.searchsorted(bq, q_idx.contiguous(), right=True) - 1  # last segment starting at or before q
        sk = torch.searchsorted(bk, kv_idx.contiguous(), right=True) - 1
        sq, sk = sq.clamp(max=len(cu_q) - 2), sk.clamp(max=len(cu_k) - 2)
        kj = kv_idx - bk[sk]
        p = (q_idx - bq[sq]) + (bk[sq + 1] - bk[sq]) - (bq[sq + 1] - bq[sq])
        e = bm.block_end(p, block, first_block)
        near = kj < e
        if window != -1:
            near = near & (kj >= e - window)
        return (sq == sk) & ((kj < sink) | near)

    return mod


def dense(cu_q, cu_k, sink, block, first_block, window) -> torch.Tensor:
    """bool [Sq, Skv] of the mask (sanitised bounds)."""
    q = torch.arange(cu_q[-1]).view(-1, 1)
    kv = torch.arange(cu_k[-1]).view(1, -1)
    return mask_fn(cu_q, cu_k, sink, block, first_block, window)(q, kv)


def item_rows(cu_q, cu_k, sink, transposed: bool):
    """[(segment, row0, nrows)] in launch order: rows cut in 256 from the start of their segment, key-major with the sink
    keys of a segment as items of their own."""
    rb = cu_k if transposed else cu_q
    out = []
    for i in range(len(rb) - 1):
        rs, re = rb[i], rb[i + 1]
        s = min(sink, re - rs) if transposed else 0
        out += [(i, a, min(a + ITEM, b) - a) for a, b in ((rs, rs + s), (rs + s, re)) for a in range(a, b, ITEM)]
    return out


def items(cu_q, cu_k, sink, block, first_block, window, transposed: bool):
    """[(row0, nrows, [(col0, valid, elem)])] in launch order, every chunk of the item's segment voted over the dense
    mask: omitted when no pair is allowed, ELEM unless all are."""
    m = dense(cu_q, cu_k, sink, block, first_block, window)
    if transposed:
        m = m.T
    cb = cu_q if transposed else cu_k
    out = []
    for i, r0, nr in item_rows(cu_q, cu_k, sink, transposed):
        lst = []
        for c0 in range(cb[i], cb[i + 1], CHUNK):
            blk = m[r0:r0 + nr, c0:min(c0 + CHUNK, cb[i + 1])]
            if bool(blk.any()):
                lst.append((c0, blk.shape[1], not bool(blk.all())))
        out.append((r0, nr, lst))
    return out


def block_last(p: int, block: int, first_block: int) -> int:
    return bm.block_end(p, block, first_block) - 1


def reach(k: int, block: int, first_block: int, W: int):
    """[lo, hi] of the positions p with k + 1 <= e(p) <= k + W (k >= 0 relative to the segment's key 0): lo the first
    position of k's block (NEG for k < F), hi one less than the last block end <= k + W."""
    C_, F = block, first_block
    lo = NEG if k < F else k - (k - F) % C_
    x = k + W
    return lo, x - (x - F) % C_ - 1


def chunk_kind(cu_q, cu_k, sink, block, first_block, W, transposed, seg, r0, r1, c0, c1) -> int:
    """0 / 1 / 2 of a chunk from the interval forms (W finite: the planner's value for an unbounded window)."""
    cq0, ck0 = cu_q[seg], cu_k[seg]
    off = (cu_k[seg + 1] - ck0) - (cu_q[seg + 1] - cq0)  # p = (q - cq0) + off
    if not transposed:
        # rows rounded to their block ends; keys c0..c1 relative; the local band (sink, W - 1, 0) on rounded rows
        e0 = block_last(r0 - cq0 + off, block, first_block)
        e1 = block_last(r1 - cq0 + off, block, first_block)
        k0, k1 = c0 - ck0, c1 - ck0
        any_ = k0 < sink or (k0 <= e1 and k1 >= e0 - (W - 1))
        ks = max(k0, sink)
        all_ = ks > k1 or (ks >= e1 - (W - 1) and k1 <= e0)
    else:
        k0, k1 = r0 - ck0, r1 - ck0
        p0, p1 = c0 - cq0 + off, c1 - cq0 + off
        ks = max(k0, sink)
        any_ = k0 < sink
        all_ = ks > k1
        if ks <= k1:
            a, b = reach(ks, block, first_block, W), reach(k1, block, first_block, W)
            any_ = any_ or (p0 <= b[1] and p1 >= a[0])
            all_ = p0 >= b[0] and p1 <= a[1]
    return 0 if not any_ else 1 if all_ else 2


def items_interval(cu_q, cu_k, sink, block, first_block, W, transposed: bool):
    """items() from the interval forms instead of the vote."""
    cb = cu_q if transposed else cu_k
    out = []
    for i, r0, nr in item_rows(cu_q, cu_k, sink, transposed):
        lst = []
        for c0 in range(cb[i], cb[i + 1], CHUNK):
            valid = min(CHUNK, cb[i + 1] - c0)
            kind = chunk_kind(cu_q, cu_k, sink, block, first_block, W, transposed, i, r0, r0 + nr - 1, c0,
                              c0 + valid - 1)
            if kind:
                lst.append((c0, valid, kind == 2))
        out.append((r0, nr, lst))
    return out
