"""The local mask inside packed variable-length segments (svgb_attn_plan_local_varlen) restated on the host for the
tests: the bounds as the planner sanitises them, the predicate of the issue's semantics, and the items of both plans
in launch order with the kind of every chunk.  TEST INFRASTRUCTURE ONLY.  With one segment and equal lengths the mask
is the local band of tests/local_mask.py, which this module defers to for its predicate there."""
from __future__ import annotations

import torch

import local_mask as lm

ITEM, CHUNK = 256, 128


def sanitize(cu, total: int) -> list:
    """The planner's copy of one cu_seqlens: first bound 0, last bound total, the others clamped to [0, total] and made
    monotone by a running maximum."""
    cu = [int(x) for x in cu]
    n = len(cu) - 1
    out, run = [], 0
    for i, x in enumerate(cu):
        x = 0 if i == 0 else total if i == n else min(max(x, 0), total)
        run = max(run, x)
        out.append(run)
    return out


def mask_fn(cu_q, cu_k, sink: int, left: int, right: int):
    """allowed(q, kv) on index tensors, for sanitised bounds: same segment, and kj < sink or the band around
    qi + Lk_i - Lq_i (FlashAttention's bottom-right alignment).  One segment with equal lengths: local_mask_fn."""
    if len(cu_q) == 2 and cu_q == cu_k:
        return lm.local_mask_fn(sink, left, right)
    cq, ck = torch.tensor(cu_q), torch.tensor(cu_k)

    def mod(q_idx, kv_idx):
        q_idx, kv_idx = torch.as_tensor(q_idx).long(), torch.as_tensor(kv_idx).long()
        bq, bk = cq.to(q_idx.device), ck.to(q_idx.device)
        sq = torch.searchsorted(bq, q_idx.contiguous(), right=True) - 1  # last segment starting at or before q
        sk = torch.searchsorted(bk, kv_idx.contiguous(), right=True) - 1
        sq, sk = sq.clamp(max=len(cu_q) - 2), sk.clamp(max=len(cu_k) - 2)
        qi = q_idx - bq[sq]
        kj = kv_idx - bk[sk]
        p = qi + (bk[sq + 1] - bk[sq]) - (bq[sq + 1] - bq[sq])  # bottom-right alignment
        return (sq == sk) & ((kj < sink) | ((p - kj <= left) & (kj - p <= right)))

    return mod


def dense(cu_q, cu_k, sink, left, right) -> torch.Tensor:
    """bool [Sq, Skv] of the mask (sanitised bounds)."""
    q = torch.arange(cu_q[-1]).view(-1, 1)
    kv = torch.arange(cu_k[-1]).view(1, -1)
    return mask_fn(cu_q, cu_k, sink, left, right)(q, kv)


def items(cu_q, cu_k, sink, left, right, transposed: bool):
    """[(row0, nrows, [(col0, valid, elem)])] in launch order.  Rows are queries (transposed: keys) cut in 256 from the
    start of their segment, key-major with the sink keys of a segment as items of their own; chunks are the columns of
    the segment cut in 128 from its start, omitted when no pair of the item is allowed and ELEM unless all are.  Launch
    order: row order (segments in turn)."""
    m = dense(cu_q, cu_k, sink, left, right)
    if transposed:
        m = m.T
    rb, cb = (cu_k, cu_q) if transposed else (cu_q, cu_k)
    out = []
    for i in range(len(rb) - 1):
        rs, re, cs, ce = rb[i], rb[i + 1], cb[i], cb[i + 1]
        s = min(sink, re - rs) if transposed else 0
        cuts = [(a, min(a + ITEM, b)) for a, b in ((rs, rs + s), (rs + s, re)) for a in range(a, b, ITEM)]
        for r0, r1 in cuts:
            lst = []
            for c0 in range(cs, ce, CHUNK):
                blk = m[r0:r1, c0:min(c0 + CHUNK, ce)]
                if bool(blk.any()):
                    lst.append((c0, blk.shape[1], not bool(blk.all())))
            out.append((r0, r1 - r0, lst))
    return out
