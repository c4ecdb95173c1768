"""Host mirror of the KV-cache plan (svgb_attn_plan_kvcache): the logical-position predicate, the clamping of lengths
and block indices, and the item and chunk lists the planner writes.  TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

ITEM_ROWS, CHUNK = 256, 128


def allowed(p: int, kv: int, sink: int, left: int, right: int) -> bool:
    """Query at logical position p sees logical key kv."""
    return kv < sink or (p - kv <= left and kv - p <= right)


def kv_len(cache_seqlen: int, new_len: int, cap: int) -> int:
    return min(max(cache_seqlen, 0) + new_len, cap)


def block_of(b, t, *, nblocks, block_rows, table=None, batch_idx=None):
    """Cache block of logical key t of stream b, clamped to [0, nblocks)."""
    if table is not None:
        blk = table[b][t // block_rows]
    else:
        blk = batch_idx[b] if batch_idx is not None else b
    return min(max(blk, 0), nblocks - 1)


def plan(seqlens, *, Sq, new_len, nblocks, block_rows, table=None, batch_idx=None, sink, left, right):
    """[(stream b, first packed row, rows, [(physical row, valid, elem, logical index j)])] in the planner's order, and
    the clamped lengths L_b.  Every chunk is classified from its pairs, not from the kernel's interval form."""
    cap = len(table[0]) * block_rows if table is not None else block_rows
    lens = [kv_len(s, new_len, cap) for s in seqlens]
    items = []
    for b, L in enumerate(lens):
        for r0 in range(0, Sq, ITEM_ROWS):
            nr = min(ITEM_ROWS, Sq - r0)
            chunks = []
            for j in range((L + CHUNK - 1) // CHUNK):
                c0, valid = j * CHUNK, min(CHUNK, L - j * CHUNK)
                pairs = [allowed(L - Sq + i, c0 + c, sink, left, right) for i in range(r0, r0 + nr) for c in range(valid)]
                if any(pairs):
                    blk = block_of(b, c0, nblocks=nblocks, block_rows=block_rows, table=table, batch_idx=batch_idx)
                    row = blk * block_rows + (c0 % block_rows if table is not None else c0)
                    chunks.append((row, valid, not all(pairs), j))
            items.append((b, b * Sq + r0, nr, chunks))
    return items, lens
