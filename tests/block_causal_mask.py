"""The block-causal mask (SVGB_MASK_BLOCK_CAUSAL) restated on the host for the tests: its predicate from the definition,
the items of its band plans in launch order, and the KV-cache plan mirror under the block rule.  TEST INFRASTRUCTURE
ONLY.  The predicate is written from the block ends themselves, not from the engine's rounding, so that the two can be
compared."""
from __future__ import annotations

import kvcache_mask as km
import local_mask as lm

MASK_BLOCK_CAUSAL = 12


def m1_of(block: int, first_block: int) -> int:
    return block | (block - first_block) << 16


def block_end(p, block: int, first_block: int):
    """e(p): the first block end (F, F + C, F + 2C, ...) greater than p; int or index tensor."""
    k = (p - first_block) // block + 1  # ends F + k C with k >= 0; floor division, so p < F gives k <= 0
    if isinstance(k, int):
        return first_block + max(k, 0) * block
    return first_block + k.clamp(min=0) * block


def block_causal_mask_fn(block: int, first_block: int, window: int, sink: int):
    """allowed(q, kv) = kv < sink | (e(q) - W <= kv < e(q)) on index tensors; window -1 is unbounded."""

    def mod(q_idx, kv_idx):
        e = block_end(q_idx, block, first_block)
        near = kv_idx < e
        if window != -1:
            near = near & (kv_idx >= e - window)
        return (kv_idx < sink) | near

    return mod


def allowed(p: int, kv: int, sink: int, block: int, first_block: int, window: int) -> bool:
    e = block_end(p, block, first_block)
    return kv < sink or (kv < e and (window == -1 or kv >= e - window))


def band_items(sink: int, window: int, S: int, transposed: bool):
    """(row0, nrows) of every item of a block-causal band plan in launch order: those of its local band (sink, W - 1, 0)."""
    return lm.band_items(lm.MASK_LOCAL, sink, window - 1, 0, S, transposed)


def kv_slots(cap: int, sink: int, window: int, block: int) -> int:
    """Chunk slots per item of a single block-causal KV-cache plan (svgb_attn_plan_kvcache_block_bytes)."""
    return min(-(-cap // 128), -(-sink // 128) + (255 + window - 1 + block - 1) // 128 + 2)


def kv_plan(seqlens, *, Sq, new_len, nblocks, block_rows, table=None, batch_idx=None, sink, block, first_block, window):
    """kvcache_mask.plan under the block rule: [(stream b, first packed row, rows, [(physical row, valid, elem, logical
    index j)])] and the clamped lengths L_b, every chunk classified from its pairs."""
    cap = len(table[0]) * block_rows if table is not None else block_rows
    lens = [km.kv_len(s, new_len, cap) for s in seqlens]
    items = []
    for b, L in enumerate(lens):
        for r0 in range(0, Sq, km.ITEM_ROWS):
            nr = min(km.ITEM_ROWS, Sq - r0)
            ends = [block_end(L - Sq + i, block, first_block) for i in range(r0, r0 + nr)]
            chunks = []
            for j in range((L + km.CHUNK - 1) // km.CHUNK):
                c0, valid = j * km.CHUNK, min(km.CHUNK, L - j * km.CHUNK)
                pairs = [c0 + c < sink or (c0 + c < e and (window == -1 or c0 + c >= e - window))
                         for e in ends for c in range(valid)]
                if any(pairs):
                    blk = km.block_of(b, c0, nblocks=nblocks, block_rows=block_rows, table=table, batch_idx=batch_idx)
                    row = blk * block_rows + (c0 % block_rows if table is not None else c0)
                    chunks.append((row, valid, not all(pairs), j))
            items.append((b, b * Sq + r0, nr, chunks))
    return items, lens
