"""The local band mask (SVGB_MASK_LOCAL) restated on the host for the tests: its predicate, and the items of its band
plans in launch order.  TEST INFRASTRUCTURE ONLY.  The other band families are restated in oracle/attention.py
(generic_mask_fn) and oracle/bwd_census.py (band_items); these functions defer to them for every other mode."""
from __future__ import annotations

from oracle import attention as oa
from oracle import bwd_census as bc

MASK_LOCAL = 10


def local_mask_fn(sink: int, left: int, right: int):
    """allowed(q, kv) = kv < sink | (q - kv <= left & kv - q <= right), on index tensors."""

    def mod(q_idx, kv_idx):
        return (kv_idx < sink) | ((q_idx - kv_idx <= left) & (kv_idx - q_idx <= right))

    return mod


def mask_fn(mode: int, m0: int, m1: int, m2: int):
    """The predicate of band mode `mode` with the engine's parameters (include/svgb200.h SVGB_MASK_*)."""
    return local_mask_fn(m0, m1, m2) if mode == MASK_LOCAL else oa.generic_mask_fn(mode, m0, m1, m2)


def band_items(mode: int, m0: int, m1: int, m2: int, S: int, transposed: bool):
    """(row0, nrows) of every item of a band plan in launch order.  Local band: key-major, the sink keys (kv < m0) are
    a segment of their own, issued first; the band segment (the only one query-major) is issued from its last item
    back when its last rows carry the longest lists: query-major when left > right, key-major when right > left."""
    if mode != MASK_LOCAL:
        return bc.band_items(mode, m0, m1, S, transposed)
    b = [0] + ([m0] if transposed and 0 < m0 < S else []) + [S]
    out = []
    for i in range(len(b) - 1):
        seg = [(r, min(256, b[i + 1] - r)) for r in range(b[i], b[i + 1], 256)]
        if i == len(b) - 2 and (m2 > m1 if transposed else m1 > m2):
            seg = seg[::-1]
        out += seg
    return out
