"""The cases of the split KV-cache census (oracle/kvsplit_census.py), shared by its CPU and GPU tests so that both
iterate one list.  TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import itertools

from oracle.kvsplit_census import Case, Mask

# causal; causal + window + a sink that ends mid-chunk; the two-sided window (255, 130) with sink 129; block-causal with
# first_block < block, a window and a sink; a causal window without sinks (rows whose keys lie only in later splits)
MASKS = {
    "causal": Mask(),
    "window_sink": Mask(sink=300, left=700),
    "two_sided": Mask(sink=129, left=255, right=130),
    "block": Mask(sink=200, block=300, first_block=170, window=900),
    "window": Mask(left=300),
}
# (format, D): bf16 at D = 128 and fp16 at D = 64, then the reverse, per-head and per-row e4m3 (D = 128)
FORMATS = [("bf16", 128), ("fp16", 64), ("fp16", 128), ("bf16", 64), ("e4m3", 128), ("e4m3_rows", 128)]
LAYOUTS = ["contig", "paged", "batch_idx"]


def _lens(Sq):
    """a stream ending mid-chunk and mid-page, one with L = 0, one shorter than its queries (L < Sq), a short one"""
    return [2900, 0, max(Sq - 13, 0) if Sq > 1 else 0, 1377]


SMALL = []
for i, (n, Sq) in enumerate(itertools.product((2, 3, 4, 7, 32), (1, 50, 256, 300))):
    fmt, D = FORMATS[i % len(FORMATS)]
    mask = list(MASKS)[i % len(MASKS)]
    SMALL.append(Case(f"n{n}_sq{Sq}_{fmt}{D}_{mask}_{LAYOUTS[i % 3]}_g{(1, 4)[(i // 3) % 2]}", _lens(Sq), Sq, 2,
                      (1, 4)[(i // 3) % 2], D, fmt, LAYOUTS[i % 3], MASKS[mask], n, seed=i))

# production shapes at 256-row pages, fp16 key census: the Wan 1.3B one-frame chunk (1 560 queries, 12 heads) and decode
# at 40 heads into a 21-frame cache with sink 1 560 and 14 040 keys back, under the automatic split count; the Wan
# block-causal chunk (three frames, 4 680 queries, one block) at forced n = 2 and 3
WAN_L, WAN_FRAME = 21 * 1560, 1560
PRODUCTION = [
    Case("wan_chunk_auto", [WAN_L], WAN_FRAME, 12, 1, 128, "fp16", "paged", Mask(sink=WAN_FRAME, left=9 * WAN_FRAME), 0),
    Case("decode40_auto", [WAN_L], 1, 40, 1, 128, "fp16", "paged", Mask(sink=WAN_FRAME, left=9 * WAN_FRAME), 0),
] + [
    Case(f"wan_block_n{n}", [WAN_L], 3 * WAN_FRAME, 12, 1, 128, "fp16", "paged",
         Mask(sink=WAN_FRAME, block=3 * WAN_FRAME, first_block=3 * WAN_FRAME, window=9 * WAN_FRAME), n)
    for n in (2, 3)
]
# the split counts plan_kvcache(num_splits=0) picks on 132 SMs (core.kvcache_num_splits); the GPU test requires the
# plan's count to be this one on a 132-SM device
AUTO_N = {"wan_chunk_auto": 3, "decode40_auto": 3}

ALL = SMALL + PRODUCTION


def splits(case):
    return case.n or AUTO_N[case.name]


# the softmax census per split (oracle.softmax's "none" case: one stream of S = 1 000 queries over its 1 000 keys, hot
# and cold tiers 160 log2 units apart, two heads): (mask, n, format, D)
SOFTMAX = [("causal", 2, "bf16", 128), ("window_sink", 3, "fp16", 64), ("two_sided", 7, "bf16", 64),
           ("block", 3, "fp16", 128), ("window", 2, "bf16", 128), ("causal", 7, "fp16", 64),
           ("block", 2, "bf16", 64), ("window_sink", 32, "fp16", 128)]


def softmax_case(i):
    """(oracle.softmax Case in logical order, Mask, n, format) of SOFTMAX[i]"""
    from oracle import softmax as sm

    mask, n, fmt, D = SOFTMAX[i]
    return sm.band_case("none", D=D, H=2, seed=i), MASKS[mask], n, fmt
