"""Attention into a KV cache for a batch of streams that are not in step, on the H100: one variable-length call
(core.kvcache_append(cu_seqlens=), core.plan_kvcache(cu_seqlens_q=), core.attn_fwd) against a per-stream loop and a
batch padded to the longest chunk.  The batch is Wan 480p (1 560 tokens per frame, D = 128) on 256-row pages under a
shuffled block table, with a one-frame sink and a 9-frame causal window, at 12 heads (Wan 1.3B) and 40 (Wan 14B):

  stream 0  a 1-frame first chunk into an empty cache
  stream 1  a 3-frame chunk against 9 cached frames
  stream 2  a 3-frame chunk against 21 cached frames
  stream 3  a 1-frame chunk against 21 cached frames

Ways, each append + plan + forward as a caller issues them:

  varlen   one call for the batch: packed q [total_q, H, D] and new rows [total_new, H, D]
  loop     one append, plan and forward per stream
  padded   every stream padded to the longest chunk (3 frames), real rows first: a uniform append of 3 frames per stream
           (the padding lands past each stream's keys and is never attended by a real row under the causal window) and
           a uniform plan and forward whose padded rows are computed and thrown away

in bf16, in e4m3 with per-head scales and in e4m3 with per-row scales, with num_splits 1 and 0 (automatic; the split
counts each way picked are reported).  Outputs are compared between the ways on the real rows: max |varlen - loop| and
max |varlen - padded|.  Each figure is the median of R rounds with the rounds' min and max; every round times N
back-to-back calls of each way with CUDA events, the ways alternated within every round.  The card name and power limit
are read in the same run.

    python tools/kvcache_varlen_perf.py [--rounds R] [--iters N] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "sparse-videogen_b200"), str(ROOT / "tools")]

from kvcache_perf import alternate  # noqa: E402
from local_attn_perf import card  # noqa: E402

D, FRAME, PAGE = 128, 1560, 256
LQ = [FRAME, 3 * FRAME, 3 * FRAME, FRAME]   # queries = new rows per stream
CACHED = [0, 9 * FRAME, 21 * FRAME, 21 * FRAME]  # keys before the append
CAP_FRAMES = 24
WIN = dict(causal=True, window_size=(9 * FRAME, 0), sink=FRAME)


def case(H, fmt, n, dev, rounds, iters):
    from svgb200 import core

    g = torch.Generator(device=dev).manual_seed(H)
    rnd = lambda *s: torch.randn(*s, device=dev, generator=g).to(torch.bfloat16)  # noqa: E731
    B, pad = len(LQ), max(LQ)
    mp = -(-CAP_FRAMES * FRAME // PAGE)
    table = torch.randperm(B * mp, device=dev, generator=g).to(torch.int32).view(B, mp)
    cache_dt = torch.bfloat16 if fmt == "bf16" else torch.float8_e4m3fn
    kc, vc = (torch.zeros(B * mp, PAGE, H, D, device=dev).to(cache_dt) for _ in range(2))
    sc = {}
    if fmt == "e4m3_head":
        sc = dict(k_scale=torch.full((H,), 4 / 448, device=dev), v_scale=torch.full((H,), 4 / 448, device=dev))
    elif fmt == "e4m3_rows":
        sc = dict(k_scale=torch.ones(B * mp, H, PAGE, device=dev), v_scale=torch.ones(B * mp, H, PAGE, device=dev))
    # the cached keys, written once by a uniform append of each stream's history
    for b in range(B):
        if CACHED[b]:
            core.kvcache_append(kc, vc, rnd(1, CACHED[b], H, D), rnd(1, CACHED[b], H, D),
                                torch.zeros(1, dtype=torch.int32, device=dev), block_table=table[b:b + 1], **sc)
    T = sum(LQ)
    q, k, v = rnd(T, H, D), rnd(T, H, D), rnd(T, H, D)
    cu = torch.tensor([0] + [sum(LQ[:i + 1]) for i in range(B)], dtype=torch.int32, device=dev)
    lens = torch.tensor(CACHED, dtype=torch.int32, device=dev)
    geo = dict(num_blocks=B * mp, page_size=PAGE, **WIN)
    rows = [(int(cu[b]), int(cu[b + 1])) for b in range(B)]
    qp, kp, vp = (torch.zeros(B, pad, H, D, device=dev, dtype=torch.bfloat16) for _ in range(3))
    for b, (r0, r1) in enumerate(rows):
        qp[b, :r1 - r0], kp[b, :r1 - r0], vp[b, :r1 - r0] = q[r0:r1], k[r0:r1], v[r0:r1]
    picked = {}

    def varlen():
        core.kvcache_append(kc, vc, k, v, lens, block_table=table, cu_seqlens=cu, **sc)
        p = core.plan_kvcache(lens, cu_seqlens_q=cu, total_q=T, max_seqlen_q=pad, cu_seqlens_new=cu, block_table=table,
                              num_splits=n, num_heads=H, **geo)
        picked["varlen"] = p.desc.max_items // p.desc.varlen_items
        return core.attn_fwd(q, kc, vc, p, **sc)

    def loop():
        outs, ns = [], []
        for b, (r0, r1) in enumerate(rows):
            core.kvcache_append(kc, vc, k[None, r0:r1], v[None, r0:r1], lens[b:b + 1], block_table=table[b:b + 1], **sc)
            p = core.plan_kvcache(lens[b:b + 1], q_len=r1 - r0, new_len=r1 - r0, block_table=table[b:b + 1],
                                  num_splits=n, num_heads=H, **geo)
            ns.append(p.desc.max_items // -(-(r1 - r0) // 256))
            outs.append(core.attn_fwd(q[None, r0:r1], kc, vc, p, **sc)[0])
        picked["loop"] = ns
        return torch.cat(outs)

    def padded():
        core.kvcache_append(kc, vc, kp, vp, lens, block_table=table, **sc)
        p = core.plan_kvcache(lens, q_len=pad, new_len=pad, block_table=table, num_splits=n, num_heads=H, **geo)
        picked["padded"] = p.desc.max_items // (B * -(-pad // 256))
        o = core.attn_fwd(qp, kc, vc, p, **sc)
        return torch.cat([o[b, :r1 - r0] for b, (r0, r1) in enumerate(rows)])

    # the padded append's extra rows land past every stream's keys, where the other ways never attend
    ov, ol, op = varlen().float(), loop().float(), padded().float()
    diff = dict(varlen_vs_loop=float((ov - ol).abs().max()), varlen_vs_padded=float((ov - op).abs().max()),
                varlen_equals_loop=bool(torch.equal(ov, ol)))
    times = alternate({"varlen": varlen, "loop": loop, "padded": padded}, rounds, iters)
    return dict(heads=H, format=fmt, num_splits=n, splits_picked=dict(picked), times=times, max_abs_diff=diff)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=9)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out")
    a = ap.parse_args()
    dev = torch.device("cuda")
    res = dict(card=card(), streams=dict(queries=LQ, cached=CACHED, frame=FRAME), rounds=a.rounds, iters=a.iters,
               cases=[])
    for H in (12, 40):
        for fmt in ("bf16", "e4m3_head", "e4m3_rows"):
            for n in (1, 0):
                r = case(H, fmt, n, dev, a.rounds, a.iters)
                res["cases"].append(r)
                t = r["times"]
                print(f"H={H:2d} {fmt:9s} n={n} picked={r['splits_picked']}  " +
                      "  ".join(f"{w} {t[w]['median_ms']:.3f} [{t[w]['min_ms']:.3f}, {t[w]['max_ms']:.3f}]" for w in t) +
                      f"  diff {r['max_abs_diff']}", flush=True)
    print(json.dumps(res["card"]))
    if a.out:
        Path(a.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
