"""Attention into a KV cache (core.kvcache_append, core.plan_kvcache, core.attn_fwd) on the H100: the Self-Forcing /
CausVid streaming shape, a chunk of 3 latent frames (4 680 queries) against a 21-frame cache (32 760 keys, 1 560 tokens
per frame at 480p) with a one-frame sink and a window of 9 frames (14 040 keys) behind each query, bf16, D = 128, for
Wan 1.3B (12 heads) and Wan 14B (40 heads).  Ways, each one call sequence as a caller would issue it:

  contiguous      plan + forward on a contiguous [1, 32 760, H, D] cache
  paged           plan + forward on the same keys in 256-row pages under a shuffled block table
  append+paged    kvcache_append of the chunk's 4 680 new rows into the pages, then plan + forward
  index+contig    the caller-side alternative: the new rows written with one slice copy, then plan + forward
  roll+contig     eviction by shifting: the window part of the cache moved down by one chunk (a slice copy of a clone,
                  as rolling caches do), the new rows written at the end, then plan + forward
  sdpa            torch scaled_dot_product_attention on the sliced cache under the same boolean mask (built once)
  decode          Sq = 1: one query against the same cache, plan + forward (one CTA per head: no split-KV)
  fp8 paged       plan + forward on the same pages in e4m3 (per-KV-head scales), q quantised inside the call
  fp8 append+paged  kvcache_append quantising the chunk's new rows into the e4m3 pages, then plan + forward
  fp8 q quant     the q quantisation of the fp8 forward alone (a transposed copy and quantize_e4m3)
  rows paged      plan + forward on the same pages in e4m3 with per-row scales, q quantised per row inside the call
  rows append+paged  kvcache_append quantising the chunk's new rows per row into those pages, then plan + forward
  rows q quant    the per-row q quantisation alone (quantize_e4m3_rows on q in place)

With --split, the split-KV table instead (plan_kvcache(num_splits=)): decode (Sq = 1) at 12 and 40 heads, the one-frame
chunk (1 560 queries) at 12 heads and the three-frame chunk at 12 and 40 heads, against the same pages in bf16, in e4m3
with per-head scales and in e4m3 with per-row scales, each as the single pass (n = 1), n = 2, 4, 8 and the automatic
choice (n = 0, reported with the n it picked): plan + forward (+ merge) as a caller issues them.

Besides the times: the bytes of each cache (K and V, one layer, and the per-row scales) and mean / max
|o_fp8 - o_bf16| of the paged forward in both formats.

Each figure is the median of R rounds with the rounds' min and max; every round times N back-to-back calls of each way
with CUDA events, the ways alternated within every round.  The card name and power limit are read in the same run.

    python tools/kvcache_perf.py [--rounds R] [--iters N] [--split] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import statistics
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "sparse-videogen_b200"), str(ROOT / "tools")]

from local_attn_perf import card  # noqa: E402

D, FRAME, FRAMES, CHUNK_FRAMES, PAGE = 128, 1560, 21, 3, 256
L, SQ, SINK, LEFT = FRAMES * FRAME, CHUNK_FRAMES * FRAME, FRAME, 9 * FRAME


def timed(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def alternate(ways, rounds, iters):
    for fn in ways.values():
        fn()  # warm-up
    torch.cuda.synchronize()
    ms = {w: [] for w in ways}
    for _ in range(rounds):
        for w, fn in ways.items():
            ms[w].append(timed(fn, iters))
    return {w: {"median_ms": round(statistics.median(v), 3), "min_ms": round(min(v), 3), "max_ms": round(max(v), 3)}
            for w, v in ms.items()}


def case(H, dev, rounds, iters):
    from svgb200 import core

    g = torch.Generator(device=dev).manual_seed(H)
    bf = torch.bfloat16
    rnd = lambda *s: torch.randn(*s, device=dev, generator=g).to(bf)  # noqa: E731
    cap = ((L + PAGE - 1) // PAGE) * PAGE
    kc, vc = rnd(1, cap, H, D), rnd(1, cap, H, D)
    q, q1 = rnd(1, SQ, H, D), rnd(1, 1, H, D)
    knew, vnew = rnd(1, SQ, H, D), rnd(1, SQ, H, D)
    npages = cap // PAGE
    perm = torch.randperm(npages, generator=torch.Generator().manual_seed(0))
    kp, vp = torch.empty(npages, PAGE, H, D, device=dev, dtype=bf), torch.empty(npages, PAGE, H, D, device=dev, dtype=bf)
    kp[perm] = kc[0].view(npages, PAGE, H, D)
    vp[perm] = vc[0].view(npages, PAGE, H, D)
    table = perm.to(torch.int32).view(1, npages).to(dev)
    lens = torch.tensor([L], dtype=torch.int32, device=dev)
    before = lens - SQ  # the chunk's rows are appended at L - SQ
    win = dict(causal=True, window_size=(LEFT, 0), sink=SINK)

    def contiguous(qq=q, new_len=0, seq=lens):
        plan = core.plan_kvcache(seq, q_len=qq.shape[1], num_blocks=1, new_len=new_len, cache_len=cap, **win)
        return core.attn_fwd(qq, kc, vc, plan)

    def paged(qq=q, new_len=0, seq=lens):
        plan = core.plan_kvcache(seq, q_len=qq.shape[1], num_blocks=npages, new_len=new_len, block_table=table,
                                 page_size=PAGE, **win)
        return core.attn_fwd(qq, kp, vp, plan)

    def append_paged():
        core.kvcache_append(kp, vp, knew, vnew, before, block_table=table)
        return paged(new_len=SQ, seq=before)

    def index_contig():
        kc[:, L - SQ:L] = knew
        vc[:, L - SQ:L] = vnew
        return contiguous()

    def roll_contig():
        n = L - SINK - SQ  # the window part that stays, moved down by one chunk
        kc[:, SINK:SINK + n] = kc[:, SINK + SQ:L].clone()
        vc[:, SINK:SINK + n] = vc[:, SINK + SQ:L].clone()
        kc[:, L - SQ:L] = knew
        vc[:, L - SQ:L] = vnew
        return contiguous()

    p = torch.arange(SQ, device=dev)[:, None] + (L - SQ)
    kv = torch.arange(L, device=dev)[None, :]
    mask = (kv < SINK) | ((p - kv <= LEFT) & (kv <= p))
    qt = q.transpose(1, 2)

    def sdpa():
        k, v = kc[:, :L].transpose(1, 2), vc[:, :L].transpose(1, 2)
        return torch.nn.functional.scaled_dot_product_attention(qt, k, v, attn_mask=mask)

    # the e4m3 pages: per-KV-head absmax scales, the append's conversion
    amax = lambda t: (t.float().abs().amax(dim=(0, 1, 3)) / 448).clamp_min(1e-12)  # noqa: E731
    ks, vs = amax(kp), amax(vp)
    e4m3 = lambda t, sc: (t.float() * (1 / sc)[:, None]).clamp(-448, 448).to(torch.float8_e4m3fn)  # noqa: E731
    kp8, vp8 = e4m3(kp, ks), e4m3(vp, vs)

    def paged_fp8(new_len=0, seq=lens):
        plan = core.plan_kvcache(seq, q_len=SQ, num_blocks=npages, new_len=new_len, block_table=table, page_size=PAGE,
                                 **win)
        return core.attn_fwd(q, kp8, vp8, plan, k_scale=ks, v_scale=vs)

    def append_paged_fp8():
        core.kvcache_append(kp8, vp8, knew, vnew, before, block_table=table, k_scale=ks, v_scale=vs)
        return paged_fp8(new_len=SQ, seq=before)

    def q_quant():
        return core.quantize_e4m3(q.reshape(SQ, H, D).transpose(0, 1).contiguous())

    # the e4m3 pages with per-row scales [pages, H, PAGE]: the rows of the per-row append
    e = lambda t: (lambda m, k: torch.where(m <= 0.875, k - 9, k - 8))(*torch.frexp(t.float().abs().amax(-1)))  # noqa: E731
    ke, ve = e(kp).clamp(-126, 127), e(vp).clamp(-126, 127)
    kpr, vpr = ((t.float() * torch.exp2(-x.float())[..., None]).to(torch.float8_e4m3fn) for t, x in ((kp, ke), (vp, ve)))
    ksr, vsr = (torch.exp2(x.float()).transpose(1, 2).contiguous() for x in (ke, ve))

    def paged_rows(new_len=0, seq=lens):
        plan = core.plan_kvcache(seq, q_len=SQ, num_blocks=npages, new_len=new_len, block_table=table, page_size=PAGE,
                                 **win)
        return core.attn_fwd(q, kpr, vpr, plan, k_scale=ksr, v_scale=vsr)

    def append_paged_rows():
        core.kvcache_append(kpr, vpr, knew, vnew, before, block_table=table, k_scale=ksr, v_scale=vsr)
        return paged_rows(new_len=SQ, seq=before)

    def q_quant_rows():
        return core.quantize_e4m3_rows(q.reshape(SQ, H, D))

    # the ways agree before they are timed
    o_c, o_p = contiguous(), paged()
    assert torch.equal(o_c, o_p), "paged and contiguous differ"
    err = (sdpa().transpose(1, 2).float() - o_c.float()).abs().max().item()
    assert err < 3e-2, f"sdpa differs by {err}"
    d = (paged_fp8().float() - o_p.float()).abs()
    dr = (paged_rows().float() - o_p.float()).abs()
    fp8 = {"cache_bytes": {"bf16": 2 * kp.numel() * 2, "e4m3": 2 * kp8.numel(),
                           "e4m3 rows": 2 * kpr.numel() + 2 * 4 * ksr.numel()},
           "o_abs_diff_vs_bf16": {"mean": d.mean().item(), "max": d.max().item()},
           "rows_o_abs_diff_vs_bf16": {"mean": dr.mean().item(), "max": dr.max().item()}}
    ways = {"contiguous": contiguous, "paged": paged, "append+paged": append_paged, "index+contig": index_contig,
            "roll+contig": roll_contig, "sdpa": sdpa, "decode": lambda: paged(qq=q1), "fp8 paged": paged_fp8,
            "fp8 append+paged": append_paged_fp8, "fp8 q quant": q_quant, "rows paged": paged_rows,
            "rows append+paged": append_paged_rows, "rows q quant": q_quant_rows}
    return {**alternate(ways, rounds, iters), "fp8": fp8}


SPLIT_ROWS = [("decode", 1, 12), ("decode", 1, 40), ("one frame", FRAME, 12), ("three frames", SQ, 12),
              ("three frames", SQ, 40)]
SPLITS = [1, 2, 4, 8, 0]


def split_case(H, queries, dev, rounds, iters):
    """One row of the split table: the ways of SPLITS in the three cache formats on the same 256-row pages."""
    from svgb200 import core

    g = torch.Generator(device=dev).manual_seed(H)
    bf = torch.bfloat16
    cap = ((L + PAGE - 1) // PAGE) * PAGE
    npages = cap // PAGE
    kp, vp = (torch.randn(npages, PAGE, H, D, device=dev, generator=g).to(bf) for _ in range(2))
    q = torch.randn(1, queries, H, D, device=dev, generator=g).to(bf)
    table = torch.randperm(npages, generator=torch.Generator().manual_seed(0)).to(torch.int32).view(1, npages).to(dev)
    lens = torch.tensor([L], dtype=torch.int32, device=dev)
    amax = lambda t: (t.float().abs().amax(dim=(0, 1, 3)) / 448).clamp_min(1e-12)  # noqa: E731
    ks, vs = amax(kp), amax(vp)
    e4m3 = lambda t, sc: (t.float() * (1 / sc)[:, None]).clamp(-448, 448).to(torch.float8_e4m3fn)  # noqa: E731
    e = lambda t: (lambda m, k: torch.where(m <= 0.875, k - 9, k - 8))(*torch.frexp(t.float().abs().amax(-1)))  # noqa: E731
    ke, ve = e(kp).clamp(-126, 127), e(vp).clamp(-126, 127)
    fmts = {"bf16": (kp, vp, {}),
            "e4m3": (e4m3(kp, ks), e4m3(vp, vs), dict(k_scale=ks, v_scale=vs)),
            "e4m3 rows": (*((t.float() * torch.exp2(-x.float())[..., None]).to(torch.float8_e4m3fn)
                            for t, x in ((kp, ke), (vp, ve))),
                          dict(zip(("k_scale", "v_scale"), (torch.exp2(x.float()).transpose(1, 2).contiguous()
                                                            for x in (ke, ve)))))}

    def way(k, v, kw, n):
        def run():
            plan = core.plan_kvcache(lens, q_len=queries, num_blocks=npages, block_table=table, page_size=PAGE,
                                     causal=True, window_size=(LEFT, 0), sink=SINK, num_splits=n, num_heads=H)
            return core.attn_fwd(q, k, v, plan, **kw)
        return run

    auto = core.plan_kvcache(lens, q_len=queries, num_blocks=npages, block_table=table, page_size=PAGE, causal=True,
                             window_size=(LEFT, 0), sink=SINK, num_splits=0, num_heads=H)
    n_auto = auto.desc.max_items // -(-queries // 256)
    ways, diff = {}, {}
    for f, (k, v, kw) in fmts.items():
        ref = way(k, v, kw, 1)().float()
        for n in SPLITS:
            name = f"{f} n={n if n else 'auto'}"
            ways[name] = way(k, v, kw, n)
            diff[name] = (ways[name]().float() - ref).abs().max().item()  # the ways agree before they are timed
            assert diff[name] < (3e-2 if f == "bf16" else 8e-2), (name, diff[name])
    return {"auto_num_splits": n_auto, "ctas_single": -(-queries // 256) * H, **alternate(ways, rounds, iters),
            "max_abs_diff_vs_single": diff}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--split", action="store_true", help="the split-KV table instead")
    ap.add_argument("--out")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("kvcache_perf needs a GPU")
    dev = torch.device("cuda:0")
    res = {"card": card(), "rounds": a.rounds, "iters": a.iters,
           "shape": dict(queries=SQ, keys=L, sink=SINK, left=LEFT, page=PAGE, D=D)}
    if a.split:
        for label, queries, H in SPLIT_ROWS:
            name = f"{label}, {H} heads"
            res[name] = split_case(H, queries, dev, a.rounds, a.iters)
            print(json.dumps({name: res[name]}), flush=True)
    for name, H in (() if a.split else (("wan1.3b", 12), ("wan14b", 40))):
        res[name] = case(H, dev, a.rounds, a.iters)
        print(json.dumps({name: res[name]}), flush=True)
    print(json.dumps(res))
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
