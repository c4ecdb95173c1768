"""Block-causal attention of autoregressive video (SVGB_MASK_BLOCK_CAUSAL) on the H100, bf16, D = 128, Wan's shapes
(1 560 tokens per latent frame, chunks of 3 frames = 4 680 tokens, 21 frames = 32 760 tokens):

  square (training): Wan 1.3B (12 heads) and 14B (40 heads), S = 32 760, forward and forward + backward
    (torch.autograd.backward) of
      block         core.plan_block_causal(block=4680)                          vs  compiled flex_attention
      block-window  core.plan_block_causal(block=4680, window=14040, sink=1560)  vs  compiled flex_attention
      token-causal  core.plan_local(causal=True), the token-level reference point at the same shape
    flex_attention runs under a BlockMask from create_block_mask on a CausVid-style `ends` mask_mod; its forward
    output is compared with svgb200's (norm-wise relative difference).
  kvcache (inference): tools/kvcache_perf.py's chunk case, 3 frames of queries against a 21-frame paged cache (256-row
    pages, shuffled table, one-frame sink), plan + forward as a caller issues them, in bf16, e4m3 with per-head scales
    and e4m3 with per-row scales:
      token  plan_kvcache(causal=True, window_size=(14040, 0), sink=1560): each query's window runs back from itself
      block  plan_kvcache(block=4680, window_size=(18720, -1), sink=1560): the chunk is one block, so every query
             attends the cache's last 18 720 keys (the first query's token window, widened to the whole chunk)
    and decode (1 query, block 1) and a one-frame chunk (1 560 queries, block 1560) under num_splits=0.

Each figure is the median of R rounds with the rounds' min and max, the ways of a case alternated within every round;
plans, key-major plans and BlockMasks are built outside the timed region (square), the kvcache plans inside it.  The
card name and power limit are read in the same run.

    python tools/block_causal_perf.py [--rounds R] [--iters N] [--only square|kvcache] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "sparse-videogen_b200"), str(ROOT / "tools")]

from kvcache_perf import alternate as alternate_n  # noqa: E402
from local_attn_perf import alternate, card, inputs, step  # noqa: E402

D, FRAME, FRAMES, CHUNK, PAGE = 128, 1560, 21, 3 * 1560, 256
S = FRAMES * FRAME
WINDOW, SINK = 9 * FRAME, FRAME
HEADS = (12, 40)


def _rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm())


def square(dev, rounds):
    from torch.nn.attention.flex_attention import create_block_mask, flex_attention

    from svgb200 import core

    flex = torch.compile(flex_attention)
    ends = torch.div(torch.arange(S, device=dev), CHUNK, rounding_mode="floor").add(1).mul(CHUNK).clamp(max=S)

    def unbounded(b, h, q, kv):  # CausVid: kv < ends[q]
        return kv < ends[q]

    def windowed(b, h, q, kv):
        return (kv < SINK) | ((kv < ends[q]) & (kv >= ends[q] - WINDOW))

    out = []
    for H in HEADS:
        x = inputs(1, H, S, dev)
        plans = {"block": core.plan_block_causal(H, S, dev, block=CHUNK),
                 "block-window": core.plan_block_causal(H, S, dev, block=CHUNK, window=WINDOW, sink=SINK),
                 "token-causal": core.plan_local(H, S, dev, causal=True)}
        for p in plans.values():
            p.key_major()
        masks = {"block": create_block_mask(unbounded, None, None, S, S, device=dev, _compile=True),
                 "block-window": create_block_mask(windowed, None, None, S, S, device=dev, _compile=True)}
        for name, plan in plans.items():
            fns = {"svgb": lambda *t, p=plan: core.attention(*t, p)}
            if name in masks:
                fns["flex"] = lambda *t, m=masks[name]: flex(*t, block_mask=m)
            case = {"case": name, "S": S, "H": H}
            for bwd in (False, True):
                case["fwd_bwd" if bwd else "fwd"] = alternate(
                    {w: (lambda f=f: step(f, x, bwd)) for w, f in fns.items()}, rounds)
            if name in masks:
                case["rel_diff_vs_flex"] = _rel(fns["svgb"](*x[:3]), fns["flex"](*x[:3]))
            print(json.dumps(case), flush=True)
            out.append(case)
        del x, plans, masks
        torch.cuda.empty_cache()
    return out


def kvcache(dev, rounds, iters):
    from svgb200 import core

    out = []
    bf = torch.bfloat16
    cap = ((S + PAGE - 1) // PAGE) * PAGE
    npages = cap // PAGE
    perm = torch.randperm(npages, generator=torch.Generator().manual_seed(0))
    table = perm.to(torch.int32).view(1, npages).to(dev)
    lens = torch.tensor([S], dtype=torch.int32, device=dev)
    for H in HEADS:
        g = torch.Generator(device=dev).manual_seed(H)
        rnd = lambda *s: torch.randn(*s, device=dev, generator=g).to(bf)  # noqa: E731
        kc, vc = rnd(cap, H, D), rnd(cap, H, D)
        kp, vp = torch.empty(npages, PAGE, H, D, device=dev, dtype=bf), torch.empty(npages, PAGE, H, D, device=dev,
                                                                                      dtype=bf)
        kp[perm], vp[perm] = kc.view(npages, PAGE, H, D), vc.view(npages, PAGE, H, D)
        amax = lambda t: (t.float().abs().amax(dim=(0, 1, 3)) / 448).clamp_min(1e-12)  # noqa: E731
        ks, vs = amax(kp), amax(vp)
        e4m3 = lambda t, sc: (t.float() * (1 / sc)[:, None]).clamp(-448, 448).to(torch.float8_e4m3fn)  # noqa: E731
        kp8, vp8 = e4m3(kp, ks), e4m3(vp, vs)
        # per-row: the append's power-of-two scales, written by the append itself into empty pages
        kr8, vr8 = (torch.zeros(npages, PAGE, H, D, device=dev, dtype=torch.float8_e4m3fn) for _ in range(2))
        ksr, vsr = (torch.zeros(npages, H, PAGE, device=dev) for _ in range(2))
        core.kvcache_append(kr8, vr8, kc.view(1, cap, H, D)[:, :S].contiguous(), vc.view(1, cap, H, D)[:, :S].contiguous(),
                            torch.zeros(1, dtype=torch.int32, device=dev), block_table=table, k_scale=ksr, v_scale=vsr)
        caches = {"bf16": (kp, vp, {}), "e4m3": (kp8, vp8, dict(k_scale=ks, v_scale=vs)),
                  "e4m3 rows": (kr8, vr8, dict(k_scale=ksr, v_scale=vsr))}
        token = dict(causal=True, window_size=(WINDOW, 0), sink=SINK)
        for Sq, blk, n in ((CHUNK, CHUNK, 1), (FRAME, FRAME, 0), (1, 1, 0)):
            q = rnd(1, Sq, H, D)
            rules = {"token": token, "block": dict(block=blk, window_size=(WINDOW + CHUNK, -1), sink=SINK)}
            for fmt, (k, v, kw) in caches.items():
                def way(rule, k=k, v=v, kw=kw):
                    plan = core.plan_kvcache(lens, q_len=Sq, num_blocks=npages, block_table=table, page_size=PAGE,
                                             num_splits=n, num_heads=H, **rule)
                    return core.attn_fwd(q, k, v, plan, **kw)

                res = alternate_n({r: (lambda r=r: way(rules[r])) for r in rules}, rounds, iters)
                case = {"case": "kvcache", "H": H, "Sq": Sq, "format": fmt, "num_splits": n, **res}
                print(json.dumps(case), flush=True)
                out.append(case)
        del kc, vc, kp, vp, kp8, vp8, kr8, vr8
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--only", choices=["square", "kvcache"], default=None)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("block_causal_perf.py measures on the GPU; no CUDA device found")
    dev = torch.device("cuda:0")
    res = {"card": card()}
    print(json.dumps(res), flush=True)
    if a.only in (None, "square"):
        res["square"] = square(dev, a.rounds)
    if a.only in (None, "kvcache"):
        res["kvcache"] = kvcache(dev, a.rounds, a.iters)
    if a.out:
        Path(a.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
