"""Causal and windowed attention inside packed variable-length segments (core.plan_local_varlen) on the H100, against
PyTorch:

  packed-causal : 32 760 + 16 380 + 8 190 + 4 680 tokens, 24 heads, causal in each segment, packed [total, H, D]:
                  svgb  vs  a Python loop of scaled_dot_product_attention(is_causal=True) per segment  vs
                  torch.compile(flex_attention) under a document-causal BlockMask
  kv-cache      : 4 680 queries against 32 760 keys (the queries are the last 4 680 positions), sink 1 560, window
                  14 040 behind, 24 heads:  svgb  vs  torch.compile(flex_attention) under the same mask

bf16, D = 128: ms of the forward and of forward + backward (torch.autograd.backward).  Each figure is the median of R
rounds with the rounds' min and max, the ways alternated within every round; plans, key-major plans and BlockMasks
are built outside the timed region.

  --order : the launch-order A/B of the planner on the packed causal batch: its items in row order (the planner's
            order: segments in turn, first rows first) against longest list first (LPT), the same plan with its item
            array sorted by list length, stable.  Forward for the query-major plan, backward for the key-major one.

    python tools/varlen_local_perf.py [--rounds R] [--order] [--out FILE]

The card name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "sparse-videogen_b200"), str(ROOT / "tools")]

from local_attn_perf import alternate, card  # noqa: E402

D, H = 128, 24
SEGS = (32760, 16380, 8190, 4680)
KV_Q, KV_K, KV_SINK, KV_LEFT = 4680, 32760, 1560, 14040


def packed(n, dev, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    return torch.randn(n, H, D, device=dev, generator=g).to(torch.bfloat16)


def step(fn, x, do, bwd):
    leaves = [t.detach().requires_grad_(bwd) for t in x]
    o = fn(*leaves)
    if bwd:
        torch.autograd.backward(o, do)


def cu_of(lens, dev):
    c = [0]
    for n in lens:
        c.append(c[-1] + n)
    return torch.tensor(c, dtype=torch.int32, device=dev), c


def versus(dev, rounds):
    from torch.nn.attention.flex_attention import create_block_mask, flex_attention

    from svgb200 import core

    flex = torch.compile(flex_attention)
    out = []
    # packed causal batch
    cu, cu_host = cu_of(SEGS, dev)
    S = cu_host[-1]
    x = [packed(S, dev, i) for i in range(3)]
    do = packed(S, dev, 3)
    plan = core.plan_local_varlen(cu, total_q=S, causal=True)
    plan.key_major()
    doc = torch.repeat_interleave(torch.arange(len(SEGS), device=dev), torch.tensor(SEGS, device=dev))

    def doc_causal(b, h, q, kv):
        return (doc[q] == doc[kv]) & (kv <= q)

    bm = create_block_mask(doc_causal, None, None, S, S, device=dev, _compile=True)

    def sdpa_loop(q, k, v):
        outs = [torch.nn.functional.scaled_dot_product_attention(
            *(t[a:b].transpose(0, 1)[None] for t in (q, k, v)), is_causal=True)[0].transpose(0, 1)
            for a, b in zip(cu_host[:-1], cu_host[1:])]
        return torch.cat(outs)

    ways = {"svgb": lambda q, k, v: core.attention(q, k, v, plan, layout="shd"),
            "sdpa_loop": sdpa_loop,
            "flex": lambda q, k, v: flex(*(t.transpose(0, 1)[None] for t in (q, k, v)),
                                         block_mask=bm)[0].transpose(0, 1)}
    case = {"case": "packed-causal", "segments": list(SEGS), "H": H}
    for bwd in (False, True):
        case["fwd_bwd" if bwd else "fwd"] = alternate({w: (lambda f=f: step(f, x, do, bwd)) for w, f in ways.items()},
                                                      rounds)
    print(json.dumps(case), flush=True)
    out.append(case)
    del x, do, plan, bm
    torch.cuda.empty_cache()

    # KV-cache chunk: queries at the last KV_Q positions of KV_K keys, sink plus a window behind
    q = packed(KV_Q, dev, 4)
    k, v = packed(KV_K, dev, 5), packed(KV_K, dev, 6)
    do = packed(KV_Q, dev, 7)
    cq, _ = cu_of([KV_Q], dev)
    ck, _ = cu_of([KV_K], dev)
    plan = core.plan_local_varlen(cq, ck, total_q=KV_Q, total_k=KV_K, causal=True, window_size=(KV_LEFT, 0),
                                  sink=KV_SINK)
    plan.key_major()
    off = KV_K - KV_Q

    def kv_mod(b, h, qi, kj):
        p = qi + off
        return (kj < KV_SINK) | ((p - kj <= KV_LEFT) & (kj <= p))

    bm = create_block_mask(kv_mod, None, None, KV_Q, KV_K, device=dev, _compile=True)
    ways = {"svgb": lambda a, b, c: core.attention(a, b, c, plan, layout="shd"),
            "flex": lambda a, b, c: flex(*(t.transpose(0, 1)[None] for t in (a, b, c)),
                                         block_mask=bm)[0].transpose(0, 1)}
    case = {"case": "kv-cache", "Sq": KV_Q, "Skv": KV_K, "sink": KV_SINK, "left": KV_LEFT, "H": H}
    for bwd in (False, True):
        case["fwd_bwd" if bwd else "fwd"] = alternate(
            {w: (lambda f=f: step(f, (q, k, v), do, bwd)) for w, f in ways.items()}, rounds)
    print(json.dumps(case), flush=True)
    out.append(case)
    return out


def longest_first(plan):
    """The same plan with its items sorted by list length, longest first, ties in row order (the lists stay where they
    are)."""
    from svgb200 import core

    d = plan.desc
    ws = plan.ws.clone()
    n = int(ws[d.counts_off: d.counts_off + 4].view(torch.int32)[0])
    items = ws[d.items_off: d.items_off + 32 * n].view(torch.int32).view(n, 8)
    items.copy_(items[(-items[:, 3]).argsort(stable=True)])
    return core.AttnPlan(type(d).from_buffer_copy(d), ws, plan.source)


def order_ab(dev, rounds):
    from svgb200 import core

    cu, cu_host = cu_of(SEGS, dev)
    S = cu_host[-1]
    x = [packed(S, dev, i) for i in range(4)]
    plan = core.plan_local_varlen(cu, total_q=S, causal=True)
    kmaj = plan.key_major()
    other = longest_first(plan)
    other_k = core.AttnPlan(plan.desc, plan.ws, plan.source, _key_major=longest_first(kmaj))
    case = {"case": "order", "segments": list(SEGS), "H": H,
            "fwd": alternate({"row_order": lambda: core.attn_fwd(*x[:3], plan, layout="shd"),
                              "longest_first": lambda: core.attn_fwd(*x[:3], other, layout="shd")}, rounds)}
    o, lse = core.attn_fwd(*x[:3], plan, layout="shd", return_lse=True)
    case["bwd"] = alternate({"row_order": lambda: core.attn_bwd(*x[:3], o, x[3], lse, plan, layout="shd"),
                             "longest_first": lambda: core.attn_bwd(*x[:3], o, x[3], lse, other_k, layout="shd")},
                            rounds)
    same = [torch.equal(a, b) for a, b in zip(core.attn_bwd(*x[:3], o, x[3], lse, plan, layout="shd"),
                                              core.attn_bwd(*x[:3], o, x[3], lse, other_k, layout="shd"))]
    case["orders_give_equal_bits"] = torch.equal(o, core.attn_fwd(*x[:3], other, layout="shd")) and all(same)
    print(json.dumps(case), flush=True)
    return case


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--order", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("varlen_local_perf needs a CUDA device")
    dev = torch.device("cuda:0")
    results = {"card_before": card(), "cases": versus(dev, args.rounds)}
    if args.order:
        results["order"] = order_ab(dev, args.rounds)
    results["card_after"] = card()
    print(json.dumps({"card_before": results["card_before"], "card_after": results["card_after"]}))
    if args.out:
        Path(args.out).write_text(json.dumps(results, indent=1))


if __name__ == "__main__":
    main()
