"""Causal and sink-plus-window attention (SVGB_MASK_LOCAL band plans) on the H100, against PyTorch's own kernels:

  causal      : core.plan_local(causal=True)  vs  scaled_dot_product_attention(is_causal=True)
  sink-window : core.plan_local(window_size=(8192, 0), sink=1024)  vs  torch.compile(flex_attention) under the same
                mask_mod and its BlockMask

at S = 32 768 (24 heads) and 75 600 (40 heads, Wan 2.1 720p), bf16, D = 128: ms of the forward and of forward +
backward (torch.autograd.backward).  Each figure is the median of R rounds with the rounds' min and max, the two
ways alternated within every round; plans, key-major plans and BlockMasks are built outside the timed region.

  --order : the launch-order A/B of the planner.  A causal plan issues its query-major items from the last rows back
            (the longest lists first) and its key-major items from the first keys on; the other order is the same plan
            with its item array reversed.  Forward for the query-major order, backward for the key-major one.
  --wan-ab PARENT_LIB : the Wan 720p MASK_WAN band (P = 3600, width of sparsity 0.2, 40 heads), forward and forward +
            backward, one child process per build (SVGB200_LIB), parent and this build alternated R times; the outputs
            of the two builds are compared bit for bit.

    python tools/local_attn_perf.py [--rounds R] [--order] [--wan-ab PARENT_LIB] [--out FILE]

The card name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "sparse-videogen_b200")]

D = 128
SHAPES = ((32768, 24), (75600, 40))
SINK, LEFT = 1024, 8192


def card():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return dict(zip(q.split(","), [x.strip() for x in r.stdout.splitlines()[0].split(",")])) if r.returncode == 0 else {}


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def alternate(ways: dict, rounds: int) -> dict:
    for fn in ways.values():
        fn()  # warm-up
    torch.cuda.synchronize()
    ms = {w: [] for w in ways}
    for _ in range(rounds):
        for w, fn in ways.items():
            ms[w].append(timed(fn))
    return {w: {"median_ms": round(statistics.median(v), 3), "min_ms": round(min(v), 3), "max_ms": round(max(v), 3)}
            for w, v in ms.items()}


def inputs(B, H, S, dev, seed=1):
    g = torch.Generator(device=dev).manual_seed(seed)
    return [torch.randn(B, H, S, D, device=dev, generator=g).to(torch.bfloat16) for _ in range(4)]


def step(fn, x, bwd):
    leaves = [t.detach().requires_grad_(bwd) for t in x[:3]]
    o = fn(*leaves)
    if bwd:
        torch.autograd.backward(o, x[3])


def versus(dev, rounds):
    from torch.nn.attention.flex_attention import create_block_mask, flex_attention

    from svgb200 import core

    flex = torch.compile(flex_attention)
    out = []
    for S, H in SHAPES:
        x = inputs(1, H, S, dev)
        causal = core.plan_local(H, S, dev, causal=True)
        window = core.plan_local(H, S, dev, window_size=(LEFT, 0), sink=SINK)
        causal.key_major(), window.key_major()

        def mod(b, h, q, kv):
            return (kv < SINK) | ((q - kv <= LEFT) & (kv <= q))

        bm = create_block_mask(mod, None, None, S, S, device=dev, _compile=True)  # no dense S x S mask
        ways = {
            "causal": {"svgb": lambda *t: core.attention(*t, causal),
                       "sdpa": lambda *t: torch.nn.functional.scaled_dot_product_attention(*t, is_causal=True)},
            "sink-window": {"svgb": lambda *t: core.attention(*t, window),
                            "flex": lambda *t: flex(*t, block_mask=bm)},
        }
        for name, fns in ways.items():
            case = {"case": name, "S": S, "H": H}
            for bwd in (False, True):
                case["fwd_bwd" if bwd else "fwd"] = alternate(
                    {w: (lambda f=f: step(f, x, bwd)) for w, f in fns.items()}, rounds)
            print(json.dumps(case), flush=True)
            out.append(case)
        del x, causal, window, bm
        torch.cuda.empty_cache()
    return out


def reversed_items(plan):
    """The same plan with its item array in the opposite launch order (the lists stay where they are)."""
    from svgb200 import core

    d = plan.desc
    ws = plan.ws.clone()
    n = d.max_items
    items = ws[d.items_off: d.items_off + 32 * n].view(torch.int32).view(n, 8)
    items.copy_(items.flip(0))
    desc = type(d).from_buffer_copy(d)
    return core.AttnPlan(desc, ws)


def order_ab(dev, rounds):
    from svgb200 import core

    out = []
    for S, H in SHAPES:
        x = inputs(1, H, S, dev)
        plan = core.plan_local(H, S, dev, causal=True)
        kmaj = plan.key_major()
        other = reversed_items(plan)  # query-major: first rows first
        other_k = core.AttnPlan(plan.desc, plan.ws, _key_major=reversed_items(kmaj))  # key-major: last keys first
        case = {"case": "order", "S": S, "H": H,
                "fwd": alternate({"last_rows_first": lambda: core.attn_fwd(*x[:3], plan),
                                  "first_rows_first": lambda: core.attn_fwd(*x[:3], other)}, rounds)}
        o, lse = core.attn_fwd(*x[:3], plan, return_lse=True)
        case["bwd"] = alternate({"first_keys_first": lambda: core.attn_bwd(*x[:3], o, x[3], lse, plan),
                                 "last_keys_first": lambda: core.attn_bwd(*x[:3], o, x[3], lse, other_k)}, rounds)
        print(json.dumps(case), flush=True)
        out.append(case)
        del x, o, lse
        torch.cuda.empty_cache()
    return out


def wan_child(rounds):
    """One build's Wan 720p band timings and an output digest, as one JSON line."""
    from oracle import attention as oa
    from svgb200 import core

    dev = torch.device("cuda:0")
    F, P, H = 21, 3600, 40
    S = F * P
    W = oa.wan_band_width(oa.sparsity_to_width(0.2, 0, F, P), P)
    plan = core.plan_band(core.MASK_WAN, P, 0, W, H, S, dev)
    plan.key_major()
    x = inputs(1, H, S, dev)
    fn = lambda *t: core.attention(*t, plan)  # noqa: E731
    res = {"fwd": alternate({"x": lambda: step(fn, x, False)}, rounds)["x"],
           "fwd_bwd": alternate({"x": lambda: step(fn, x, True)}, rounds)["x"]}
    leaves = [t.detach().requires_grad_() for t in x[:3]]
    o = core.attention(*leaves, plan)
    o.backward(x[3])
    h = hashlib.sha256()
    for t in [o.detach()] + [t.grad for t in leaves]:
        h.update(t.contiguous().view(torch.int16).cpu().numpy().tobytes())
    res["digest"] = h.hexdigest()
    print(json.dumps(res), flush=True)


def wan_ab(parent_lib, rounds):
    runs = {"parent": [], "this": []}
    this_lib = str(ROOT / "sparse-videogen_b200" / "svgb200" / "_lib" / "libsvgb200.so")
    for _ in range(rounds):
        for name, lib in (("parent", parent_lib), ("this", this_lib)):
            r = subprocess.run([sys.executable, __file__, "--wan-child", "--rounds", "3"], capture_output=True,
                               text=True, env={**os.environ, "SVGB200_LIB": lib}, check=True)
            runs[name].append(json.loads(r.stdout.strip().splitlines()[-1]))
    res = {"case": "wan720-band-ab", "digests_equal": len({r["digest"] for v in runs.values() for r in v}) == 1}
    for name, v in runs.items():
        for k in ("fwd", "fwd_bwd"):
            ms = [r[k]["median_ms"] for r in v]
            res[f"{name}_{k}"] = {"median_ms": round(statistics.median(ms), 3), "min_ms": min(ms), "max_ms": max(ms)}
    print(json.dumps(res), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--order", action="store_true")
    ap.add_argument("--wan-ab", default=None, metavar="PARENT_LIB")
    ap.add_argument("--wan-child", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("local_attn_perf needs a CUDA device")
    if args.wan_child:
        return wan_child(args.rounds)
    dev = torch.device("cuda:0")
    results = {"card_before": card(), "cases": versus(dev, args.rounds)}
    if args.order:
        results["order"] = order_ab(dev, args.rounds)
    if args.wan_ab:
        results["wan_ab"] = wan_ab(args.wan_ab, args.rounds)
    results["card_after"] = card()
    print(json.dumps({"card_before": results["card_before"], "card_after": results["card_after"]}))
    if args.out:
        Path(args.out).write_text(json.dumps(results, indent=1))


if __name__ == "__main__":
    main()
