"""Attention on strided views on the H100: a diffusers-style call on transposed [B, S, H, D] projections three ways,

  views : core.attention on q.transpose(1, 2) etc. as they are (svgb_attn_fwd_strided / svgb_attn_bwd_strided)
  copies: core.attention after .contiguous() copies of q, k, v (and of the transposed dO in the backward), the copies
          timed with it
  sdpa  : torch.nn.functional.scaled_dot_product_attention on the same views (dense: a different amount of work)

at two shapes, B in {1, 2}:

  wan : Wan 2.1 720p, 75 600 tokens, 40 heads, a variable-block map of 300 x 1000 random blocks at density 0.3
  hy  : HunyuanVideo 720p SVG1 band (33 frames x 3600 + 256 text tokens, width 19 072)

    python tools/strided_attn_perf.py [--rounds R] [--out FILE]

For every case: ms of the forward, and of forward + backward through torch.autograd.backward with a transposed output
gradient.  Each figure is the median of R rounds with the rounds' min and max, the three ways alternated within every
round.  Plans (and their key-major companions) are built outside the timed region.  The card name and power limit are
read in the same run.
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "sparse-videogen_b200")]

D = 128


def card():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return dict(zip(q.split(","), [x.strip() for x in r.stdout.splitlines()[0].split(",")])) if r.returncode == 0 else {}


def plan_for(shape, B, dev):
    from svgb200 import core

    g = torch.Generator().manual_seed(0)
    if shape == "wan":
        H, S = 40, 75600
        sizes = lambda n: torch.full((B * H, n), S // n, dtype=torch.int32)  # noqa: E731
        bm = torch.rand(B * H, 300, 1000, generator=g) < 0.3
        plan = core.plan_varblock(bm.to(dev), sizes(300).to(dev), sizes(1000).to(dev), S)
    else:
        F, P, ctx, plen, W = 33, 3600, 256, 71, 19072
        H, S = 24, F * P + ctx
        plan = core.plan_band(core.MASK_HY, F * P, F * P + plen, W, B * H, S, dev)
    plan.key_major()
    return H, S, plan


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from svgb200 import core

    if not torch.cuda.is_available():
        raise SystemExit("strided_attn_perf needs a CUDA device")
    dev = torch.device("cuda:0")
    results = {"card_before": card(), "cases": []}
    for shape in ("wan", "hy"):
        for B in (1, 2):
            H, S, plan = plan_for(shape, B, dev)
            g = torch.Generator(device=dev).manual_seed(1)
            x = [torch.randn(B, S, H, D, device=dev, generator=g).to(torch.bfloat16) for _ in range(4)]
            grad_out = x[3].transpose(1, 2)

            def run(way, bwd):
                leaves = [t.detach().requires_grad_(bwd) for t in x[:3]]
                views = [t.transpose(1, 2) for t in leaves]
                if way == "copies":
                    views = [t.contiguous() for t in views]
                if way == "sdpa":
                    o = torch.nn.functional.scaled_dot_product_attention(*views)
                else:
                    o = core.attention(*views, plan)
                if bwd:
                    torch.autograd.backward(o, grad_out.contiguous() if way == "copies" else grad_out)

            case = {"shape": shape, "B": B, "H": H, "S": S}
            for bwd in (False, True):
                ways = ("views", "copies", "sdpa")
                for w in ways:
                    run(w, bwd)  # warm-up
                ms = {w: [] for w in ways}
                for _ in range(args.rounds):
                    for w in ways:
                        ms[w].append(timed(lambda: run(w, bwd)))
                key = "fwd_bwd" if bwd else "fwd"
                case[key] = {w: {"median_ms": round(statistics.median(v), 3), "min_ms": round(min(v), 3),
                                 "max_ms": round(max(v), 3)} for w, v in ms.items()}
            print(json.dumps(case), flush=True)
            results["cases"].append(case)
            del x, grad_out, plan
            torch.cuda.empty_cache()
    results["card_after"] = card()
    print(json.dumps({"card_before": results["card_before"], "card_after": results["card_after"]}))
    if args.out:
        Path(args.out).write_text(json.dumps(results, indent=1))


if __name__ == "__main__":
    main()
