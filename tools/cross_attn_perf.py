"""Cross-attention on the H100: queries of one length against keys / values of another (svgb_attn_fwd_kv /
svgb_attn_bwd_kv under a dense rectangular plan) next to torch.nn.functional.scaled_dot_product_attention on the same
inputs, at the two shapes the Wan blocks run beside the sparse self-attention:

  text : Wan 720p text cross-attention, 75 600 queries x 512 text keys, 40 heads, D = 128, bf16
  i2v  : the Wan I2V image branch, 75 600 queries x 257 image keys, 40 heads, D = 128, bf16

    python tools/cross_attn_perf.py [--iters N] [--rounds R] [--out FILE]

Reports ms of the forward (with LSE), of the backward (delta pre-pass + dK/dV + dQ kernels) and of forward + backward
through core.attention, the same for SDPA (forward; forward + backward through autograd), TFLOP/s on 4 D FLOP per
pair forward and 10 D backward, and the largest |o_svgb - o_sdpa|.  Each figure is the median of R rounds (the
rounds of every case alternated), a round being at least N calls and at least 0.5 s of them, with the rounds' min and
max beside it.  The autograd cases take the gradients with torch.autograd.grad, so no .grad accumulation is timed on
either side.  The card name and power limit are read in the same run, before and after.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "sparse-videogen_b200")]

SHAPES = {"text": 512, "i2v": 257}
H, SQ, D = 40, 75600, 128


def card():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return dict(zip(q.split(","), [x.strip() for x in r.stdout.splitlines()[0].split(",")])) if r.returncode == 0 else {}


def timed(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def measure(skv, iters, rounds, dev):
    from svgb200 import core

    g = torch.Generator(device=dev).manual_seed(skv)
    q, do = (torch.randn(1, H, SQ, D, device=dev, generator=g).to(torch.bfloat16) for _ in range(2))
    k, v = (torch.randn(1, H, skv, D, device=dev, generator=g).to(torch.bfloat16) for _ in range(2))
    one = torch.ones(H, 1, 1, dtype=torch.bool, device=dev)
    plan = core.plan_varblock(one, torch.full((H, 1), SQ, device=dev), torch.full((H, 1), skv, device=dev), SQ,
                              S_kv=skv)
    plan.key_major()  # built once, outside the timed region (cached on the plan)
    o, lse = core.attn_fwd(q, k, v, plan, return_lse=True)
    sdpa = torch.nn.functional.scaled_dot_product_attention
    err = float((o.float() - sdpa(q, k, v).float()).abs().max())
    x = [t.detach().clone().requires_grad_() for t in (q, k, v)]
    cases = {
        "svgb_fwd": lambda: core.attn_fwd(q, k, v, plan, return_lse=True),
        "svgb_bwd": lambda: core.attn_bwd(q, k, v, o, do, lse, plan),
        "svgb_fwd_bwd": lambda: torch.autograd.grad(core.attention(*x, plan), x, do),
        "sdpa_fwd": lambda: sdpa(q, k, v),
        "sdpa_fwd_bwd": lambda: torch.autograd.grad(sdpa(*x), x, do),
    }
    n = {}
    for name, fn in cases.items():  # warm-up (module loads, SDPA's backend choice), then calls per >= 0.5 s window
        for _ in range(3):
            fn()
        n[name] = max(iters, int(500.0 / timed(fn, 3)) + 1)
    ms = {name: [] for name in cases}
    for _ in range(rounds):
        for name, fn in cases.items():
            ms[name].append(timed(fn, n[name]))
    res = {"workload": f"Wan 720p cross-attention {SQ} x {skv}, {H} heads, D={D}, bf16, dense",
           "sdpa_backend": "torch default", "calls_per_round": n, "rounds": rounds}
    for name, t in ms.items():
        t = sorted(t)
        res[f"{name}_ms"] = t[len(t) // 2]
        res[f"{name}_ms_min_max"] = [t[0], t[-1]]
    pairs = H * SQ * skv
    res["svgb_fwd_tflops"] = 4.0 * D * pairs / res["svgb_fwd_ms"] / 1e9
    res["svgb_bwd_tflops"] = 10.0 * D * pairs / res["svgb_bwd_ms"] / 1e9
    res["max_abs_diff_vs_sdpa"] = err
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("cross_attn_perf needs a GPU")
    dev = torch.device("cuda:0")
    res = {"card": card()}
    for name, skv in SHAPES.items():
        res[name] = measure(skv, a.iters, a.rounds, dev)
    res["card_after"] = card()
    line = json.dumps(res)
    print(line, flush=True)
    if a.out:
        Path(a.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
