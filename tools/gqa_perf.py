"""Grouped-query attention on the H100: the GQA entry points (svgb_attn_fwd_gqa / svgb_attn_bwd_gqa) with Hkv key/value
heads next to the MHA entries on K / V repeated to Hq heads (the same outputs: o and dq bit for bit), at two shapes:

  wan : Wan 2.1 720p, 75 600 tokens, 40 query heads, a variable-block map of 300 x 1000 random blocks at density 0.3
        (per key/value head; the MHA run repeats it per query head), Hkv in {40, 8, 1}
  hy  : HunyuanVideo 720p SVG1 band (33 frames x 3600 + 256 text tokens, width at sparsity 0.3), 24 query heads,
        Hkv in {24, 8, 1}
  dense: 40 query heads, 16 384 tokens, one all-ones block, beside scaled_dot_product_attention(..., enable_gqa=True)
        on the same inputs (fused SDPA backends only: a case no fused backend takes is reported, not run on the math
        backend), Hkv in {40, 8, 1}

    python tools/gqa_perf.py [--iters N] [--rounds R] [--out FILE]

For every case: ms of the forward (with LSE), of the backward (delta pre-pass + dK/dV + dQ) and of forward + backward
through core.attention (gradients through torch.autograd.grad).  Each figure is the median of R rounds, the rounds of
every case alternated, a round being at least N calls and at least 0.3 s of them, with the rounds' min and max beside
it.  Plans (and their key-major companions) are built outside the timed region.  The card name and power limit are
read in the same run, before and after.  At Hkv = 1 the dK/dV launch has G times fewer CTAs than MHA's, fewer than the
132 SMs when the key-major plan has few items per head.
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

D = 128


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


def partition(n, blocks, g):
    cuts, _ = torch.sort(torch.randperm(n - 1, generator=g)[: blocks - 1] + 1)
    return torch.diff(torch.cat([torch.tensor([0]), cuts, torch.tensor([n])])).to(torch.int32)


def plans(shape, Hq, Hkv, dev):
    """(GQA plan over Hkv heads, MHA plan over Hq heads, S)"""
    from svgb200 import core

    if shape == "hy":
        from oracle import attention as oa
        from oracle import census as oc

        ctx, F, P, plen = 256, 33, 3600, 71
        args, _ = oc.band_args("hy", F, P, ctx, plen, oa.sparsity_to_width(0.3, ctx, F, P))
        S = ctx + F * P
        p = core.plan_band(*args, Hkv, S, dev)
        return p, p, S
    S = 16384 if shape == "dense" else 75600
    if shape == "dense":
        one = torch.ones(Hkv, 1, 1, dtype=torch.bool)
        bm, rows, cols = one, torch.full((Hkv, 1), S), torch.full((Hkv, 1), S)
    else:
        g = torch.Generator().manual_seed(720)
        rows = torch.stack([partition(S, 300, g) for _ in range(Hkv)])
        cols = torch.stack([partition(S, 1000, g) for _ in range(Hkv)])
        bm = torch.rand(Hkv, 300, 1000, generator=g) < 0.3
    G = Hq // Hkv
    mk = lambda b, r, c: core.plan_varblock(b.to(dev), r.to(dev), c.to(dev), S)  # noqa: E731
    pg = mk(bm, rows, cols)
    pm = pg if G == 1 else mk(*(t.repeat_interleave(G, 0) for t in (bm, rows, cols)))
    return pg, pm, S


def measure(shape, Hq, Hkv, iters, rounds, dev):
    from svgb200 import core

    pg, pm, S = plans(shape, Hq, Hkv, dev)
    pg.key_major(), pm.key_major()  # built once, outside the timed region (cached on the plan)
    G = Hq // Hkv
    g = torch.Generator(device=dev).manual_seed(Hq + Hkv)
    q, do = (torch.randn(1, Hq, S, D, device=dev, generator=g).to(torch.bfloat16) for _ in range(2))
    k, v = (torch.randn(1, Hkv, S, D, device=dev, generator=g).to(torch.bfloat16) for _ in range(2))
    kr, vr = (t.repeat_interleave(G, 1).contiguous() for t in (k, v))
    o, lse = core.attn_fwd(q, k, v, pg, return_lse=True)
    o_m, lse_m = core.attn_fwd(q, kr, vr, pm, return_lse=True)
    same_o = bool(torch.equal(o, o_m) and torch.equal(lse, lse_m))
    dq = core.attn_bwd(q, k, v, o, do, lse, pg)[0]
    same_dq = bool(torch.equal(dq, core.attn_bwd(q, kr, vr, o_m, do, lse_m, pm)[0]))
    del dq
    x = [t.detach().clone().requires_grad_() for t in (q, k, v)]
    xm = [t.detach().clone().requires_grad_() for t in (q, kr, vr)]
    cases = {
        "gqa_fwd": lambda: core.attn_fwd(q, k, v, pg, return_lse=True),
        "gqa_bwd": lambda: core.attn_bwd(q, k, v, o, do, lse, pg),
        "gqa_fwd_bwd": lambda: torch.autograd.grad(core.attention(*x, pg), x, do),
    }
    if G > 1:
        cases.update({
            "mha_fwd": lambda: core.attn_fwd(q, kr, vr, pm, return_lse=True),
            "mha_bwd": lambda: core.attn_bwd(q, kr, vr, o_m, do, lse_m, pm),
            "mha_fwd_bwd": lambda: torch.autograd.grad(core.attention(*xm, pm), xm, do),
        })
    if shape == "dense":
        from torch.nn.attention import SDPBackend, sdpa_kernel

        fused = [SDPBackend.FLASH_ATTENTION, SDPBackend.CUDNN_ATTENTION, SDPBackend.EFFICIENT_ATTENTION]

        def sdpa(*a, **kw):
            with sdpa_kernel(fused):
                return torch.nn.functional.scaled_dot_product_attention(*a, **kw)

        cases.update({
            "sdpa_fwd": lambda: sdpa(q, k, v, enable_gqa=True),
            "sdpa_fwd_bwd": lambda: torch.autograd.grad(sdpa(*x, enable_gqa=True), x, do),
        })
    n, skipped = {}, {}
    for name, fn in list(cases.items()):
        try:
            for _ in range(2):
                fn()
        except RuntimeError as e:  # SDPA without a fused backend for these inputs
            skipped[name] = str(e).splitlines()[0][:200]
            del cases[name]
            continue
        n[name] = max(iters, int(300.0 / timed(fn, 2)) + 1)
    ms = {name: [] for name in cases}
    for _ in range(rounds):
        for name, fn in cases.items():
            ms[name].append(timed(fn, n[name]))
    res = {"shape": shape, "Hq": Hq, "Hkv": Hkv, "S": S, "o_lse_bitwise_vs_mha": same_o,
           "dq_bitwise_vs_mha": same_dq, "dkdv_ctas": [pg.key_major().desc.max_items, Hkv],
           "calls_per_round": n, "rounds": rounds, "skipped": skipped}
    for name, t in ms.items():
        t = sorted(t)
        res[f"{name}_ms"] = round(t[len(t) // 2], 3)
        res[f"{name}_ms_min_max"] = [round(t[0], 3), round(t[-1], 3)]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gqa_perf needs a GPU")
    dev = torch.device("cuda:0")
    res = {"card": card(), "cases": []}
    for shape, Hq in (("wan", 40), ("hy", 24), ("dense", 40)):
        for Hkv in (Hq, 8, 1):
            r = measure(shape, Hq, Hkv, a.iters, a.rounds, dev)
            print(json.dumps(r), flush=True)
            res["cases"].append(r)
            torch.cuda.empty_cache()
    res["card_after"] = card()
    if a.out:
        Path(a.out).write_text(json.dumps(res) + "\n")
    print(json.dumps({"card": res["card"], "card_after": res["card_after"]}), flush=True)


if __name__ == "__main__":
    main()
