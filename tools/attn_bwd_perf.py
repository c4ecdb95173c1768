"""Forward + backward of the block-sparse attention on the H100, at the two shapes bench.py measures the forward at:

  band : HunyuanVideo 720p SVG1 band (S = 119 056, 24 heads, D = 128, W = 19 072, bf16)
  svg2 : the bench's SVG2 map (QC = 400 / KC = 1000 Bernoulli(0.30) + prompt / padding blocks, 24 heads)

    python tools/attn_bwd_perf.py [--iters N] [--no-flex] [--out FILE]

Reports ms of the forward (with LSE), of the backward (delta pre-pass + dK/dV + dQ kernels) and of both, and TFLOP/s of
the backward on two counts: the algorithmic 10 D FLOP per allowed (query, key) pair (S, dP, dV, dK, dQ: 2.5x the
forward's 4 D), and the FLOP the kernels execute (S and dP are recomputed in both kernels, 14 D per pair, over whole
128-row tiles and 64-column halves of each chunk).  The comparison point is torch.compile(flex_attention)'s forward +
backward under the same band mask, when it compiles.  The card name and power limit are read in the same run.
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


def card():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return dict(zip(q.split(","), [x.strip() for x in r.stdout.splitlines()[0].split(",")])) if r.returncode == 0 else {}


def timed(fn, iters, warm=2):
    for _ in range(warm):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def executed_cols(plan):
    """sum over the plan's streams of 128 rows x (each chunk's columns rounded up to the 64-column halves)"""
    d = plan.desc
    ws = plan.ws.cpu()
    heads = d.BH if d.items_stride else 1
    counts = ws[d.counts_off:d.counts_off + 4 * heads].view(torch.int32)
    items = ws[d.items_off:d.items_off + 32 * heads * d.max_items].view(torch.int32).view(heads, d.max_items, 2, 4)
    chunks = ws[d.chunks_off:].view(torch.int32)[: (ws.numel() - d.chunks_off) // 8 * 2].view(-1, 2)
    total = 0
    for h in range(heads):
        for it in items[h, : int(counts[h])].reshape(-1, 4).tolist():
            if it[1] == 0 or it[3] == 0:
                continue
            valid = (chunks[it[2]: it[2] + it[3], 1] & 0xff) + 1
            total += 128 * int(((valid + 63) // 64 * 64).sum())
    return total * (1 if d.items_stride else d.BH)


def measure(name, q, k, v, do, plan, pairs, iters, D):
    from svgb200 import core

    o, lse = core.attn_fwd(q, k, v, plan, return_lse=True)
    plan.key_major()  # built once, outside the timed region (cached on the plan)
    fwd = timed(lambda: core.attn_fwd(q, k, v, plan, return_lse=True), iters)
    bwd = timed(lambda: core.attn_bwd(q, k, v, o, do, lse, plan), iters)
    x = [t.detach().clone().requires_grad_() for t in (q, k, v)]
    total = timed(lambda: core.attention(*x, plan).backward(do), iters)
    alg = 10.0 * D * pairs
    exe = 6.0 * D * executed_cols(plan) + 8.0 * D * executed_cols(plan.key_major())
    return {"workload": name, "fwd_ms": fwd, "bwd_ms": bwd, "fwd_bwd_ms": total,
            "bwd_tflops_algorithmic": alg / bwd / 1e9, "bwd_tflops_executed": exe / bwd / 1e9,
            "bwd_flop_algorithmic": alg, "bwd_flop_executed": exe, "density": pairs / q.shape[1] / q.shape[2] ** 2}


def flex_point(q, k, v, do, mask_mod, iters):
    from torch.nn.attention.flex_attention import create_block_mask, flex_attention

    B, H, S, D = q.shape
    # _compile=True builds the block mask tile by tile instead of evaluating the S x S index grid (105 GiB here)
    bm = create_block_mask(mask_mod, None, None, S, S, device=q.device, _compile=True)
    fa = torch.compile(flex_attention)
    x = [t.detach().clone().requires_grad_() for t in (q, k, v)]
    ms = timed(lambda: fa(*x, block_mask=bm).backward(do), iters)
    return {"fwd_bwd_ms": ms}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--no-flex", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("attn_bwd_perf needs a GPU")
    import bench
    from oracle.attention import generic_mask_fn
    from svgb200 import core

    dev = torch.device("cuda:0")
    res = {"card": card()}
    H, D, S = bench.H_TOTAL, bench.D, bench.S
    V = bench.F * bench.P
    W = 19072
    g = torch.Generator(device=dev).manual_seed(0)
    q, k, v, do = (torch.randn(1, H, S, D, device=dev, generator=g).to(torch.bfloat16) for _ in range(4))

    mode, m0, m1, m2 = core.MASK_HY, V, V + bench.PROMPT_LEN, W
    mod = generic_mask_fn(mode, m0, m1, m2)
    kv = torch.arange(S, device=dev).view(1, -1)
    pairs = sum(int(mod(torch.arange(r, min(S, r + 2048), device=dev).view(-1, 1), kv).sum())
                for r in range(0, S, 2048)) * H
    band = core.plan_band(mode, m0, m1, m2, H, S, dev)
    res["band"] = measure(f"HunyuanVideo 720p band W={W}, S={S}, {H} heads, D={D}, bf16", q, k, v, do, band, pairs,
                          a.iters, D)

    bm, row, col, fl = bench.svg2_map(H)
    plan = core.plan_varblock(bm.to(dev), row.to(dev), col.to(dev), S)
    res["svg2"] = measure(f"SVG2 map QC=400+2 KC=1000+2 Bernoulli(0.30), S={S}, {H} heads, D={D}, bf16", q, k, v, do,
                          plan, fl / (4.0 * D), a.iters, D)

    emit(res, a.out)  # the comparison point below compiles first and may take long
    if not a.no_flex:
        try:
            res["flex_attention_band"] = flex_point(q, k, v, do, lambda b, h, qi, ki: mod(qi, ki), a.iters)
        except Exception as e:  # noqa: BLE001 -- the comparison point is optional; record why it is missing
            res["flex_attention_band"] = {"error": f"{type(e).__name__}: {str(e)[:300]}"}
    res["card_after"] = card()
    emit(res, a.out)


def emit(res, out):
    line = json.dumps(res)
    print(line, flush=True)
    if out:
        Path(out).write_text(line + "\n")


if __name__ == "__main__":
    main()
