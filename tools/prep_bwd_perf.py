"""Forward and backward of the fused pre-attention pass (core.qkv_prep / core.qkv_prep_bwd) on the H100, at two shapes:

  hunyuan : HunyuanVideo 720p single block, S = 119 056, H = 24, D = 128, RMS per head, RoPE text last (256 text rows)
  wan     : Wan 720p, S = 75 600, H = 40, D = 128, RMS over the hidden row (H*D = 5120), complex RoPE on every row

    python tools/prep_bwd_perf.py [--iters N] [--out FILE]

Reports ms and GB/s on algorithmic bytes: the forward reads q_in, k_in, v_in and writes q, k, v (6 tensor passes); the
backward reads dQ, dK, dV and the saved q_in, k_in and writes dq_in, dk_in, dv_in (8 passes); both also read the RoPE
tables.  Bytes the kernels read again (the hidden-row RMS backward reads dQ / dK and q_in / k_in twice) are not
counted.  The card name and power limit are read in the same run.
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


def timed(fn, iters, warm=3):
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


SHAPES = {
    "hunyuan": dict(S=119056, H=24, D=128, norm=1, rope=1, txt=256),
    "wan": dict(S=75600, H=40, D=128, norm=3, rope=2, txt=0),
}


def run(name, iters):
    from svgb200 import core

    c = SHAPES[name]
    S, H, D, norm, rope, txt = c["S"], c["H"], c["D"], c["norm"], c["rope"], c["txt"]
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(0)
    dt = torch.bfloat16
    packed = torch.randn(1, S, 3 * H * D, device=dev, generator=g).to(dt)  # one packed QKV projection output
    qi, ki, vi = packed[..., :H * D], packed[..., H * D:2 * H * D], packed[..., 2 * H * D:]
    gw = H * D if norm == core.NORM_RMS_HIDDEN else D
    gq, gk = ((1 + 0.1 * torch.randn(gw, device=dev, generator=g)).to(dt) for _ in range(2))
    n = S - txt
    width = D // 2 if rope == 2 else D
    cos, sin = (torch.randn(n, width, device=dev, generator=g) for _ in range(2))
    kw = dict(norm=norm, gamma_q=gq, gamma_k=gk, eps=1e-6, rope=rope, cos=cos, sin=sin, rope_lo=0, rope_n=n)
    grads = [torch.randn(1, H, S, D, device=dev, generator=g).to(dt) for _ in range(3)]
    with torch.no_grad():
        fwd = timed(lambda: core.qkv_prep(qi, ki, vi, H, **kw), iters)
        bwd = timed(lambda: core.qkv_prep_bwd(*grads, H, S, q_in=qi, k_in=ki, **kw), iters)
    t = S * H * D * 2
    tables = 2 * n * width * 4
    return dict(shape=name, S=S, H=H, D=D, norm=norm, rope=rope, fwd_ms=round(fwd, 4), bwd_ms=round(bwd, 4),
                fwd_GBps=round((6 * t + tables) / fwd / 1e6, 1), bwd_GBps=round((8 * t + tables) / bwd / 1e6, 1),
                fwd_bytes=6 * t + tables, bwd_bytes=8 * t + tables)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("prep_bwd_perf.py needs a GPU")
    info = card()
    rows = []
    for name in SHAPES:
        r = dict(run(name, a.iters), **{"gpu": info.get("name"), "power_limit": info.get("power.limit")})
        print(json.dumps(r), flush=True)
        rows.append(r)
        torch.cuda.empty_cache()
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text("\n".join(json.dumps(r) for r in rows) + "\n")


if __name__ == "__main__":
    main()
