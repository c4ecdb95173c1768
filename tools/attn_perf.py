"""Attention-kernel timing matrix at HunyuanVideo-720p size (bring-up tool): JSON lines to
gpurun_out/attn_perf.jsonl."""
import json
import os
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "sparse-videogen_b200"))
sys.path.insert(0, str(ROOT))
import bench  # noqa: E402
from svgb200 import core  # noqa: E402

dev = torch.device("cuda:0")
OUT = ROOT / "gpurun_out"
OUT.mkdir(exist_ok=True)
TAG = os.environ.get("PERF_TAG", "")


def emit(**kw):
    kw["tag"] = TAG
    print(json.dumps(kw), flush=True)
    with open(OUT / "attn_perf.jsonl", "a") as f:
        f.write(json.dumps(kw) + "\n")


def t(fn, warm=2, iters=4):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


H, S, D = 24, bench.S, bench.D
q, k, v = (torch.randn(1, H, S, D, device=dev, dtype=torch.bfloat16) for _ in range(3))
W, _ = bench.band_width()
plan = core.plan_band(core.MASK_HY, bench.F * bench.P, bench.F * bench.P + bench.PROMPT_LEN, W, H, S, dev)
for tune in os.environ.get("PERF_TUNES", "").split(","):
    if tune:
        os.environ["SVGB_ATTN_TUNE"] = tune
    ms = t(lambda: core.attn_fwd(q, k, v, plan))
    emit(case="band_hy_rho0.30", tune=tune, ms=ms, tflops=4.0 * D * bench.band_pairs(W) * H / ms / 1e9)
if os.environ.get("PERF_BAND_ONLY"):
    sys.exit(0)

g = torch.Generator().manual_seed(0)


def sizes(n, heads):
    b = torch.full((heads, n), S // n, dtype=torch.int32)
    b[:, : S - (S // n) * n] += 1
    return b


for QC, KC, rho, heads in [(465, 931, 0.3, 24), (400, 1000, 0.3, 24), (400, 1000, 0.15, 24), (1, 1, 1.0, 4)]:
    row, col = sizes(QC, heads), sizes(KC, heads)
    bm = torch.rand(heads, QC, KC, generator=g) < rho
    bm[:, :, 0] = True
    fl = 4.0 * D * (row.double()[:, :, None] * col.double()[:, None, :] * bm).sum().item()
    pl = core.plan_varblock(bm.to(dev), row.to(dev), col.to(dev), S)
    qq, kk, vv = q[:, :heads], k[:, :heads], v[:, :heads]
    if heads != H:
        qq, kk, vv = qq.contiguous(), kk.contiguous(), vv.contiguous()
    ms = t(lambda: core.attn_fwd(qq, kk, vv, pl))
    emit(case=f"varblock_QC{QC}_KC{KC}_rho{rho}_h{heads}", ms=ms, tflops=fl / ms / 1e9)
    plg = core.plan_varblock(bm.to(dev), row.to(dev), col.to(dev), S, gather=True)
    ms = t(lambda: core.attn_fwd(qq, kk, vv, plg))
    emit(case=f"varblock_GATHER_QC{QC}_KC{KC}_rho{rho}_h{heads}", ms=ms, tflops=fl / ms / 1e9)

# ---- FP8 (e4m3) path on the band mask and the dense map
try:
    (q8, sq), (k8, sk), (v8, sv) = (core.quantize_e4m3(x) for x in (q, k, v))
    ms = t(lambda: core.attn_fwd_fp8(q8, k8, v8, sq, sk, sv, plan))
    emit(case="FP8_band_hy_rho0.30", ms=ms, tflops=4.0 * D * bench.band_pairs(W) * H / ms / 1e9)
    ms = t(lambda: core.quantize_e4m3(q))
    emit(case="quantize_e4m3_one_tensor", ms=ms, gbs=q.numel() * 3 / ms / 1e6)
except Exception as e:  # noqa: BLE001
    emit(case="FP8", error=repr(e)[:300])
