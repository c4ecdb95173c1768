"""A/B two builds of the attention kernel on the tools/attn_perf.py cases at HunyuanVideo-720p size: outputs must be
bitwise equal, and the timings sit side by side.

    SVGB200_LIB=<build A> python tools/attn_ab.py run DIR_A
    SVGB200_LIB=<build B> python tools/attn_ab.py run DIR_B
    python tools/attn_ab.py compare DIR_A DIR_B

`run` (one process launch per build: the library is loaded once) writes each case's output as .npy plus
timings.json under DIR; the inputs come from a fixed seed, so both builds see the same tensors.  `compare` prints one
JSON line per case and exits non-zero if any output differs in any bit."""
import json
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent


def run(out: Path):
    import torch

    sys.path.insert(0, str(ROOT / "sparse-videogen_b200"))
    sys.path.insert(0, str(ROOT))
    import bench  # noqa: E402
    from svgb200 import core  # noqa: E402

    dev = torch.device("cuda:0")
    out.mkdir(parents=True, exist_ok=True)

    def t(fn, warm=3, iters=10):
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

    torch.manual_seed(0)
    H, S, D = 24, bench.S, bench.D
    q, k, v = (torch.randn(1, H, S, D, device=dev, dtype=torch.bfloat16) for _ in range(3))
    (q8, sq), (k8, sk), (v8, sv) = (core.quantize_e4m3(x) for x in (q, k, v))
    W, _ = bench.band_width()
    band = core.plan_band(core.MASK_HY, bench.F * bench.P, bench.F * bench.P + bench.PROMPT_LEN, W, H, S, dev)
    g = torch.Generator().manual_seed(0)
    QC, KC, rho = 465, 931, 0.3
    row = torch.full((H, QC), S // QC, dtype=torch.int32)
    row[:, : S - (S // QC) * QC] += 1
    col = torch.full((H, KC), S // KC, dtype=torch.int32)
    col[:, : S - (S // KC) * KC] += 1
    bm = torch.rand(H, QC, KC, generator=g) < rho
    bm[:, :, 0] = True
    vb = core.plan_varblock(bm.to(dev), row.to(dev), col.to(dev), S)
    vbg = core.plan_varblock(bm.to(dev), row.to(dev), col.to(dev), S, gather=True)

    cases = {
        "band": lambda: core.attn_fwd(q, k, v, band),
        "varblock": lambda: core.attn_fwd(q, k, v, vb),
        "gather": lambda: core.attn_fwd(q, k, v, vbg),
        "fp8_band": lambda: core.attn_fwd_fp8(q8, k8, v8, sq, sk, sv, band),
        "fp8_gather": lambda: core.attn_fwd_fp8(q8, k8, v8, sq, sk, sv, vbg),
        "quantize_e4m3": lambda: core.quantize_e4m3(q)[0],
    }
    ms = {}
    for name, fn in cases.items():
        res = fn()
        torch.cuda.synchronize()
        np.save(out / f"{name}.npy", res.contiguous().view(torch.uint8).cpu().numpy())
        ms[name] = t(fn)
        print(json.dumps({"case": name, "ms": round(ms[name], 4)}), flush=True)
    (out / "timings.json").write_text(json.dumps(ms))


def compare(a: Path, b: Path) -> int:
    ta, tb = json.loads((a / "timings.json").read_text()), json.loads((b / "timings.json").read_text())
    bad = 0
    for name in ta:
        xa, xb = np.load(a / f"{name}.npy"), np.load(b / f"{name}.npy")
        same = xa.shape == xb.shape and np.array_equal(xa, xb)
        bad += not same
        print(json.dumps({"case": name, "bit_identical": bool(same), "ms_a": round(ta[name], 4),
                          "ms_b": round(tb[name], 4), "b_over_a": round(tb[name] / ta[name], 4)}), flush=True)
    return 1 if bad else 0


if __name__ == "__main__":
    if len(sys.argv) == 3 and sys.argv[1] == "run":
        run(Path(sys.argv[2]))
    elif len(sys.argv) == 4 and sys.argv[1] == "compare":
        sys.exit(compare(Path(sys.argv[2]), Path(sys.argv[3])))
    else:
        sys.exit(__doc__)
