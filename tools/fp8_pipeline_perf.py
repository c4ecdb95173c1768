"""FP8 (e4m3) attention cores against the 16-bit ones at full size, in one process: JSON lines on stdout.

  * Wan 2.1 720p SVG2 (H = 40, S = 75 600, QC = 300 / KC = 1000, clustered synthetic tokens): the WanSAPCore step in
    bf16 and fp8, alternated, with warm centroids; the stages on their own (three quantizes, FP8 gather attention,
    FP8 TMA attention on e4m3 bytes permuted beforehand, bf16 attention and the permutes both TMA forms need); a
    density sweep of the whole step through the k-means maps of unclustered tokens (top_p varied, the reached
    density reported).  Every timing is the median over rounds in which each variant runs once.
  * HunyuanVideo 720p SVG1 (H = 24, S = 119 056): the HunyuanSVG1Core step in bf16 and fp8, alternated.
Every FP8 output is reported with its max / mean absolute difference from the bf16 output of the same inputs.

    python tools/fp8_pipeline_perf.py [--reps N]
"""
import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "sparse-videogen_b200"))
sys.path.insert(0, str(ROOT))

from svgb200 import core  # noqa: E402
from svgb200.models import hyvideo as hy  # noqa: E402
from svgb200.models import wan  # noqa: E402


def emit(**kw):
    print(json.dumps(kw), flush=True)


def card():
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader,nounits"], capture_output=True, text=True)
    name, power, clk = (x.strip() for x in q.stdout.strip().split(","))
    return {"gpu": name, "power_limit_w": float(power), "sm_max_mhz": int(clk),
            "torch_device": torch.cuda.get_device_name(0)}


def timed(fn):
    """(result, ms) of one call, bracketed by CUDA events."""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    r = fn()
    b.record()
    torch.cuda.synchronize()
    return r, a.elapsed_time(b)


def round_robin(fns, reps):
    """{name: median ms} of the callables, one call of each per round, so that clock changes under the card's power
    limit fall on every variant alike."""
    for fn in fns.values():
        fn()
    t = {name: [] for name in fns}
    for _ in range(reps):
        for name, fn in fns.items():
            t[name].append(timed(fn)[1])
    return {name: statistics.median(v) for name, v in t.items()}


def diff(a, b):
    d = (a.float() - b.float()).abs()
    return {"max_abs_diff": float(d.max()), "mean_abs_diff": float(d.mean())}


def steps(c16, c8, q, k, v, reps, **kw):
    """Median times of the two cores' steps, alternated (both warm), and their outputs on the same inputs."""
    t = round_robin({"bf16_ms": lambda: c16.sparse_core(q, k, v, **kw), "fp8_ms": lambda: c8.sparse_core(q, k, v, **kw)},
                    reps)
    return c16.sparse_core(q, k, v, **kw), c8.sparse_core(q, k, v, **kw), t


def wan_inputs(H, S, D, dev, seed, clusters):
    """clusters > 0: tokens with cluster structure, as tests/test_configs_gpu.py::test_wan720p_svg2_fullsize_pipeline
    builds them; 0: unclustered noise, whose near-flat centroid scores let top_p set the density."""
    g = torch.Generator(device=dev).manual_seed(seed)
    q, k, v = (torch.randn(1, H, S, D, device=dev, generator=g).to(torch.bfloat16) for _ in range(3))
    if clusters:
        base = torch.randn(1, H, clusters, D, device=dev, generator=g) * 1.5
        which = torch.randint(0, clusters, (S,), device=dev, generator=g)
        q = (q.float() * 0.7 + base[:, :, which]).to(torch.bfloat16)
        k = (k.float() * 0.7 + base[:, :, which]).to(torch.bfloat16)
    return q, k, v


def block_density(m, rs, cs, S):
    return float((m.float() * rs[:, :, None].float() * cs[:, None, :].float()).sum((1, 2)).mean() / (S * S))


def wan_pair(F, P, top_p, min_kc_ratio, q, k, v):
    kw = dict(num_q_centroids=300, num_k_centroids=1000, top_p_kmeans=top_p, min_kc_ratio=min_kc_ratio,
              kmeans_iter_init=4, kmeans_iter_step=2)
    c16, c8 = wan.WanSAPCore(F, P, **kw), wan.WanSAPCore(F, P, fp8=True, **kw)
    for c in (c16, c8):  # cold step from the same initial centroids: the warm steps start from equal states
        torch.manual_seed(0)
        c.sparse_core(q, k, v)
    return c16, c8


def wan_svg2(dev, reps):
    H, F, P, D = 40, 21, 3600, 128
    S = F * P
    shape = f"H={H} S={S} QC=300 KC=1000 kmeans_iter_step=2"
    q, k, v = wan_inputs(H, S, D, dev, 5, 64)
    c16, c8 = wan_pair(F, P, 0.9, 0.1, q, k, v)
    o16, o8, t = steps(c16, c8, q, k, v, reps)
    same = all(torch.equal(c16.last[x], c8.last[x]) for x in c16.last)
    last = c8.last
    m, rs, cs = last["dynamic_map"], last["q_sizes"], last["k_sizes"]
    qperm, kperm = last["q_sorted_indices"], last["k_sorted_indices"]
    emit(case="wan720p_svg2_step", shape=shape + " top_p=0.9 min_kc_ratio=0.1 (clustered tokens)",
         density=block_density(m, rs, cs, S), maps_and_permutations_identical=same, **t, **diff(o8, o16))

    # the stages on the last map
    (q8, sq), (k8, sk), (v8, sv) = (core.quantize_e4m3(x) for x in (q, k, v))
    plan_g = core.plan_varblock(m, rs, cs, S, gather=True)
    plan_t = core.plan_varblock(m, rs, cs, S)

    def perm8(x8, p):  # e4m3 bytes moved as 16-bit pairs
        return core.permute_gather(x8.view(torch.int16), p).view(torch.uint8)
    q8p, k8p, v8p = perm8(q8, qperm), perm8(k8, kperm), perm8(v8, kperm)
    qp, kp, vp = core.permute_gather(q, qperm), core.permute_gather(k, kperm), core.permute_gather(v, kperm)
    fns = {
        "quantize_x3_ms": lambda: [core.quantize_e4m3(x) for x in (q, k, v)],
        "fp8_gather_attn_ms": lambda: core.attn_fwd_fp8(q8, k8, v8, sq, sk, sv, plan_g, q_rows=qperm, kv_rows=kperm,
                                                        o_rows=qperm),
        "fp8_permute_x3_ms": lambda: (perm8(q8, qperm), perm8(k8, kperm), perm8(v8, kperm)),
        "fp8_tma_attn_on_permuted_ms": lambda: core.attn_fwd_fp8(q8p, k8p, v8p, sq, sk, sv, plan_t, o_rows=qperm),
        "bf16_permute_x3_ms": lambda: (core.permute_gather(q, qperm), core.permute_gather(k, kperm),
                                       core.permute_gather(v, kperm)),
        "bf16_attn_ms": lambda: core.attn_fwd(qp, kp, vp, plan_t, o_rows=qperm),
    }
    o_g, o_t, o_b = fns["fp8_gather_attn_ms"](), fns["fp8_tma_attn_on_permuted_ms"](), fns["bf16_attn_ms"]()
    emit(case="wan720p_svg2_stages", **round_robin(fns, reps),
         fp8_gather_vs_bf16=diff(o_g, o_b), fp8_tma_vs_bf16=diff(o_t, o_b), fp8_gather_vs_fp8_tma=diff(o_g, o_t))
    del c16, c8, q8p, k8p, v8p, qp, kp, vp, o_g, o_t, o_b, q8, k8, v8

    # density sweep (BASELINE config 5): the k-means maps of unclustered tokens, top_p varied, min_kc_ratio 0
    q, k, v = wan_inputs(H, S, D, dev, 6, 0)
    for top_p in (0.1, 0.2, 0.3, 0.4, 0.5):
        c16, c8 = wan_pair(F, P, top_p, 0.0, q, k, v)
        o16, o8, t = steps(c16, c8, q, k, v, max(2, reps // 2))
        m, rs, cs = (c8.last[x] for x in ("dynamic_map", "q_sizes", "k_sizes"))
        emit(case="wan720p_svg2_density_sweep", shape=shape + f" top_p={top_p} min_kc_ratio=0 (unclustered tokens)",
             density=block_density(m, rs, cs, S), **t, **diff(o8, o16))
        del c16, c8, o16, o8


def hunyuan_svg1(dev, reps):
    H, ctx, plen, F, P, D, sparsity = 24, 256, 71, 33, 3600, 128, 0.25
    S = ctx + F * P
    g = torch.Generator(device=dev).manual_seed(7)
    q, k, v = (torch.randn(1, H, S, D, device=dev, generator=g).to(torch.bfloat16) for _ in range(3))
    k[:, : H // 2] = (k[:, : H // 2].float() * 0.2 + q[:, : H // 2].float()).to(torch.bfloat16)  # local heads
    c16 = hy.HunyuanSVG1Core(ctx, plen, F, P, H, D, sparsity, dev)
    c8 = hy.HunyuanSVG1Core(ctx, plen, F, P, H, D, sparsity, dev, fp8=True)
    rows = torch.randint(0, 10000, (64,), generator=torch.Generator().manual_seed(0))
    o16, o8, t = steps(c16, c8, q, k, v, reps, sampled_rows=rows)
    emit(case="hunyuan720p_svg1_step", shape=f"H={H} S={S} sparsity={sparsity}", **t, **diff(o8, o16))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fp8_pipeline_perf.py measures on the GPU; no CUDA device found")
    dev = torch.device("cuda:0")
    core.device_check()
    emit(case="card", **card())
    wan_svg2(dev, args.reps)
    torch.cuda.empty_cache()
    hunyuan_svg1(dev, args.reps)
    emit(case="card_after", **card())


if __name__ == "__main__":
    main()
