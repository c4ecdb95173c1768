"""identify_dynamic_map (csrc/dynmap.cu) bit for bit, at every block width of torch's CUDA scan, every head dim and
both 16-bit types.

The inputs (oracle.kmeans.onehot_dynmap_inputs, checked on the CPU by test_dynmap_construction_cpu.py) make every
score, exp and softmax denominator exact, so the map is fully determined by the documented roundings: the kernel must
match two oracles exactly --
  1. oracle.kmeans.identify_dynamic_map(cumsum="cuda") on the CPU (the scan emulated by cumsum_like_torch_cuda), and
  2. the reference's torch ops (svg/kmeans_utils.py:864-896) run on this GPU, torch.cumsum included, with a stable sort
     (the engine pins ties to the lower column).
If 1 and 2 disagree the emulation is wrong, not the inputs."""
import pytest
import torch

from oracle import kmeans as ok

pytestmark = pytest.mark.gpu

DTYPES = [torch.bfloat16, torch.float16]

# (BH, QC, KC) -> log2 of torch's scan block half-width nx for BH * QC rows of KC (blocks of 2 * nx elements)
SCAN_SHAPES = [
    (24, 400, 1000, 4),  # HunyuanVideo 720p: 24 heads x 400 q-centroids
    (4, 64, 1000, 5),
    (2, 32, 1000, 6),
    (2, 8, 1000, 7),
    (2, 2, 1000, 8),
    (1, 2, 257, 8),
    (1, 2, 1024, 9),  # nx = 512 > 256 threads: each thread runs two network lanes
    (2, 1, 4096, 9),
    (1, 3, 3000, 9),  # three 1024-blocks, the running total carried twice
]


def reference_map_cuda(qc, kc, ks, p, preserve):
    """svg/kmeans_utils.py:864-896 on [1, BH, QC, KC] CUDA tensors (torch's own matmul, softmax, sort and cumsum)."""
    B, H, QC, D = qc.shape
    KC = kc.shape[2]
    scores = torch.matmul(qc, kc.transpose(-2, -1)) / (D ** 0.5)
    probs = ok.weighted_softmax(scores, ks.unsqueeze(-2).float())
    sorted_probs, sorted_idx = torch.sort(probs, dim=-1, descending=True, stable=True)
    cums = torch.cumsum(sorted_probs, dim=-1)
    remove = cums > p
    remove[..., 1:] = remove[..., :-1].clone()
    remove[..., 0] = False
    if preserve > 0:
        remove[..., :preserve] = False
    out = torch.zeros(B, H, QC, KC, dtype=torch.bool, device=qc.device)
    out.scatter_(-1, sorted_idx, ~remove)
    return out


def check_exact(cuda, BH, QC, KC, D, dtype, top_p, preserve, seed):
    from svgb200 import core

    g = torch.Generator().manual_seed(seed)
    qc, kc, ks = ok.onehot_dynmap_inputs(BH, QC, KC, D, dtype, g)
    got = core.dynamic_map(qc.to(cuda), kc.to(cuda), ks.to(cuda), top_p, preserve).cpu()
    # oracle 1 takes the reference's min_kc_ratio: int(ratio * KC) == preserve
    ratio = (preserve + 0.5) / KC if preserve > 0 else 0.0
    ref_cpu = ok.identify_dynamic_map(qc[None], kc[None], None, ks[None], top_p, ratio, cumsum="cuda")[0]
    ref_gpu = reference_map_cuda(qc[None].to(cuda), kc[None].to(cuda), ks[None].to(cuda), top_p, preserve)[0].cpu()
    emu = (ref_cpu != ref_gpu).any(-1)
    assert not emu.any(), f"scan emulation disagrees with torch.cumsum on {int(emu.sum())} of {emu.numel()} rows"
    bad = (got != ref_gpu).any(-1)
    assert not bad.any(), f"kernel map differs on {int(bad.sum())} of {bad.numel()} rows"
    return got


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("D", [64, 128, 192, 256])
@pytest.mark.parametrize("BH,QC,KC,log_nx", SCAN_SHAPES)
def test_dynamic_map_exact_every_scan_width(cuda, BH, QC, KC, log_nx, D, dtype):
    assert ok.cuda_scan_log_threads(BH * QC, KC) == log_nx
    got = check_exact(cuda, BH, QC, KC, D, dtype, 0.9, 0, seed=BH * QC * KC + D)
    # the cut is not trivial: some rows keep a strict subset of their live columns
    assert bool((got.sum(-1) < KC).any()) and bool((got.sum(-1) > 1).any())


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("top_p", [0.9, 1.0, 0.01])
@pytest.mark.parametrize("preserve", [(0, 0), (0, 1), (1, -1), (1, 0), (1, 7)], ids=["0", "1", "KC-1", "KC", "KC+7"])
@pytest.mark.parametrize("BH,QC,KC", [(2, 16, 257), (4, 64, 1000)])
def test_dynamic_map_exact_edges(cuda, BH, QC, KC, preserve, top_p, dtype):
    """top_p 1.0 (the 16-bit running sum can pass 1 and cut), 0.01 (only the first column survives) and the preserve
    prefix around its limits; every row kind of the construction (zero-size live columns, no live column, a single
    live column, a run of equal probabilities across the cut) is in every case."""
    pres = preserve[0] * KC + preserve[1]
    got = check_exact(cuda, BH, QC, KC, 128, dtype, top_p, pres, seed=KC + int(top_p * 100))
    if pres >= KC:
        assert bool(got.all())
    elif pres == 0 and top_p == 0.01:
        # rows with one dominant column keep exactly it
        assert bool((got.sum(-1) == 1).any())


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("D", [64, 256])
@pytest.mark.parametrize("preserve", [0, 1, 3])
def test_dynamic_map_exact_single_column(cuda, D, dtype, preserve):
    got = check_exact(cuda, 3, 40, 1, D, dtype, 0.9, preserve, seed=D)
    assert bool(got.all())


@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("rows,cols,log_nx", [(r * q, c, lg) for r, q, c, lg in SCAN_SHAPES])
def test_cumsum_oracle_matches_torch_cuda(cuda, rows, cols, log_nx, dtype):
    """cumsum_like_torch_cuda, on which test_golden_kmeans_cpu.py and test_svg2_ops_gpu.py rely, is torch.cumsum of a
    CUDA tensor bit for bit at every block width: positive probabilities and signed values."""
    assert ok.cuda_scan_log_threads(rows, cols) == log_nx
    g = torch.Generator().manual_seed(rows + cols)
    for x in (torch.rand(rows, cols, generator=g) * (3.0 / cols), torch.randn(rows, cols, generator=g)):
        x = x.to(dtype)
        got = torch.cumsum(x.to(cuda), dim=-1).cpu()
        ref = ok.cumsum_like_torch_cuda(x)
        assert torch.equal(got.view(torch.int16), ref.view(torch.int16))


@pytest.mark.xfail(strict=True, reason="a single row (BH * QC == 1) is outside the bit-exact contract: torch.cumsum "
                   "then runs cub::DeviceScan, whose 16-bit adds associate differently from the block scan")
@pytest.mark.parametrize("dtype", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("KC", [1000, 4096])
def test_dynamic_map_single_row_is_not_torch_exact(cuda, KC, dtype):
    """Records, on the H100, that torch's one-row scan differs from the block scan the kernel follows: on a zero q row
    (every column live) the two keep different column sets.  Production has thousands of rows."""
    check_exact(cuda, 1, 1, KC, 128, dtype, 0.9, 0, seed=KC)
