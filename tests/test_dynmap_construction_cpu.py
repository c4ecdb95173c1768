"""The exact-arithmetic inputs of tests/test_dynmap_exact_gpu.py, checked without a GPU: on them the reference's
weighted softmax (oracle.kmeans.weighted_softmax) must give exactly round16(fl32(w / W)) -- scores of two values only,
exp exactly 1 or 0, an exact fp32 denominator.  A broken construction fails here, before it can make a GPU test vacuous."""
import pytest
import torch

from oracle import kmeans as ok


@pytest.mark.parametrize("D", [64, 128, 192, 256])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("BH,QC,KC", [(2, 40, 1000), (1, 3, 4096), (3, 9, 1)])
def test_onehot_softmax_is_exactly_rounded_quotient(BH, QC, KC, D, dtype):
    g = torch.Generator().manual_seed(KC * 1000 + D)
    qc, kc, ks = ok.onehot_dynmap_inputs(BH, QC, KC, D, dtype, g)
    scores = torch.matmul(qc, kc.transpose(-2, -1)) / (D ** 0.5)
    top = scores.float().amax(-1, keepdim=True)
    live = scores.float() == top
    # two values per row: the live score and 0, at least 256 apart (fp32 exp(-256) == 0)
    assert torch.all(live | (scores.float() == 0))
    assert torch.all((top == 0) | (top >= 256))
    assert torch.exp(torch.tensor(-256.0)) == 0
    w = torch.where(live, ks[:, None, :].float(), 0.0)
    W = w.double().sum(-1, keepdim=True)
    assert torch.all(W < 2 ** 24)
    expect = (w / W.float().clamp(min=1e-12)).to(dtype)
    got = ok.weighted_softmax(scores, ks[:, None, :].float())
    assert torch.equal(got.view(torch.int16), expect.view(torch.int16))
    # every case the construction promises is present
    rows_live = live.sum(-1)
    assert bool((rows_live == KC).any())  # a zero q row
    if KC > 1:
        assert bool((rows_live == 1).any()) or QC < 4  # the single key of direction 2
        zero_w = (W[..., 0] == 0) & (rows_live < KC)  # direction 1: live columns of size 0 only
        assert bool(zero_w.any()) and torch.all(got[zero_w] == 0)
    if KC >= 1000:
        ties = (ks == 7).sum(-1)
        assert bool((ties > 0.2 * KC).all())  # the run of equal sizes


def test_onehot_inputs_cover_every_scan_width():
    """The shapes the GPU test runs reach every block width of torch's CUDA scan, 32 to 1024 elements."""
    widths = {ok.cuda_scan_log_threads(r, c) for r, c in
              [(24 * 400, 1000), (4 * 64, 1000), (2 * 32, 1000), (2 * 8, 1000), (2 * 2, 1000), (2, 257), (2, 1024),
               (3, 3000), (2, 4096)]}
    assert widths == {4, 5, 6, 7, 8, 9}
