"""CPU proof that the attention census (tests/test_attention_census_gpu.py, oracle/census.py) sees one key.

The census compares round16(cnt / n) bit for bit and exp(lse) with n.  A key wrongly kept or dropped moves n by one
and one count of each encoding by one.  This module shows, without a GPU, that
  * every count any census case can produce stays below the output format's distinguishability limit, so
    round16((cnt +- 1) / n) != round16(cnt / n) wherever cnt +- 1 is a possible count;
  * exp(lse) lands within 0.5 of n at every n the census runs at, given a log2 within one ulp, so n +- 1 fails;
  * the census tables equal brute-force counts over the oracle's dense element masks.
"""
import pytest
import torch

from oracle import attention as oa
from oracle import census as oc

# (largest S, D, output format) of the census cases: fp16 band / variable-block / gather cases, fp8 cases (bf16 out)
CASES = [(oc.N_MAX, 128, torch.float16), (6000, 64, torch.float16), (8000, 128, torch.bfloat16)]


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_census_distinguishable_limit(dtype):
    """The first count at which round(c / n) == round((c + 1) / n) for some n <= N_MAX, per output format."""
    assert oc.distinguishable_limit(oc.N_MAX, dtype) == oc.COUNT_LIMIT[dtype]


@pytest.mark.parametrize("S,D,dtype", CASES)
def test_census_sees_one_key(S, D, dtype):
    """Every table of every census case: counts (and their +-1 neighbours) stay distinguishable, and the lse pins n.
    column_bound grows with S, so the largest S of a (D, format) class covers all its cases."""
    for enc in oc.ENCODINGS:
        assert oc.column_bound(S, D, enc) < oc.COUNT_LIMIT[dtype]  # pairs (c, c + 1) with c < limit differ
    assert oc.lse_count_error(S) < 0.5
    # and concretely, at the worst n and count: a one-key change is visible in the rounded output
    n = torch.tensor([S], dtype=torch.int64)
    c = oc.column_bound(S, D, 1)
    base = oc.expected_output(torch.tensor([[c]]), n, dtype)
    assert base.view(torch.int16) != oc.expected_output(torch.tensor([[c - 1]]), n, dtype).view(torch.int16)
    assert base.view(torch.int16) != oc.expected_output(torch.tensor([[c + 1]]), n, dtype).view(torch.int16)


@pytest.mark.parametrize("D", [64, 128])
def test_census_tables_match_dense_masks(D):
    """band_census / blockmap_census / scatter_rows against counts over materialised element masks."""
    S = 700

    def brute(mask):
        out = []
        for enc in oc.ENCODINGS:
            onehot = torch.nn.functional.one_hot(oc.key_codes(S, D, enc), D).long()
            out.append(mask.long() @ onehot)
        return torch.stack(out), mask.sum(1)

    mod = oa.hy_mask_mod(48, 20, 4, 158, 1.3)
    dense = mod(torch.arange(S).view(-1, 1), torch.arange(S).view(1, -1))
    cnt, n = oc.band_census(mod, S, D, "cpu", row_chunk=128)
    rc, rn = brute(dense)
    assert torch.equal(cnt.long(), rc) and torch.equal(n, rn)

    g = torch.Generator().manual_seed(0)
    rows = torch.tensor([100, 0, 250, 1, 349])
    cols = torch.tensor([0, 120, 80, 0, 300, 200])
    bm = torch.rand(5, 6, generator=g) < 0.5
    key_ids = torch.randperm(S, generator=g)
    o_rows = torch.randperm(S, generator=g)
    cnt, n = oc.scatter_rows(*oc.blockmap_census(bm, rows, cols, D, key_ids), o_rows)
    elem = oa.block_mask_to_element_mask(bm, rows, cols)  # plan order: row r, key position p
    mask = torch.zeros(S, S, dtype=torch.bool)
    mask[o_rows[:, None], key_ids[None, :]] = elem          # output row o_rows[r], key identity key_ids[p]
    rc, rn = brute(mask)
    assert torch.equal(cnt, rc) and torch.equal(n, rn)
    # rows without keys produce exact zeros
    assert torch.all(oc.expected_output(cnt[0], n, torch.float16)[n == 0] == 0)
