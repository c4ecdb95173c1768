"""svgb_sample_mse against its closed form (oracle/smse_census.py) within the oracle's derived rounding bound.

Every case runs at a named split count: BH comes from the device's SM count (smse_cases.bh_for), the oracle's mirror
of smse_layout must agree with svgb_sample_mse_bytes (so the split count the oracle assumed is the one the kernel ran),
and the heads of a call are compared one by one with the closed form, with argmin(spatial, temporal) equal wherever
the two MSEs are further apart than their bounds.  Test ids name nsplit; "empty" marks trailing empty splits.
"""
import ctypes as C

import pytest
import torch

from oracle import smse_census as sc
from smse_cases import CASES, bh_for, build

pytestmark = pytest.mark.gpu


def n_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def run(case_obj, dtype, cuda):
    from svgb200 import core

    q, k, v = sc.tensors(case_obj, dtype, cuda)
    rows = case_obj.rows.to(cuda)
    L = sc.LAYOUTS[case_obj.lay]
    a = core.sample_mse(q, k, v, rows, L, case_obj.ctx, case_obj.F, case_obj.P)
    b = core.sample_mse(q, k, v, rows, L, case_obj.ctx, case_obj.F, case_obj.P)
    torch.cuda.synchronize()
    assert torch.equal(a.view(torch.int32), b.view(torch.int32)), "two calls differ"
    return a.double().cpu()


def check_layout(c, nsplit):
    from svgb200._lib import lib

    ns, cps, nch, nbytes = sc.layout(c.BH, c.S, c.D, n_sms())
    got = C.c_size_t()
    assert lib().svgb_sample_mse_bytes(c.BH, c.S, c.D, c.n, C.byref(got)) == 0
    assert got.value == nbytes, (got.value, nbytes)
    assert ns == nsplit, (ns, nsplit)
    empty = sum(1 for a, b in sc.split_ranges(c.S, ns) if b <= a)
    print(f"{c.lay} S={c.S} BH={c.BH} SMs={n_sms()}: nsplit={ns} cps={cps} n_chunks={nch} empty splits={empty}")
    return ns


def compare(got, want, bnd, label):
    bad = (got - want).abs() > bnd
    if bool(bad.any()):
        m, h = [int(x) for x in bad.nonzero()[0]]
        raise AssertionError(f"{label}: {int(bad.sum())} MSEs off, first mask {m} head {h}: kernel {float(got[m, h]):.9e}"
                             f" closed form {float(want[m, h]):.9e} bound {float(bnd[m, h]):.3e}")
    clear = (want[0] - want[1]).abs() > bnd[0] + bnd[1]
    assert torch.equal(got.argmin(0)[clear], want.argmin(0)[clear]), label


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_sample_mse_census(cuda, case):
    name, lay, ctx, F, P, D, dtype, n, nsplit, hot, seed = case
    c = build(case, bh_for(nsplit, n_sms()))
    ns = check_layout(c, nsplit)
    want, bnd = sc.bound(c, ns, device=cuda)
    got = run(c, dtype, cuda)
    compare(got, want, bnd, name)


@pytest.mark.parametrize("case", [CASES[0], CASES[4], CASES[9]], ids=[CASES[i][0] for i in (0, 4, 9)])
def test_same_head_at_every_split_count(cuda, case):
    """DESIGN.md §3: a different split count changes only the order of the LSE merge.  Heads 0..2 of one case at
    nsplit = 1, 2, 3 and the largest (32, or capped by the chunk count): equal within the two bounds."""
    dtype = case[6]
    res = []
    for target in (1, 2, 3, 32):
        c = build(case, bh_for(target, n_sms()))
        ns = check_layout(c, min(target, sc.layout(c.BH, c.S, c.D, n_sms())[2]))
        want, bnd = sc.bound(c, ns, device=cuda)
        got = run(c, dtype, cuda)
        compare(got, want, bnd, f"{case[0]} at nsplit {ns}")
        res.append((ns, got[:, :3], bnd[:, :3]))
    for ns, got, bnd in res[1:]:
        ns0, got0, bnd0 = res[0]
        assert bool(((got - got0).abs() <= bnd + bnd0).all()), (ns0, ns, got0, got)


def prod_rows(lay, ctx, F, P, n, seed, limit):
    from smse_cases import pick_rows

    rows = pick_rows(lay, ctx, F, P, 10 * n, seed)
    rows = rows[rows < limit][:n]
    return rows


@pytest.mark.parametrize("shape", [
    # HunyuanVideo 720p (bench.py): 64 rows below 10 000, per rank on 8 GPUs (3 heads), one GPU (24), cfg (48)
    ("hy", 256, 33, 3600, 24, 10000, True),
    ("hy", 256, 33, 3600, 48, 10000, True),
    ("hy", 256, 33, 3600, 3, 10000, False),
    # Wan 720p: S = 21 x 3600 = 75 600
    ("wan", 0, 21, 3600, 40, 75600, True),
    ("wan", 0, 21, 3600, 80, 75600, False),
    # CogVideoX: 226 text tokens first, 13 frames of 1350; rows over the whole sequence, text rows included
    ("cog", 226, 13, 1350, 30, 226 + 13 * 1350, True),
], ids=["hy720_bh24", "hy720_bh48", "hy720_bh3_census", "wan720_bh40", "wan720_bh80_census", "cog_bh30"])
def test_sample_mse_production_shapes(cuda, shape):
    lay, ctx, F, P, BH, limit, hot = shape
    D = 128
    rows = prod_rows(lay, ctx, F, P, 64, 21, limit)
    if lay == "cog":
        rows[:4] = torch.tensor([0, 1, ctx - 1, 100])  # text rows: every key spatially, none temporally
    c = sc.make_case(lay, ctx, F, P, D, BH, rows, hot=hot, seed=31)
    ns, _, _, _ = sc.layout(BH, c.S, D, n_sms())
    check_layout(c, ns)
    want, bnd = sc.bound(c, ns, device=cuda)
    got = run(c, torch.bfloat16, cuda)
    compare(got, want, bnd, f"{lay} BH={BH}")
