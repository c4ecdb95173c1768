"""sample_mse's closed-form oracle on the CPU (oracle/smse_census.py), and svgb_sample_mse's argument refusals.

The GPU suite (test_sample_mse_census_gpu.py) compares the kernel with the closed form within the rounding bound the
oracle derives.  Here: every plausible bug of the sample_mse flow (smse_census.MUTATIONS) moves some GPU case by at
least 10x that bound; the inputs are exact in bf16 and fp16 and keep their hot / cold gap; the closed form agrees with
the fp32 oracle (oracle.attention.sample_mse); the split simulation matches the closed form at every split count.
The refusals need the built library but no GPU: each must come back before the device is queried.
"""
import ctypes as C
import math
from pathlib import Path

import pytest
import torch

from oracle import attention as oa
from oracle import smse_census as sc
from smse_cases import CASES, build

ROOT = Path(__file__).resolve().parent.parent
CPU_HEADS = 3  # heads 0..2 of every case (a head does not depend on BH)


@pytest.fixture(scope="module")
def cpu_cases():
    out = []
    for case in CASES:
        c = build(case, CPU_HEADS)
        mse, b = sc.bound(c, case[8])
        out.append((case, c, mse, b))
    return out


@pytest.mark.parametrize("mutation", sc.MUTATIONS)
def test_every_mutant_moves_a_gpu_case_past_ten_bounds(cpu_cases, mutation):
    best = 0.0
    for case, c, mse, b in cpu_cases:
        got = sc.simulate(c, case[8], mutation)
        moved = (got - mse).abs() / b
        if bool(torch.isnan(got).any()):
            return
        best = max(best, float(moved.max()))
        if best >= 10:
            return
    raise AssertionError(f"{mutation}: largest move {best:.2f} bounds")


def test_bounds_are_small(cpu_cases):
    """the stated bound stays a small fraction of the MSE: the tests compare to within ~1e-4 relative or better"""
    for case, c, mse, b in cpu_cases:
        assert bool((b <= 1e-3 * mse.abs() + 1e-9).all()), (case[0], b, mse)


@pytest.mark.parametrize("nsplit", [1, 2, 3, 5, 7, 32])
def test_split_simulation_equals_closed_form(nsplit):
    """any split partition, empty splits included, merges back to cnt / n"""
    for case in CASES[:2] + CASES[8:9]:
        c = build(case, 2)
        cf = sc.closed_form(c)
        assert torch.allclose(sc.simulate(c, nsplit), cf, rtol=1e-12, atol=0), case[0]


def test_inputs_exact_and_gap_holds():
    for case in CASES:
        c = build(case, 2)
        for dt in (torch.bfloat16, torch.float16):
            q, k, v = sc.tensors(c, dt, "cpu")
            q32, k32, v32 = sc.tensors(c, torch.float32, "cpu")
            assert torch.equal(q.float(), q32) and torch.equal(k.float(), k32) and torch.equal(v.float(), v32)
        s = sc.HOT_Q * sc.HOT_K
        assert math.log2(s) == int(math.log2(s))  # power of two: p = 1 exactly for hot keys
        gap = s * math.log2(math.e) / math.sqrt(c.D)
        assert gap >= 259, gap  # ex2(-gap) is 0 in fp32: cold keys vanish next to hot ones
        # every key holds one class entry and every sampled position one class entry
        assert int((k32 != 0).sum(-1).max()) <= 1 and int((q32 != 0).sum(-1).max()) <= 1
        # the full pass's hot tier of a row stays far below fp32's exact-integer range
        assert int(c.S) < 2 ** 24


@pytest.mark.parametrize("case", [CASES[0], CASES[3], CASES[5], CASES[6], CASES[8], CASES[10]], ids=lambda x: x[0])
def test_closed_form_matches_fp32_oracle(case):
    c = build(case, 2)
    q, k, v = sc.tensors(c, torch.float32, "cpu")
    masks = [sc.mask_rows(c.lay, X, c.rows, c.ctx, c.F, c.P) for X in ("spatial", "temporal")]
    ref = oa.sample_mse(q[None], k[None], v[None], c.rows, masks)[:, 0].double()
    cf = sc.closed_form(c)
    # a row that sees no key (COG text rows under the temporal mask) is NaN in the reference and 0 here
    empty = [bool((m.sum(1) == 0).any()) for m in masks]
    for x in range(2):
        if empty[x]:
            assert bool(torch.isnan(ref[x]).all())
            continue
        # fp32 softmax over S keys and fp32 squares: a few 1e-6 relative
        assert torch.allclose(ref[x], cf[x], rtol=2e-5, atol=1e-12), (x, ref[x], cf[x])


def test_layout_mirror_split_partition():
    # n_chunks = 33 at nsplit = 32: cps = 2, splits 17..31 empty, split 16 ends on the partial chunk
    ns, cps, nch, _ = sc.layout(4, 4200, 64, 132)
    assert (ns, cps, nch) == (32, 2, 33)
    r = sc.split_ranges(4200, ns)
    assert r[16] == (4096, 4200) and all(b <= a for a, b in r[17:])
    assert sc.layout(200, 1000, 64, 132)[0] == 1 and sc.layout(44, 119056, 128, 132)[0] == 3
    assert sc.layout(1, 700, 128, 132)[0] == 6  # capped by the chunk count


# --------------------------------------------------------------------------------------------
# C ABI refusals: before the device query, so they hold on a machine without a GPU
# --------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    import importlib.util

    spec = importlib.util.spec_from_file_location("svgb200_build", ROOT / "sparse-videogen_b200" / "build.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.build_lib()
    from svgb200 import _lib

    return _lib.lib()


# BH, S, D, dtype, layout, ctx, F, P -> reason in the message
REFUSALS = [
    ("e4m3", (2, 1024, 128, 2, 0, 0, 4, 256), b"16-bit"),
    ("f32", (2, 1024, 128, 3, 0, 0, 4, 256), b"16-bit"),
    ("dtype_neg", (2, 1024, 128, -1, 0, 0, 4, 256), b"16-bit"),
    ("layout3", (2, 1024, 128, 0, 3, 0, 4, 256), b"layout 3 unsupported"),
    ("seq_len", (2, 1000, 128, 0, 0, 0, 4, 256), b"seq_len 1000 != ctx 0 + F 4 * P 256"),
    ("wan_ctx", (2, 1056, 128, 1, 1, 32, 4, 256), b"WAN layout has no text tokens"),
    ("cog_ctx", (2, (1 << 19) + 1024, 128, 0, 2, 1 << 19, 4, 256), b"context length 524288 too large"),
    ("thres", (2, 4 * 350000, 128, 0, 0, 0, 4, 350000), b"band threshold 4101 too large"),
]


@pytest.mark.parametrize("args,reason", [r[1:] for r in REFUSALS], ids=[r[0] for r in REFUSALS])
def test_sample_mse_refuses_before_any_device_work(lib, args, reason):
    BH, S, D, dtype, layout, ctx, F, P = args
    fake = C.c_void_p(256)  # never dereferenced: the call must return first
    mse = C.c_void_p(256)
    rc = lib.svgb_sample_mse(fake, fake, fake, fake, 64, BH, S, D, dtype, layout, ctx, F, P, mse, fake,
                             C.c_size_t(1 << 40), None)
    msg = lib.svgb_last_error()
    assert rc < 0
    assert reason in msg, msg
    assert b"cuda" not in msg.lower()
