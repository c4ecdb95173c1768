"""Exact censuses of the attention backward, on every gradient element of every head (oracle/bwd_census.py).

Key census: Q, K, V, O, dO and lse chosen so that every score is 0, every P is 2^-L and every dS is +-2^-L, which
makes each stored dQ / dK / dV value a count of allowed (query, key) pairs times a power of two: the query-major
(dQ) and the key-major (dK, dV) launches are both checked against the forward's census tables and their transposes,
at full size.  Gradient census: small integers on real scores, values and deltas, every intermediate exact, so the
stored gradients equal the fp64 sums after the kernel's two roundings, on all eight backward instantiations.

Gradients are written into NaN-filled buffers (attn_bwd(..., out=)): an element no stream stores stays NaN and fails.
The comparison is by value, so the only two bit patterns it does not tell apart are +0 and -0.  The key-major band
plans are also checked structurally (every key in exactly one stream, each list exactly the query chunks with an
allowed pair, ELEM exactly where not every pair is allowed), which the census cannot see: a superfluous or
over-flagged chunk only costs time.  Budgets, representability, coverage and the oracle mutants are shown on the CPU
(tests/test_attention_bwd_census_cpu.py).
"""
import pytest
import torch

from oracle import bwd_census as bc
from oracle import census as oc

pytestmark = pytest.mark.gpu

DT = {"bf16": torch.bfloat16, "fp16": torch.float16}
NAMES = ("dq", "dk", "dv")


def to_layout(x, layout, B=1):
    """[BH, S, D] -> [B, BH / B, S, D] ('bhsd') or [S, BH, D] ('shd'), contiguous"""
    if layout == "shd":
        return x.transpose(0, 1).contiguous()
    return x.reshape(B, x.shape[0] // B, *x.shape[1:]).contiguous()


def from_layout(x, layout):
    return x.transpose(0, 1) if layout == "shd" else x.reshape(-1, *x.shape[2:])


def run_bwd(cuda, plan, tensors, lse, dtype, sm_scale, layout="bhsd", B=1):
    """attn_bwd on [BH, S, D] inputs in the given layout, into NaN-filled out= buffers -> [dq, dk, dv] [BH, S, D]"""
    from svgb200 import core

    q, k, v, o, do = (to_layout(t.to(dtype), layout, B).to(cuda) for t in tensors)
    out = tuple(torch.full_like(q, float("nan")) for _ in range(3))
    got = core.attn_bwd(q, k, v, o, do, lse.to(cuda), plan, layout=layout, sm_scale=sm_scale, out=out)
    assert all(g is b for g, b in zip(got, out))
    return [from_layout(g, layout).cpu() for g in got]


def first_bad(got, exp):
    """(row, column, rows differing) of the first element where got != exp by value (NaN never matches), or None"""
    bad = ~(got.float() == exp.float())
    if not bool(bad.any()):
        return None
    r, c = (int(x) for x in bad.nonzero()[0])
    return r, c, int(bad.any(1).sum())


# --------------------------------------------------------------------------------------------
# key census
# --------------------------------------------------------------------------------------------
def run_key(cuda, plan, tables, S, D, dtype, what, layout="bhsd", B=1):
    """tables[h] = (cnt [2, S, D'], n [S], cnt_t [2, S, D']) of head h."""
    n_rows = torch.stack([t[1] for t in tables])
    for enc in oc.ENCODINGS:
        *ts, lse = bc.key_inputs(S, D, enc, n_rows)
        got = run_bwd(cuda, plan, ts, lse, dtype, bc.KEY_SCALE, layout, B)
        exp, last = None, None
        for h, tab in enumerate(tables):
            if tab is not last:
                exp = bc.key_expected(tab[0][enc], tab[2][enc], S, D, enc)
                for name, e in zip(NAMES, exp):
                    assert torch.equal(e.to(dtype).double(), e), f"{what}: {name} leaves the exact range of {dtype}"
                last = tab
            for name, g, e in zip(NAMES, got, exp):
                b = first_bad(g[h], e.to(dtype))
                if b is not None:
                    r, c, nr = b
                    raise AssertionError(
                        f"{what}, encoding {enc}: {name} first differs at (head {h}, row {r}, column {c}) of {nr} rows: "
                        f"expected {float(e[r, c])!r}, kernel {float(g[h, r, c])!r}")


def check_band_plans(cuda, plan, args, mod, S, structure=True):
    """Both band plans' items against the planner's segment rules, and the key-major plan's lists against the mask.
    Returns the key-major plan's plan_stats."""
    stats = None
    for p, transposed in ((plan, False), (plan.key_major(), True)):
        (items,), chunks = bc.read_plan(p, 1)
        got = [(int(it[0, 0]), int(it[0, 1]) + int(it[1, 1])) for it in items]
        assert got == bc.band_items(args[0], args[1], args[2], S, transposed), f"transposed={transposed}: items"
        n0, n1 = items[:, 0, 1], items[:, 1, 1]
        assert bool(((n0 == torch.clamp(n0 + n1, max=128)) & (items[:, 1, 0] == items[:, 0, 0] + 128)).all())
        if transposed:
            stats = bc.plan_stats(items)
            if structure:
                msg = bc.check_band_t_structure(items, chunks, mod, S, cuda)
                assert msg is None, f"key-major band plan: {msg}"
    assert stats["two"]
    return stats


@pytest.mark.parametrize("kind,density", bc.KEY_BAND_FULL)
def test_key_census_band_fullsize(cuda, kind, density):
    """The forward census's full-size band list: HunyuanVideo 720p at 0.1, 0.3 and dense, Wan 720p at 0.2, 0.45 and
    the generic W = 4990, CogVideoX at 0.25 with and without the sink; fp16, D = 128, two heads."""
    from svgb200 import core

    args, mod, S = bc.key_band_case(kind, density)
    plan = core.plan_band(*args, 2, S, cuda)
    check_band_plans(cuda, plan, args, mod, S)
    tab = bc.band_tables(mod, S, 128, cuda)
    assert int(tab[0].max()) <= bc.MAX_COUNT[torch.float16] and int(tab[2].max()) <= bc.MAX_COUNT[torch.float16]
    run_key(cuda, plan, [tab] * 2, S, 128, torch.float16, f"band {kind} {density}")


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("case", bc.KEY_BAND_SMALL, ids=lambda c: "-".join(map(str, c)))
def test_key_census_band_small(cuda, case, D, dtype):
    """The forward census's small band list: widths 77, 1, 129, 254 and 255, mode NONE, S not a multiple of 128."""
    from svgb200 import core

    args, mod, S = bc.key_band_case(case)
    plan = core.plan_band(*args, 2, S, cuda)
    check_band_plans(cuda, plan, args, mod, S)
    run_key(cuda, plan, [bc.band_tables(mod, S, D, cuda)] * 2, S, D, DT[dtype], f"band {case} D={D} {dtype}")


def varblock_tables(bm, rows, cols, D):
    return [bc.blockmap_tables(bm[h], rows[h], cols[h], D) for h in range(bm.shape[0])]


@pytest.mark.parametrize("shape", ["hunyuan", "wan"])
def test_key_census_varblock_fullsize(cuda, shape):
    """The forward census's full-size variable-block maps (HunyuanVideo: 3 heads, QC = 402, KC = 1002; Wan: 2 heads,
    QC = 300, KC = 1000) with q-block AND key-block sizes from q_sizes: the key-major plan's rows are the key blocks,
    so its tail pairing and every r % 256 class are hit from that side too.  Empty q- and key blocks, an
    all-selected and an all-empty row (the "joined" head) and column (the "alternating" head)."""
    from svgb200 import core

    bm, rows, cols, S = bc.varblock_fullsize(shape)
    plan = core.plan_varblock(bm.to(cuda), rows.to(cuda), cols.to(cuda), S)
    H = bm.shape[0]
    for p in (plan, plan.key_major()):
        items, _ = bc.read_plan(p, H)
        st = [bc.plan_stats(it) for it in items]
        assert all(s["two"] and s["one"] for s in st), st
    run_key(cuda, plan, varblock_tables(bm, rows, cols, 128), S, 128, torch.float16, f"varblock {shape}")


@pytest.mark.parametrize("layout,B", [("bhsd", 1), ("shd", 1), ("bhsd", 2)], ids=["bhsd", "shd", "bhsd-B2"])
def test_key_census_varblock_small(cuda, layout, B):
    """The gradient census's variable-block map (S = 6000, edge block sizes on both sides, keyless rows, unreached
    keys, an empty key-major list paired with a non-empty one) in the [S, H, D] layout and with B = 2 (four heads,
    each with its own map); bf16, D = 128."""
    from svgb200 import core

    case = bc.grad_varblock_case(H=2 * B)
    plan = core.plan_varblock(case.bm.to(cuda), case.rows.to(cuda), case.cols.to(cuda), case.S)
    items, _ = bc.read_plan(plan.key_major(), case.H)
    assert bc.plan_stats(items[0])["empty_next"]
    run_key(cuda, plan, varblock_tables(case.bm, case.rows, case.cols, 128), case.S, 128, torch.bfloat16,
            f"varblock {layout} B={B}", layout=layout, B=B)


def bsr_plan(cuda, notes):
    from svgb200.ops import attention_ops

    F, P, text, Rb = notes["bsr"]
    plan = attention_ops.bsr_to_plan(notes["indptr"], notes["indices"], (Rb, Rb), F * P, text, cuda)
    assert plan.desc.items_stride == 0 and plan.key_major().desc.items_stride == 0
    return plan


def test_key_census_bsr_shared_plan(cuda):
    """One BSR plan, and its key-major plan, shared by both heads (items_stride = 0)."""
    case = bc.grad_bsr_case()
    plan = bsr_plan(cuda, case.notes)
    tab = bc.blockmap_tables(case.bm[0], case.rows[0], case.cols[0], 128)
    run_key(cuda, plan, [tab] * case.H, case.S, 128, torch.float16, "shared BSR plan")


# --------------------------------------------------------------------------------------------
# gradient census
# --------------------------------------------------------------------------------------------
def grad_plan(cuda, case):
    from svgb200 import core

    if "bsr" in case.notes:
        return bsr_plan(cuda, case.notes)
    if case.mod is not None:
        return core.plan_band(*case.band, case.H, case.S, cuda)
    return core.plan_varblock(case.bm.to(cuda), case.rows.to(cuda), case.cols.to(cuda), case.S)


def run_grad(cuda, case, dtype, what, layout="bhsd", B=1):
    plan = grad_plan(cuda, case)
    got = run_bwd(cuda, plan, (case.q, case.k, case.v, case.o, case.do), case.lse(), dtype, case.sm_scale, layout, B)
    for h in range(case.H):
        _, budget, stats = bc.grad_exact(case, h, cuda)
        assert max(budget) < bc.BUDGET and stats["ds_exact"] and stats["ds_max"] <= 8, f"{what}: head {h} not exact"
        for name, g, e in zip(NAMES, got, bc.grad_expected(case, h, dtype, cuda)):
            b = first_bad(g[h], e.cpu())
            if b is not None:
                r, c, nr = b
                raise AssertionError(f"{what}: {name} first differs at (head {h}, row {r}, column {c}) of {nr} rows: "
                                     f"expected {float(e[r, c])!r}, kernel {float(g[h, r, c])!r}")


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("name", list(bc.GRAD_BAND))
def test_grad_census_band(cuda, name, D, dtype):
    """HunyuanVideo, Wan, CogVideoX and mode NONE at S = 1, 64, 65 and 127 mod 128; with both directions, all eight
    backward instantiations (D 64 / 128 x bf16 / fp16 x query- / key-major)."""
    run_grad(cuda, bc.grad_band_case(name, D=D), DT[dtype], f"band {name} D={D} {dtype}")


@pytest.mark.parametrize("c", [0.5, 2.0])
def test_grad_census_scale(cuda, c):
    """sm_scale giving c = 1/2 and 2 exactly: the score scale of P and the sm_scale epilogue of dQ and dK."""
    run_grad(cuda, bc.grad_band_case("hy", c=c), torch.bfloat16, f"band hy c={c}")


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("D", [64, 128])
def test_grad_census_varblock(cuda, D, dtype):
    """Variable-block plan with edge block sizes on both sides, keyless rows and unreached keys."""
    run_grad(cuda, bc.grad_varblock_case(D=D), DT[dtype], f"varblock D={D} {dtype}")


@pytest.mark.parametrize("layout,B", [("shd", 1), ("bhsd", 2)], ids=["shd", "bhsd-B2"])
def test_grad_census_layouts(cuda, layout, B):
    """The [S, H, D] layout, and B = 2 in [B, H, S, D] (four heads with their own maps)."""
    run_grad(cuda, bc.grad_varblock_case(H=2 * B), torch.bfloat16, f"varblock {layout} B={B}", layout, B)


def test_grad_census_bsr_shared_plan(cuda):
    run_grad(cuda, bc.grad_bsr_case(), torch.float16, "shared BSR plan")
