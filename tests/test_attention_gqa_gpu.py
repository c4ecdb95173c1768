"""Grouped-query attention on the GPU (svgb_attn_fwd_gqa / svgb_attn_bwd_gqa through core).

Exact checks.  The GQA forward and dQ run the MHA kernels' row operations in the same order, so o, lse and dq are
compared bit for bit with the MHA call on K / V repeated per group (repeat_interleave over the head dimension) under
the map repeated per query head.  dK / dV sum G query heads in one accumulator, so they are checked with the key census
(oracle/bwd_census.py) on every head of a group: each stored value is then the group's allowed-pair count times a power
of two, exact while key_counts_representable holds.  Gradients go into NaN-filled out= buffers.
Against fp64: dK / dV (and dQ, o) of core.attention under autograd against tests/gqa_fp64.py, with the tolerances of
test_attention_bwd_gpu.py; the patched flash_attn_varlen_func against scaled_dot_product_attention(enable_gqa=True).
"""
import pytest
import torch

from oracle import bwd_census as bc
from oracle import census as oc

pytestmark = pytest.mark.gpu

TOL = {torch.bfloat16: 4e-2, torch.float16: 1e-2}
MASK_NONE, MASK_HY, MASK_WAN, MASK_COG = 0, 1, 2, 3
BANDS = {  # (mode, m0, m1, m2, S), the band shapes of test_attention_bwd_gpu.py
    "hy": (MASK_HY, 300, 320, 150, 344),
    "wan": (MASK_WAN, 100, 0, 130, 300),
    "cog": (MASK_COG, 20, 20, 140, 320),
}


def partition(n, blocks, gen):
    cuts, _ = torch.sort(torch.randperm(n - 1, generator=gen)[: blocks - 1] + 1)
    return torch.diff(torch.cat([torch.tensor([0]), cuts, torch.tensor([n])])).to(torch.int32)


def varblock(Hkv, Sq, Skv, MB, NB, density, gen):
    """(map [Hkv, MB, NB], row sizes, column sizes): random partitions, map entries kept with probability density"""
    rows = torch.stack([partition(Sq, MB, gen) for _ in range(Hkv)])
    cols = torch.stack([partition(Skv, NB, gen) for _ in range(Hkv)])
    return torch.rand(Hkv, MB, NB, generator=gen) < density, rows, cols


def element_masks(bm, rows, cols, G):
    """bool [Hkv * G, Sq, Skv]: the element mask of query head h is its key/value head h // G's"""
    from oracle.attention import block_mask_to_element_mask

    return torch.stack([block_mask_to_element_mask(bm[h], rows[h], cols[h]) for h in range(bm.shape[0])]
                       ).repeat_interleave(G, 0)


def plans(cuda, bm, rows, cols, Sq, Skv, G):
    """(GQA plan over the key/value heads, MHA plan of the map repeated per query head)"""
    from svgb200 import core

    args = [(t.to(cuda), r.to(cuda), c.to(cuda)) for t, r, c in ((bm, rows, cols), (bm.repeat_interleave(G, 0),
                                                                 rows.repeat_interleave(G, 0),
                                                                 cols.repeat_interleave(G, 0)))]
    return [core.plan_varblock(*a, Sq, S_kv=Skv) for a in args]


def lay(x, layout, B):
    """[BH, S, D] -> [B, BH / B, S, D] ('bhsd') or [S, BH, D] ('shd', B = 1), contiguous"""
    return x.transpose(0, 1).contiguous() if layout == "shd" else x.reshape(B, -1, *x.shape[1:]).contiguous()


def unlay(x, layout):
    return x.transpose(0, 1) if layout == "shd" else x.reshape(-1, *x.shape[2:])


def repeat_kv(x, G):
    return x.repeat_interleave(G, 1).contiguous()  # the head dimension is 1 in both layouts


def run_both(cuda, plan_g, plan_m, Hq, Hkv, Sq, Skv, D, dtype, layout="bhsd", B=1, seed=0):
    """o, lse, dq, dk, dv of the GQA call and of the MHA call on repeated K / V (gradients into NaN buffers)"""
    from svgb200 import core

    g = torch.Generator().manual_seed(seed)
    q, do = (lay(torch.randn(B * Hq, Sq, D, generator=g).to(dtype), layout, B).to(cuda) for _ in range(2))
    k, v = (lay(torch.randn(B * Hkv, Skv, D, generator=g).to(dtype), layout, B).to(cuda) for _ in range(2))
    out = []
    for kk, vv, p in ((k, v, plan_g), (repeat_kv(k, Hq // Hkv), repeat_kv(v, Hq // Hkv), plan_m)):
        o, lse = core.attn_fwd(q, kk, vv, p, layout=layout, return_lse=True)
        grads = tuple(torch.full_like(t, float("nan")) for t in (q, kk, vv))
        core.attn_bwd(q, kk, vv, o, do, lse, p, layout=layout, out=grads)
        out.append((o, lse) + grads)
    return out


def check_exact(got, ref, G, dtype, layout, what):
    (o, lse, dq, dk, dv), (o_m, lse_m, dq_m, dk_m, dv_m) = got, ref
    for name, a, b in (("o", o, o_m), ("lse", lse, lse_m), ("dq", dq, dq_m)):
        assert torch.equal(a, b), f"{what}: {name} differs from MHA on repeated K/V in {int((a != b).sum())} elements"
    for name, a, b in (("dk", dk, dk_m), ("dv", dv, dv_m)):
        a = unlay(a, layout).float()
        b = unlay(b, layout).float()
        ref = b.reshape(-1, G, *b.shape[1:]).sum(1)  # fp32 group sum of the MHA heads
        assert torch.isfinite(a).all(), f"{what}: {name} has unwritten (NaN) elements"
        err = float((a - ref).abs().max())
        assert err <= TOL[dtype] * float(ref.abs().max()) + 1e-6, f"{what}: {name} max error {err}"


GRID = [(hq, hkv, s, mb, nb, d) for hq, hkv in ((4, 1), (16, 4), (16, 1)) for s in (256, 4096)
        for mb, nb in ((10, 50), (20, 100)) for d in (0.2, 0.7)]


@pytest.mark.parametrize("Hq,Hkv,S,MB,NB,density", GRID)
def test_reference_grid_matches_repeated_mha(cuda, Hq, Hkv, S, MB, NB, density):
    """The reference's variable-block parity grid with its Hkv axis: o, lse, dq bit for bit, dk / dv the group sums;
    bf16, D = 128."""
    gen = torch.Generator().manual_seed(Hq * 1000 + Hkv * 100 + S + MB + int(density * 10))
    G = Hq // Hkv
    bm, rows, cols = varblock(Hkv, S, S, MB, NB, density, gen)
    pg, pm = plans(cuda, bm, rows, cols, S, S, G)
    check_exact(*run_both(cuda, pg, pm, Hq, Hkv, S, S, 128, torch.bfloat16), G, torch.bfloat16, "bhsd",
                f"Hq={Hq} Hkv={Hkv} S={S} {MB}x{NB} {density}")


@pytest.mark.parametrize("layout,B", [("bhsd", 1), ("shd", 1), ("bhsd", 2)])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_dtypes_layouts_batch(cuda, dtype, D, layout, B):
    """Both 16-bit types, both head dims, both layouts, and B = 2 (query head b * Hq + h reads key/value head
    b * Hkv + h // G, with its own map)."""
    gen = torch.Generator().manual_seed(D + B)
    Hq, Hkv, S = 6, 2, 1000
    bm, rows, cols = varblock(B * Hkv, S, S, 9, 33, 0.5, gen)
    pg, pm = plans(cuda, bm, rows, cols, S, S, Hq // Hkv)
    check_exact(*run_both(cuda, pg, pm, Hq, Hkv, S, S, D, dtype, layout, B), Hq // Hkv, dtype, layout,
                f"{dtype} D={D} {layout} B={B}")


@pytest.mark.parametrize("Sq,Skv", [(1000, 300), (300, 1000), (75600 // 8, 512)])
def test_rectangular(cuda, Sq, Skv):
    """GQA with keys of another length (a rectangular plan over the key/value heads)."""
    gen = torch.Generator().manual_seed(Sq + Skv)
    Hq, Hkv = 8, 2
    bm, rows, cols = varblock(Hkv, Sq, Skv, 7, 3, 0.6, gen)
    pg, pm = plans(cuda, bm, rows, cols, Sq, Skv, Hq // Hkv)
    check_exact(*run_both(cuda, pg, pm, Hq, Hkv, Sq, Skv, 128, torch.bfloat16), Hq // Hkv, torch.bfloat16, "bhsd",
                f"Sq={Sq} Skv={Skv}")


@pytest.mark.parametrize("band", sorted(BANDS))
def test_band_masks(cuda, band):
    """The HY / WAN / COG band masks: one plan for every head, GQA or not."""
    from svgb200 import core

    mode, m0, m1, m2, S = BANDS[band]
    Hq, Hkv = 8, 2
    p = core.plan_band(mode, m0, m1, m2, Hkv, S, cuda)
    check_exact(*run_both(cuda, p, p, Hq, Hkv, S, S, 128, torch.float16), Hq // Hkv, torch.float16, "bhsd", band)


# --------------------------------------------------------------------------------------------
# dK / dV key census over groups
# --------------------------------------------------------------------------------------------
def run_key_gqa(cuda, plan, tables, S, D, dtype, G, what):
    """tables[h] = (cnt, n, cnt_t) of key/value head h; every query head of its group gets the census inputs, so dk
    and dv are G times the one-head closed form and dq is the one-head closed form."""
    from svgb200 import core

    Hkv = len(tables)
    n_rows = torch.stack([t[1] for t in tables]).repeat_interleave(G, 0)
    for enc in oc.ENCODINGS:
        q, k, v, o, do, lse = bc.key_inputs(S, D, enc, n_rows)
        q, o, do = (t.to(dtype)[None].contiguous().to(cuda) for t in (q, o, do))
        k, v = (t[:Hkv].to(dtype)[None].contiguous().to(cuda) for t in (k, v))
        out = tuple(torch.full_like(t, float("nan")) for t in (q, k, v))
        dq, dk, dv = (t[0].cpu() for t in core.attn_bwd(q, k, v, o, do, lse.to(cuda), plan, sm_scale=bc.KEY_SCALE,
                                                         out=out))
        for h, tab in enumerate(tables):
            eq, ek, ev = bc.key_expected(tab[0][enc], tab[2][enc], S, D, enc)
            for name, got, e in (("dk", dk[h], G * ek), ("dv", dv[h], G * ev)) + tuple(
                    ("dq", dq[h * G + g], eq) for g in range(G)):
                assert torch.equal(e.to(dtype).double(), e), f"{what}: {name} leaves the exact range of {dtype}"
                bad = ~(got.float() == e.to(dtype).float())
                if bool(bad.any()):
                    r, c = (int(x) for x in bad.nonzero()[0])
                    raise AssertionError(f"{what}, encoding {enc}: {name} of head {h} first differs at ({r}, {c}): "
                                         f"expected {float(e[r, c])!r}, kernel {float(got[r, c])!r}")


@pytest.mark.parametrize("G", [2, 4])
@pytest.mark.parametrize("case", [("generic_wan", 50, 0, 77, 1100), ("generic_hy", 900, 1000, 255, 1093)],
                         ids=lambda c: "-".join(map(str, c)))
def test_key_census_band(cuda, case, G):
    from svgb200 import core

    args, mod, S = bc.key_band_case(case)
    tab = bc.band_tables(mod, S, 128, cuda)
    assert bc.key_counts_representable(G * max(int(tab[0].max()), int(tab[2].max())), torch.float16)
    plan = core.plan_band(*args, 2, S, cuda)
    run_key_gqa(cuda, plan, [tab] * 2, S, 128, torch.float16, G, f"band {case} G={G}")


@pytest.mark.parametrize("G,dtype", [(2, torch.bfloat16), (3, torch.float16)])
def test_key_census_varblock(cuda, G, dtype):
    """The gradient census's variable-block map (keyless rows, unreached keys, edge block sizes) over two key/value
    heads, each shared by G query heads (up to 128 pairs per count: G = 3 leaves bf16's exact range, so fp16)."""
    from svgb200 import core

    case = bc.grad_varblock_case(H=2)
    tabs = [bc.blockmap_tables(case.bm[h], case.rows[h], case.cols[h], 128) for h in range(2)]
    top = max(max(int(t[0].max()), int(t[2].max())) for t in tabs)
    assert bc.key_counts_representable(G * top, dtype), top
    plan = core.plan_varblock(case.bm.to(cuda), case.rows.to(cuda), case.cols.to(cuda), case.S)
    run_key_gqa(cuda, plan, tabs, case.S, 128, dtype, G, f"varblock G={G}")


def test_deterministic_and_launch_counts(cuda):
    """Two backward runs give the same bits; GQA and MHA calls make one forward launch and three backward launches."""
    from svgb200 import core

    gen = torch.Generator().manual_seed(5)
    Hq, Hkv, S, D = 8, 2, 2000, 128
    bm, rows, cols = varblock(Hkv, S, S, 9, 33, 0.5, gen)
    pg, pm = plans(cuda, bm, rows, cols, S, S, Hq // Hkv)
    pg.key_major(), pm.key_major()
    q, do = (torch.randn(1, Hq, S, D, generator=gen).to(torch.bfloat16).to(cuda) for _ in range(2))
    k, v = (torch.randn(1, Hkv, S, D, generator=gen).to(torch.bfloat16).to(cuda) for _ in range(2))
    for kk, vv, p in ((k, v, pg), (repeat_kv(k, 4), repeat_kv(v, 4), pm)):
        n0 = core.launch_count
        o, lse = core.attn_fwd(q, kk, vv, p, return_lse=True)
        assert core.launch_count - n0 == 1
        n0 = core.launch_count
        a = core.attn_bwd(q, kk, vv, o, do, lse, p)
        assert core.launch_count - n0 == 3
        b = core.attn_bwd(q, kk, vv, o, do, lse, p)
        assert all(torch.equal(x, y) for x, y in zip(a, b))


# --------------------------------------------------------------------------------------------
# against fp64
# --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("kind", ["hy", "wan", "vb0.5", "rect"])
def test_attention_autograd_vs_fp64(cuda, kind, dtype, D):
    """core.attention under autograd with GQA leaves (Hq = 6, Hkv = 2 and, for vb, Hkv = 1): o, dq, dk, dv against
    the fp64 oracle."""
    import gqa_fp64
    from oracle.attention import generic_mask_fn
    from svgb200 import core

    gen = torch.Generator().manual_seed(D + len(kind))
    Hq, Hkv = 6, (1 if kind == "vb0.5" else 2)
    if kind in BANDS:
        mode, m0, m1, m2, S = BANDS[kind]
        Skv = S
        plan = core.plan_band(mode, m0, m1, m2, Hkv, S, cuda)
        masks = generic_mask_fn(mode, m0, m1, m2)(torch.arange(S).view(-1, 1), torch.arange(S).view(1, -1))
        masks = masks.expand(Hq, S, S)
    else:
        S, Skv = (1000, 1000) if kind == "vb0.5" else (700, 300)
        bm, rows, cols = varblock(Hkv, S, Skv, 9, 5, 0.5, gen)
        plan = core.plan_varblock(bm.to(cuda), rows.to(cuda), cols.to(cuda), S, S_kv=Skv)
        masks = element_masks(bm, rows, cols, Hq // Hkv)
    q, do = (torch.randn(Hq, S, D, generator=gen).to(dtype) for _ in range(2))
    k, v = (torch.randn(Hkv, Skv, D, generator=gen).to(dtype) for _ in range(2))
    x = [t[None].to(cuda).requires_grad_() for t in (q, k, v)]
    o = core.attention(*x, plan)
    o.backward(do[None].to(cuda))
    ref = gqa_fp64.gqa_grads(q, k, v, do, masks)
    for name, g, r in zip(("o", "dq", "dk", "dv"), (o.detach(),) + tuple(t.grad for t in x), ref):
        g = g[0].double().cpu()
        assert g.shape == r.shape and torch.isfinite(g).all(), name
        err = float((g - r).abs().max())
        assert err <= TOL[dtype] * float(r.abs().max()) + 1e-6, f"{name}: max error {err} vs {float(r.abs().max())}"


def test_flash_attn_varlen_gqa_vs_sdpa(cuda):
    """The patched flash_attn_varlen_func with k, v of fewer heads ([L, H, D], nheads_k | nheads) against
    scaled_dot_product_attention(enable_gqa=True) per segment, for both the forward and the gradients."""
    from svgb200 import patch

    gen = torch.Generator().manual_seed(9)
    Hq, Hkv, D = 8, 2, 128
    seg_q, seg_kv = [700, 77, 300], [500, 77, 129]
    cu_q = torch.tensor([0, 700, 777, 1077], dtype=torch.int32)
    cu_kv = torch.tensor([0, 500, 577, 706], dtype=torch.int32)
    q = torch.randn(sum(seg_q), Hq, D, generator=gen).to(torch.bfloat16).to(cuda).requires_grad_()
    k, v = (torch.randn(sum(seg_kv), Hkv, D, generator=gen).to(torch.bfloat16).to(cuda).requires_grad_()
            for _ in range(2))
    do = torch.randn(sum(seg_q), Hq, D, generator=gen).to(torch.bfloat16).to(cuda)
    o = patch.flash_attn_varlen_func(q, k, v, cu_q, cu_kv, max(seg_q), max(seg_kv))
    o.backward(do)
    got = [o.detach(), q.grad, k.grad, v.grad]
    x = [t.detach().double().requires_grad_() for t in (q, k, v)]
    outs = []
    for (a, b), (c, d) in zip(zip(cu_q[:-1].tolist(), cu_q[1:].tolist()), zip(cu_kv[:-1].tolist(), cu_kv[1:].tolist())):
        seg = [t.transpose(0, 1)[None] for t in (x[0][a:b], x[1][c:d], x[2][c:d])]
        outs.append(torch.nn.functional.scaled_dot_product_attention(*seg, enable_gqa=True)[0].transpose(0, 1))
    ref_o = torch.cat(outs)
    ref_o.backward(do.double())
    for name, g, r in zip(("o", "dq", "dk", "dv"), got, [ref_o.detach()] + [t.grad for t in x]):
        err = float((g.double() - r).abs().max())
        assert err <= TOL[torch.bfloat16] * float(r.abs().max()), f"{name}: max error {err}"


# --------------------------------------------------------------------------------------------
# production size
# --------------------------------------------------------------------------------------------
def test_wan_720p_varblock(cuda):
    """Wan 2.1 720p: 40 query heads over 8 key/value heads, 75 600 tokens, an SVG2-like map (300 x 1000 clusters)
    at density ~0.3."""
    gen = torch.Generator().manual_seed(720)
    Hq, Hkv, S = 40, 8, 75600
    bm, rows, cols = varblock(Hkv, S, S, 300, 1000, 0.3, gen)
    pg, pm = plans(cuda, bm, rows, cols, S, S, Hq // Hkv)
    check_exact(*run_both(cuda, pg, pm, Hq, Hkv, S, S, 128, torch.bfloat16), Hq // Hkv, torch.bfloat16, "bhsd",
                "wan 720p")


def test_hunyuan_720p_band(cuda):
    """HunyuanVideo 720p band (SVG1 spatial-temporal mask, 33 frames of 3600 tokens and 256 text tokens): 24 query
    heads over 8 key/value heads."""
    from oracle import attention as oa
    from svgb200 import core

    c = bc.HY720
    mul = oa.sparsity_to_width(0.3, c["ctx"], c["F"], c["P"])
    args, _ = oc.band_args("hy", c["F"], c["P"], c["ctx"], c["plen"], mul)
    S = c["ctx"] + c["F"] * c["P"]
    p = core.plan_band(*args, 8, S, cuda)
    check_exact(*run_both(cuda, p, p, 24, 8, S, S, 128, torch.bfloat16), 3, torch.bfloat16, "bhsd", "hunyuan 720p")
