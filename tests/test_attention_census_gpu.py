"""Exact census of the attention kernel's executed mask, on every row of every head (oracle/census.py).

q = 0 turns every allowed score into 0 and every masked one into -inf, so the kernel's l is the number of allowed keys
and, with a one-hot key-identity V, its output is round16(count / n) per column: the test compares the output BIT FOR
BIT and exp(lse) to the key count of every row.  One key wrongly kept or dropped anywhere fails the test and the
message names the first differing (head, row).  The expected tables come from the oracle's mask predicates and block
maps, never from the engine.  The distinguishability of every table is proven on the CPU
(tests/test_census_cpu.py).
"""
import pytest
import torch

from oracle.census import band_args as _band_args
from oracle.census import partition as _partition
from oracle.census import q_sizes as _q_sizes
from oracle.census import varblock_head as _varblock_head

pytestmark = pytest.mark.gpu

# the HunyuanVideo 720p and Wan 2.1 720p shapes of BASELINE.json, and a CogVideoX-like one
HY = dict(ctx=256, F=33, P=3600, plen=71)
WAN = dict(F=21, P=3600)
COG = dict(ctx=226, F=13, P=1350)


def check_census(o, lse, cnt, n, enc, what):
    """o [H, S, D] kernel output, lse [H, S]; cnt[h] [2, S, D], n[h] [S]: expected tables in output-row order."""
    from oracle import census as oc

    o, lse = o.cpu(), lse.cpu()
    for h in range(o.shape[0]):
        exp_o = oc.expected_output(cnt[h][enc], n[h], o.dtype)
        nh = n[h].cpu()
        bad_o = (o[h].view(torch.int16) != exp_o.view(torch.int16)).any(1)
        live = nh > 0
        lse_h = lse[h].double()
        bad_l = torch.where(live, ~((lse_h.exp() - nh.double()).abs() < 0.5), lse_h != float("-inf"))
        bad = bad_o | bad_l
        if bool(bad.any()):
            r = int(bad.nonzero()[0])
            col = int((o[h, r].view(torch.int16) != exp_o[r].view(torch.int16)).nonzero()[0]) if bad_o[r] else 0
            raise AssertionError(
                f"{what}, encoding {enc}: first differing (head {h}, row {r}) of {int(bad.sum())} rows: expected "
                f"n = {int(nh[r])}, exp(lse) = {float(lse_h[r].exp()):.3f}; column {col}: expected count "
                f"{int(cnt[h][enc][r, col])} -> {float(exp_o[r, col])!r}, kernel {float(o[h, r, col])!r} "
                f"(~{float(o[h, r, col]) * max(int(nh[r]), 1):.2f} keys)")


def bound_ok(cnt, out_dtype):
    from oracle import census as oc

    assert max(int(c.max()) for c in cnt) < oc.COUNT_LIMIT[out_dtype], "a count left the range where one key shows"


def run_band(cuda, mode, m0, m1, m2, mod, H, S, D):
    from oracle import census as oc
    from svgb200 import core

    plan = core.plan_band(mode, m0, m1, m2, H, S, cuda)
    cnt, n = oc.band_census(mod, S, D, cuda)
    cnt, n = cnt.cpu(), n.cpu()
    bound_ok([cnt], torch.float16)
    q = torch.zeros(1, H, S, D, dtype=torch.float16, device=cuda)
    k = torch.randn(1, H, S, D, device=cuda).half()
    for enc in oc.ENCODINGS:
        v = oc.identity_values(S, D, enc, H, torch.float16, cuda)
        o, lse = core.attn_fwd(q, k, v, plan, return_lse=True)
        check_census(o[0], lse, [cnt] * H, [n] * H, enc, f"band mode {mode} m=({m0},{m1},{m2}) S={S} D={D}")


@pytest.mark.parametrize("kind,density", [("hy", 0.1), ("hy", 0.3), ("hy", "dense"), ("wan", 0.2), ("wan", 0.45),
                                          ("wan_generic", 4990), ("cog", 0.25), ("cog_sink", 0.25)])
def test_census_band_fullsize(cuda, kind, density):
    """SVG1 band plans at full size: HunyuanVideo 720p (text last, 71 prompt + 185 padding rows), Wan 720p
    (first-frame sink), CogVideoX-like (text first, with and without the attention sink).  The widths of the
    reference are multiples of 128; "dense" has W >= S.  wan_generic: the engine's Wan mask with W = 4990
    (= 126 mod 128): the last column of the chunk [q0 + W - 126, q0 + W + 2) is masked for the first row of every
    256-row item and allowed for all its other rows, so the plan's all-rows vote decides that key."""
    from oracle import attention as oa

    if kind == "wan_generic":
        S = WAN["F"] * WAN["P"]
        run_band(cuda, 2, WAN["P"], 0, density, oa.generic_mask_fn(2, WAN["P"], 0, density), 2, S, 128)
        return
    if kind == "hy":
        c = HY
        mul = 40.0 if density == "dense" else oa.sparsity_to_width(density, c["ctx"], c["F"], c["P"])
        args, mod = _band_args("hy", c["F"], c["P"], c["ctx"], c["plen"], mul)
        S = c["ctx"] + c["F"] * c["P"]
        if density == "dense":
            assert args[3] >= S
    elif kind == "wan":
        c = WAN
        args, mod = _band_args("wan", c["F"], c["P"], 0, 0, oa.sparsity_to_width(density, 0, c["F"], c["P"]))
        S = c["F"] * c["P"]
    else:
        c = COG
        mul = oa.sparsity_to_width(density, c["ctx"], c["F"], c["P"])
        args, mod = _band_args("cog", c["F"], c["P"], c["ctx"], c["ctx"], mul, attn_sink=kind == "cog_sink")
        S = c["ctx"] + c["F"] * c["P"]
    run_band(cuda, *args, mod, 2, S, 128)


@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("case", [
    ("hy", 6, 200, 48, 20, 1.4), ("hy", 5, 333, 64, 64, 0.9), ("wan", 7, 180, 0, 0, 1.2), ("cog", 4, 260, 40, 40, 1.1),
    ("generic_wan", 50, 0, 77, 1100), ("generic_hy", 900, 1000, 1, 1093), ("generic_cog", 3, 130, 129, 1031),
    ("generic_wan", 50, 0, 254, 1100), ("generic_hy", 900, 1000, 255, 1093), ("generic_cog", 3, 130, 255, 1031),
    ("none", 0, 0, 0, 1000)])
def test_census_band_small(cuda, case, D):
    """Small band plans, S not a multiple of 128, incl. the engine's generic parameters (include/svgb200.h
    SVGB_MASK_*) with widths that are not multiples of 128 and the dense plan (mode NONE).  The widths 254 (|d| <= W)
    and 255 (|d| < W) leave one chunk per 256-row item that every row but the first sees in full: they pin the
    plan's all-rows vote, which decides whether a chunk skips the element mask."""
    from oracle import attention as oa

    kind = case[0]
    if kind.startswith("generic") or kind == "none":
        mode = {"generic_hy": 1, "generic_wan": 2, "generic_cog": 3, "none": 0}[kind]
        _, m0, m1, m2, S = case
        run_band(cuda, mode, m0, m1, m2, oa.generic_mask_fn(mode, m0, m1, m2), 2, S, D)
    else:
        _, F, P, ctx, plen, mul = case
        args, mod = _band_args(kind, F, P, ctx, plen, mul)
        run_band(cuda, *args, mod, 2, ctx + F * P, D)


# --------------------------------------------------------------------------------------------
# variable-block plans
# --------------------------------------------------------------------------------------------
def run_varblock(cuda, bms, rows, cols, S, D, o_rows=None, key_ids=None, q_rows=None, gather=False, what="",
                 plan=None):
    """bms [H, QC, KC], rows [H, QC], cols [H, KC]; o_rows / key_ids / q_rows [H, S] or None.  `plan`: a prebuilt
    plan of the same maps (default: plan_varblock of them)."""
    from oracle import census as oc
    from svgb200 import core

    H = bms.shape[0]
    if plan is None:
        plan = core.plan_varblock(bms.to(cuda), rows.to(cuda), cols.to(cuda), S, gather=gather)
    cnt, n = [], []
    for h in range(H):
        c, nn = oc.blockmap_census(bms[h], rows[h], cols[h], D, None if key_ids is None else key_ids[h])
        c, nn = oc.scatter_rows(c, nn, None if o_rows is None else o_rows[h])
        cnt.append(c)
        n.append(nn)
    bound_ok(cnt, torch.float16)
    q = torch.zeros(1, H, S, D, dtype=torch.float16, device=cuda)
    k = torch.randn(1, H, S, D, device=cuda).half()
    kw = {}
    if o_rows is not None:
        kw["o_rows"] = o_rows.to(cuda)
    if gather:
        kw["q_rows"] = None if q_rows is None else q_rows.to(cuda)
        kw["kv_rows"] = None if key_ids is None else key_ids.to(cuda)
    for enc in oc.ENCODINGS:
        v = oc.identity_values(S, D, enc, H, torch.float16, cuda)
        if key_ids is not None and not gather:
            # TMA path: the plan reads V in cluster order -- V is the gather of the identity-coded tensor
            v = core.permute_gather(v, key_ids.to(cuda))
        o, lse = core.attn_fwd(q, k, v, plan, return_lse=True, **kw)
        check_census(o[0], lse, cnt, n, enc, what)


@pytest.mark.parametrize("shape", ["hunyuan", "wan"])
def test_census_varblock_fullsize_o_rows(cuda, shape):
    """The production SVG2 path (models/common.py SAPCore.sparse_core): variable-block TMA plan, output through the
    fused inverse permutation.  HunyuanVideo: QC = 400 + 2, KC = 1000 + 2 with the prompt / padding blocks of
    dynamic_map_post_processing; Wan: QC = 300, KC = 1000.  Heads carry maps built for the builder's edges:
    alternating blocks (most runs, 1-column chunks), runs joined across empty key blocks with all-selected and
    all-empty rows, and a random map with empty key clusters; every head has empty q-blocks, q-blocks of every
    r % 256 class and an odd number of tails."""
    g = torch.Generator().manual_seed(17 if shape == "hunyuan" else 18)
    if shape == "hunyuan":
        ctx, plen, V, QC, KC = HY["ctx"], HY["plen"], HY["F"] * HY["P"], 400, 1000
        kinds = ["alternating", "joined", "random"]
    else:
        ctx, plen, V, QC, KC = 0, 0, WAN["F"] * WAN["P"], 300, 1000
        kinds = ["alternating", "joined"]
    S, D, H = V + ctx, 128, len(kinds)
    bms, rows, cols = [], [], []
    for kind in kinds:
        bm, col = _varblock_head(kind, QC, KC, V, g)
        extra = (plen, ctx - plen) if ctx else ()
        row = _q_sizes(V, QC, g, extra)
        if ctx:
            bm = torch.nn.functional.pad(bm, (0, 2, 0, 2), value=False)
            bm[-2, :-1] = True
            bm[:-1, -2] = True
            bm[-1, -1] = True
            if kind == "joined":
                bm[4, :] = False  # the all-empty row stays empty
            col = torch.cat([col, torch.tensor(extra)])
        bms.append(bm)
        rows.append(row)
        cols.append(col)
    bms, rows, cols = torch.stack(bms), torch.stack(rows).int(), torch.stack(cols).int()
    o_rows = torch.stack([torch.randperm(S, generator=g) for _ in range(H)]).int()
    run_varblock(cuda, bms, rows, cols, S, D, o_rows=o_rows, what=f"varblock {shape}")


def test_census_wan_sap_last(cuda):
    """The map, cluster sizes and permutations WanSAPCore produces at Wan 720p (QC = 300, KC = 1000, 2 heads), run
    as sparse_core runs them: V gathered into cluster order, output scattered back through q_sorted_indices."""
    from svgb200.models import wan

    H, F, P, D = 2, WAN["F"], WAN["P"], 128
    S = F * P
    g = torch.Generator(device=cuda).manual_seed(5)
    q, k, v = (torch.randn(1, H, S, D, device=cuda, generator=g).to(torch.bfloat16) for _ in range(3))
    base = torch.randn(1, H, 64, D, device=cuda, generator=g) * 1.5
    which = torch.randint(0, 64, (S,), device=cuda, generator=g)
    q = (q.float() * 0.7 + base[:, :, which]).to(torch.bfloat16)
    k = (k.float() * 0.7 + base[:, :, which]).to(torch.bfloat16)
    sap = wan.WanSAPCore(F, P, num_q_centroids=300, num_k_centroids=1000, top_p_kmeans=0.9, min_kc_ratio=0.1,
                         kmeans_iter_init=4, kmeans_iter_step=2)
    sap.sparse_core(q, k, v)
    last = sap.last
    run_varblock(cuda, last["dynamic_map"].cpu(), last["q_sizes"].cpu(), last["k_sizes"].cpu(), S, D,
                 o_rows=last["q_sorted_indices"].cpu(), key_ids=last["k_sorted_indices"].cpu(), what="WanSAPCore.last")


@pytest.mark.parametrize("D,KC", [(64, 101), (128, 101), (64, 4096), (128, 4096)],
                         ids=["64", "128", "64-kc4096", "128-kc4096"])
def test_census_gather_plan(cuda, D, KC):
    """Row-gather plan with q_rows / kv_rows / o_rows (cluster argsorts).  KC = 101: empty clusters and a query
    cluster that selects nothing.  KC = 4096 (the k-means limit): two keys per key cluster and every other cluster
    selected, so every q-block reads 2048 runs."""
    from svgb200 import core

    g = torch.Generator().manual_seed(23)
    if KC == 4096:
        H, S, QC = 2, 8192, 23
        ql = torch.randint(0, QC, (H, S), generator=g)
        kl = torch.stack([torch.randperm(S, generator=g) // 2 for _ in range(H)])
        bm = torch.zeros(H, QC, KC, dtype=torch.bool)
        bm[:, :, 0::2] = True
    else:
        H, S, QC = 3, 6000, 37
        ql = torch.randint(0, QC, (H, S), generator=g)
        kl = torch.randint(0, KC, (H, S), generator=g)
        ql[0][ql[0] == 5] = 6   # an empty query cluster
        kl[1][kl[1] == 3] = 4   # an empty key cluster
        bm = torch.rand(H, QC, KC, generator=g) < 0.4
        bm[2, 7, :] = False     # a query cluster that sees nothing
        bm[2, 8, :] = True      # and one that sees everything
    qperm, qcnt = core.argsort_labels(ql.to(cuda), QC)
    kperm, kcnt = core.argsort_labels(kl.to(cuda), KC)
    run_varblock(cuda, bm, qcnt.cpu(), kcnt.cpu(), S, D, o_rows=qperm.cpu(), key_ids=kperm.cpu(), q_rows=qperm.cpu(),
                 gather=True, what=f"gather plan D={D} KC={KC}")


def test_census_bsr_shared_plan(cuda):
    """One BSR plan serving every head (items_stride = 0, svgb200.ops.attention_ops.bsr_to_plan):
    the reference's temporal BSR blocks over the video plus an all-to-all text prefix."""
    from oracle import attention as oa
    from svgb200.ops import attention_ops

    H, F, P, text, D = 3, 8, 300, 40, 128
    blocks, (R, Cb) = oa.ref_gen_temporal_mask(F, P, 1.5)
    keep = torch.from_numpy(blocks >= 0)
    MB = keep.shape[0]
    indptr = torch.cat([torch.zeros(1, dtype=torch.long), keep.sum(1).cumsum(0)])
    indices = keep.nonzero()[:, 1]
    plan = attention_ops.bsr_to_plan(indptr, indices, (R, Cb), F * P, text, cuda)
    assert plan.desc.items_stride == 0 and plan.desc.BH == 1
    bm = torch.ones(MB + 1, MB + 1, dtype=torch.bool)  # text rows / columns see everything
    bm[1:, 1:] = keep
    sz = torch.tensor([text] + [R] * MB, dtype=torch.int32)
    S = text + F * P
    run_varblock(cuda, bm.expand(H, -1, -1).contiguous(), sz.expand(H, -1).contiguous(), sz.expand(H, -1).contiguous(),
                 S, D, what="shared BSR plan", plan=plan)


# --------------------------------------------------------------------------------------------
# FP8: q8 = 0, v8 = one-hot (e4m3 1.0), v_scale = 1; the output is bf16, so counts stay <= 128
# --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("plan_kind", ["band", "varblock"])
def test_census_fp8(cuda, plan_kind):
    from oracle import attention as oa
    from oracle import census as oc
    from svgb200 import core

    g = torch.Generator().manual_seed(29)
    H, D = 2, 128
    if plan_kind == "band":
        args, mod = _band_args("hy", 6, 200, 48, 20, 1.4)
        S = 48 + 6 * 200
        plan = core.plan_band(*args, H, S, cuda)
        c, nn = oc.band_census(mod, S, D, cuda)
        cnt, n = [c.cpu()] * H, [nn.cpu()] * H
        o_rows = None
    else:
        S, QC, KC = 8000, 24, 60
        rows = torch.stack([_q_sizes(S, QC, g) for _ in range(H)]).int()
        cols = torch.stack([_partition(S, KC, g) for _ in range(H)]).int()
        bm = torch.rand(H, QC, KC, generator=g) < 0.4
        plan = core.plan_varblock(bm.to(cuda), rows.to(cuda), cols.to(cuda), S)
        o_rows = torch.stack([torch.randperm(S, generator=g) for _ in range(H)]).int()
        cnt, n = [], []
        for h in range(H):
            c, nn = oc.scatter_rows(*oc.blockmap_census(bm[h], rows[h], cols[h], D), o_rows[h])
            cnt.append(c)
            n.append(nn)
        o_rows = o_rows.to(cuda)
    bound_ok(cnt, torch.bfloat16)
    q8 = torch.zeros(1, H, S, D, dtype=torch.uint8, device=cuda)
    k8, sk = core.quantize_e4m3(torch.randn(1, H, S, D, device=cuda).bfloat16())
    sq = torch.tensor([0.5, 3.0], device=cuda)
    sv = torch.ones(H, device=cuda)
    for enc in oc.ENCODINGS:
        v8 = oc.identity_values(S, D, enc, H, torch.float8_e4m3fn, cuda).view(torch.uint8)
        o, lse = core.attn_fwd_fp8(q8, k8, v8, sq, sk, sv, plan, o_rows=o_rows, return_lse=True)
        check_census(o[0], lse, cnt, n, enc, f"fp8 {plan_kind}")
