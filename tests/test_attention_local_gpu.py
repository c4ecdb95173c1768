"""The local band mask (SVGB_MASK_LOCAL: causal, sliding-window and sink-plus-window attention) on the GPU: the exact
key census of the forward on every row, the online-softmax census, the backward's key and gradient censuses and its
key-major plan structure, bit-for-bit equality with MASK_WAN where the two coincide, the references (SDPA causal, fp64
autograd), every layout band plans take, and the launch counts."""
import pytest
import torch

import local_mask as lm
from oracle import bwd_census as bc
from oracle import census as oc
from test_attention_bwd_census_gpu import run_grad as _run_grad
from test_attention_bwd_census_gpu import run_key
from test_attention_census_gpu import bound_ok, check_census
from test_attention_gqa_gpu import check_exact, run_both

pytestmark = pytest.mark.gpu

DT = {"bf16": torch.bfloat16, "fp16": torch.float16}
S_SMALL = 1100  # = 8 * 128 + 76
# (sink, left, right): causal, left-only and right-only windows, widths 254 / 255 / 256 on either side (one chunk per
# 256-row item that every row but the first or last sees in full: the plan's all-rows vote), sinks that are not
# multiples of 128, a two-sided window with a sink, the diagonal alone
SMALL = [(0, S_SMALL, 0), (0, 300, 0), (0, 0, 300), (0, 254, 0), (0, 255, 0), (0, 256, 0), (0, 0, 254), (0, 0, 255),
         (0, 0, 256), (37, 200, 0), (130, 77, 5), (3, 40, 129), (0, 0, 0)]
WAN720 = dict(F=21, P=3600)
HY720_S = 256 + 33 * 3600  # 119 056


def _ids(c):
    return "-".join(map(str, c))


def _plan(cuda, args, H, S):
    from svgb200 import core

    return core.plan_band(lm.MASK_LOCAL, *args, H, S, cuda)


# --------------------------------------------------------------------------------------------
# forward key census
# --------------------------------------------------------------------------------------------
def run_census(cuda, args, H, S, D, dtype, plan=None):
    from svgb200 import core

    plan = plan or _plan(cuda, args, H, S)
    cnt, n = oc.band_census(lm.local_mask_fn(*args), S, D, cuda)
    cnt, n = cnt.cpu(), n.cpu()
    bound_ok([cnt], dtype)
    q = torch.zeros(1, H, S, D, dtype=dtype, device=cuda)
    k = torch.randn(1, H, S, D, device=cuda).to(dtype)
    for enc in oc.ENCODINGS:
        v = oc.identity_values(S, D, enc, H, dtype, cuda)
        o, lse = core.attn_fwd(q, k, v, plan, return_lse=True)
        check_census(o[0], lse, [cnt] * H, [n] * H, enc, f"LOCAL{args} S={S} D={D} {dtype}")


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("args", SMALL, ids=_ids)
def test_census_local_small(cuda, args, D, dtype):
    run_census(cuda, args, 2, S_SMALL, D, DT[dtype])


@pytest.mark.parametrize("args", [(0, HY720_S, 0), (1000, HY720_S, 3)], ids=["causal", "sink-causal"])
def test_census_local_fullsize(cuda, args):
    """S = 119 056 (HunyuanVideo 720p): causal, the largest window the census allows (every count below the fp16
    limit at this S), with and without a 1000-key sink; plan_local builds the first."""
    from svgb200 import core

    plan = core.plan_local(2, HY720_S, cuda, causal=True) if args[0] == 0 else None
    run_census(cuda, args, 2, HY720_S, 128, torch.float16, plan)


# --------------------------------------------------------------------------------------------
# online-softmax census
# --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("args", [(0, 1260, 0), (37, 300, 0), (0, 0, 255)], ids=_ids)
def test_softmax_local(cuda, args, D, dtype):
    """The softmax census's Wan case (S = 1260) under LOCAL masks: integer log2 scores that move the running max,
    every row bit for bit."""
    from oracle import softmax as sm
    from test_softmax_census_gpu import run

    case = sm.band_case("wan", D=D)
    case.band, case.mod = (lm.MASK_LOCAL, *args), lm.local_mask_fn(*args)
    run(cuda, case, DT[dtype], f"LOCAL{args} D={D} {dtype}")


# --------------------------------------------------------------------------------------------
# backward: key census, key-major structure, gradient census
# --------------------------------------------------------------------------------------------
def check_plans(cuda, plan, args, S):
    """Both plans' items against the host mirror's segments and launch order; the key-major lists against the mask."""
    mod = lm.local_mask_fn(*args)
    for p, transposed in ((plan, False), (plan.key_major(), True)):
        (items,), chunks = bc.read_plan(p, 1)
        got = [(int(it[0, 0]), int(it[0, 1]) + int(it[1, 1])) for it in items]
        assert got == lm.band_items(lm.MASK_LOCAL, *args, S, transposed), f"transposed={transposed}: items"
        if transposed:
            msg = bc.check_band_t_structure(items, chunks, mod, S, cuda)
            assert msg is None, f"key-major band plan: {msg}"


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("args", SMALL, ids=_ids)
def test_key_census_local_small(cuda, args, D, dtype):
    plan = _plan(cuda, args, 2, S_SMALL)
    check_plans(cuda, plan, args, S_SMALL)
    tab = bc.band_tables(lm.local_mask_fn(*args), S_SMALL, D, cuda)
    run_key(cuda, plan, [tab] * 2, S_SMALL, D, DT[dtype], f"LOCAL{args} D={D} {dtype}")


@pytest.mark.parametrize("args", [(0, HY720_S, 0), (1000, 4990, 0)], ids=["causal", "sink-window"])
def test_key_census_local_fullsize(cuda, args):
    S = HY720_S
    plan = _plan(cuda, args, 2, S)
    check_plans(cuda, plan, args, S)
    tab = bc.band_tables(lm.local_mask_fn(*args), S, 128, cuda)
    assert int(tab[0].max()) <= bc.MAX_COUNT[torch.float16] and int(tab[2].max()) <= bc.MAX_COUNT[torch.float16]
    run_key(cuda, plan, [tab] * 2, S, 128, torch.float16, f"LOCAL{args} S={S}")


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("args,S", [((0, 1025, 0), 1025), ((37, 300, 0), 960), ((0, 0, 255), 1089),
                                    ((5, 129, 77), 1151)], ids=["causal", "sink-left", "right", "two-sided"])
def test_grad_census_local(cuda, args, S, D, dtype):
    """Real scores and values with every intermediate exact, all eight backward instantiations, at S = 1, 64, 65 and
    127 mod 128."""
    g = torch.Generator().manual_seed(S)
    case = bc.GradCase(f"LOCAL{args}", S, D, 2, 1.0, *bc._grad_inputs(2, S, D, 1.0, g), band=(lm.MASK_LOCAL, *args),
                       mod=lm.local_mask_fn(*args))
    _run_grad(cuda, case, DT[dtype], f"LOCAL{args} D={D} {dtype}")


# --------------------------------------------------------------------------------------------
# LOCAL(P, W, W) == WAN(P, W), bit for bit
# --------------------------------------------------------------------------------------------
def _fwd_bwd(cuda, plan, q, k, v, do):
    from svgb200 import core

    o, lse = core.attn_fwd(q, k, v, plan, return_lse=True)
    grads = tuple(torch.full_like(t, float("nan")) for t in (q, k, v))
    core.attn_bwd(q, k, v, o, do, lse, plan, out=grads)
    return (o, lse) + grads


@pytest.mark.parametrize("shape", ["wan720", "hy720"])
def test_local_equals_wan(cuda, shape):
    """The Wan 720p band (P = 3600, width of sparsity 0.2) at the Wan 720p and HunyuanVideo 720p lengths: o, lse, dq,
    dk and dv of a LOCAL(P, W, W) plan are those of the MASK_WAN(P, W) plan, bit for bit."""
    from oracle import attention as oa
    from svgb200 import core

    P = WAN720["P"]
    W = oa.wan_band_width(oa.sparsity_to_width(0.2, 0, WAN720["F"], P), P)
    S = WAN720["F"] * P if shape == "wan720" else HY720_S
    g = torch.Generator().manual_seed(7)
    q, k, v, do = (torch.randn(1, 2, S, 128, generator=g).to(torch.bfloat16).to(cuda) for _ in range(4))
    a = _fwd_bwd(cuda, core.plan_band(lm.MASK_LOCAL, P, W, W, 2, S, cuda), q, k, v, do)
    b = _fwd_bwd(cuda, core.plan_band(core.MASK_WAN, P, 0, W, 2, S, cuda), q, k, v, do)
    for name, x, y in zip(("o", "lse", "dq", "dk", "dv"), a, b):
        assert torch.equal(x, y), f"{name}: {int((x != y).sum())} elements differ"


# --------------------------------------------------------------------------------------------
# references
# --------------------------------------------------------------------------------------------
def _rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm())


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("S", [4096, 32768])
def test_causal_matches_sdpa(cuda, S, dtype):
    """plan_local(causal=True) against scaled_dot_product_attention(is_causal=True), forward and gradients, both in
    16 bits: norm-wise relative differences within the two kernels' rounding."""
    from svgb200 import core

    dt = DT[dtype]
    g = torch.Generator().manual_seed(S)
    q, k, v, do = (torch.randn(1, 4, S, 128, generator=g).to(dt).to(cuda) for _ in range(4))
    plan = core.plan_local(4, S, cuda, causal=True)
    outs = []
    for f in (lambda a, b, c: core.attention(a, b, c, plan),
              lambda a, b, c: torch.nn.functional.scaled_dot_product_attention(a, b, c, is_causal=True)):
        x = [t.clone().requires_grad_() for t in (q, k, v)]
        o = f(*x)
        o.backward(do)
        outs.append([o.detach()] + [t.grad for t in x])
    tol = 1e-2 if dt == torch.bfloat16 else 2e-3
    for name, a, b in zip(("o", "dq", "dk", "dv"), *outs):
        assert _rel(a, b) < tol, f"{name}: relative difference {_rel(a, b):.2e}"


def test_sink_window_matches_fp64_autograd(cuda):
    """A sink-plus-window mask (sink 37, 300 keys back, none ahead) against fp64 autograd through the oracle's masked
    attention: o, dq, dk, dv norm-wise."""
    from oracle import attention as oa
    from svgb200 import core

    S, H, D, args = 1500, 2, 64, (37, 300, 0)
    g = torch.Generator().manual_seed(11)
    q, k, v, do = (torch.randn(1, H, S, D, generator=g).to(torch.bfloat16) for _ in range(4))
    ref = [t[0].double().requires_grad_() for t in (q, k, v)]
    o_ref = oa.masked_attention_bhsd(*ref, lm.local_mask_fn(*args), dtype=torch.float64)
    o_ref.backward(do[0].double())
    x = [t.to(cuda).requires_grad_() for t in (q, k, v)]
    o = core.attention(*x, core.plan_local(H, S, cuda, window_size=(300, 0), sink=37))
    o.backward(do.to(cuda))
    for name, a, b in zip(("o", "dq", "dk", "dv"), [o.detach()] + [t.grad for t in x], [o_ref.detach()] +
                          [t.grad for t in ref]):
        assert _rel(a[0].cpu(), b) < 1e-2, f"{name}: relative difference {_rel(a[0].cpu(), b):.2e}"


# --------------------------------------------------------------------------------------------
# layouts, determinism, launch counts
# --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("Hkv", [16, 8, 1])
def test_gqa_local(cuda, Hkv):
    """GQA / MQA on a causal-with-sink plan built over the key/value heads: o, lse, dq bit for bit the MHA call on
    repeated K / V, dk / dv its group sums."""
    from svgb200 import core

    Hq, S = 16, 3000
    p = core.plan_local(Hkv, S, cuda, causal=True, sink=37)
    check_exact(*run_both(cuda, p, p, Hq, Hkv, S, S, 128, torch.bfloat16), Hq // Hkv, torch.bfloat16, "bhsd",
                f"Hkv={Hkv}")


@pytest.mark.parametrize("view", ["bshd-B1", "bshd-B2", "shd"])
def test_views_local(cuda, view):
    """Transposed [B, S, H, D] views (B = 1, 2) and the [S, H, D] layout match the contiguous [B, H, S, D] call bit
    for bit, forward and backward, and a second backward gives the same bits."""
    from svgb200 import core

    B = 2 if view == "bshd-B2" else 1
    H, S, D = 4, 2000, 128
    plan = core.plan_local(B * H, S, cuda, window_size=(255, 40), sink=130)
    g = torch.Generator().manual_seed(B)
    base = [torch.randn(B, S, H, D, generator=g).to(torch.bfloat16).to(cuda) for _ in range(4)]
    ref = _fwd_bwd(cuda, plan, *(t.transpose(1, 2).contiguous() for t in base))
    if view == "shd":
        o, lse = core.attn_fwd(*(t[0].contiguous() for t in base[:3]), plan, layout="shd", return_lse=True)
        got = [o[None].transpose(1, 2), lse]
        for _ in range(2):
            dq, dk, dv = core.attn_bwd(*(t[0].contiguous() for t in base[:3]), o, base[3][0].contiguous(), lse, plan,
                                       layout="shd")
            got.append([t[None].transpose(1, 2) for t in (dq, dk, dv)])
    else:
        views = [t.transpose(1, 2) for t in base]
        o, lse = core.attn_fwd(*views[:3], plan, return_lse=True)
        got = [o, lse]
        for _ in range(2):
            got.append(list(core.attn_bwd(*views[:3], o, views[3], lse, plan)))
    for name, a, b in zip(("o", "lse"), got[:2], ref[:2]):
        assert torch.equal(a, b), f"{view}: {name}"
    for name, a, a2, b in zip(("dq", "dk", "dv"), got[2], got[3], ref[2:]):
        assert torch.equal(a, b) and torch.equal(a, a2), f"{view}: {name}"


def test_launch_counts(cuda):
    """One launch to plan, one forward launch, three backward launches (delta, dQ, dK / dV) once the key-major plan
    exists (one more launch the first time)."""
    from svgb200 import core

    S = 3000
    n0 = core.launch_count
    plan = core.plan_local(2, S, cuda, causal=True)
    assert core.launch_count - n0 == 1
    q, k, v, do = (torch.randn(1, 2, S, 128, device=cuda).to(torch.bfloat16) for _ in range(4))
    n0 = core.launch_count
    o, lse = core.attn_fwd(q, k, v, plan, return_lse=True)
    assert core.launch_count - n0 == 1
    n0 = core.launch_count
    core.attn_bwd(q, k, v, o, do, lse, plan)
    assert core.launch_count - n0 == 4
    n0 = core.launch_count
    core.attn_bwd(q, k, v, o, do, lse, plan)
    assert core.launch_count - n0 == 3
