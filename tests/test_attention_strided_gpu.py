"""Attention on strided views on the GPU (svgb_attn_fwd_strided / svgb_attn_bwd_strided through core).

Exact checks.  A strided call runs every row through the same operations in the same order as the call on contiguous
copies (only the addresses of the loads and stores change), so o, lse, dq, dk and dv are compared bit for bit
(torch.equal) with core.attn_fwd / attn_bwd on .contiguous() copies, which take the flat entry points.  Outputs written
into views of NaN-filled buffers must leave every element outside the view NaN.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

MASK_NONE, MASK_HY, MASK_WAN, MASK_COG = 0, 1, 2, 3
BANDS = {  # (mode, m0, m1, m2), at S = 344 (the band shapes of test_attention_bwd_gpu.py)
    "none": (MASK_NONE, 0, 0, 0),
    "hy": (MASK_HY, 300, 320, 150),
    "wan": (MASK_WAN, 100, 0, 130),
    "cog": (MASK_COG, 20, 20, 140),
}
VIEWS = ("transposed", "packed", "heads", "batch", "padded")


def partition(n, blocks, gen):
    cuts, _ = torch.sort(torch.randperm(n - 1, generator=gen)[: blocks - 1] + 1)
    return torch.diff(torch.cat([torch.tensor([0]), cuts, torch.tensor([n])])).to(torch.int32)


def varblock_plan(cuda, BHkv, Sq, Skv, gen, MB=7, NB=9, density=0.5):
    from svgb200 import core

    rows = torch.stack([partition(Sq, MB, gen) for _ in range(BHkv)])
    cols = torch.stack([partition(Skv, NB, gen) for _ in range(BHkv)])
    bm = torch.rand(BHkv, MB, NB, generator=gen) < density
    return core.plan_varblock(bm.to(cuda), rows.to(cuda), cols.to(cuda), Sq, S_kv=Skv)


def view(kind, B, H, S, D, dtype, cuda, gen, fill=None):
    """A [B, H, S, D] view of kind `kind` over a larger buffer (random, or `fill`): the buffer is returned too"""
    shape = {"transposed": (B, S, H, D), "packed": (B, S, 3, H, D), "heads": (B, 2 * H, S, D),
             "batch": (2 * B, H, S, D), "padded": (B, H, S, D + 64)}[kind]
    buf = (torch.randn(shape, generator=gen) if fill is None else torch.full(shape, fill)).to(dtype).to(cuda)
    x = {"transposed": lambda: buf.transpose(1, 2), "packed": lambda: buf.unbind(2)[1].transpose(1, 2),
         "heads": lambda: buf[:, ::2], "batch": lambda: buf[::2], "padded": lambda: buf[..., :D]}[kind]()
    assert x.shape == (B, H, S, D)  # contiguous only where a dimension of extent 1 hides the stride (B = 1, H = 1)
    return x, buf


def run(q, k, v, do, plan, layout="bhsd", out=None, gout=None):
    from svgb200 import core

    o, lse = core.attn_fwd(q, k, v, plan, layout=layout, return_lse=True, out=out)
    return (o, lse) + tuple(core.attn_bwd(q, k, v, o, do, lse, plan, layout=layout, out=gout))


def check_equal(got, ref, what):
    for name, a, b in zip(("o", "lse", "dq", "dk", "dv"), got, ref):
        assert a.shape == b.shape, f"{what}: {name} shape"
        assert torch.equal(a, b), f"{what}: {name} differs from the contiguous call in {int((a != b).sum())} elements"


def check_views(cuda, kind, B, Hq, Hkv, Sq, Skv, D, dtype, plan, seed=0):
    """The views' call against the contiguous copies' call, and a second strided call writing o and the gradients
    into views of NaN-filled buffers, whose gaps must stay NaN."""
    gen = torch.Generator().manual_seed(seed)
    q, do = (view(kind, B, Hq, Sq, D, dtype, cuda, gen)[0] for _ in range(2))
    k, v = (view(kind, B, Hkv, Skv, D, dtype, cuda, gen)[0] for _ in range(2))
    ref = run(*(t.contiguous() for t in (q, k, v, do)), plan)
    what = f"{kind} B={B} Hq={Hq} Hkv={Hkv} Sq={Sq} Skv={Skv} D={D} {dtype}"
    got = run(q, k, v, do, plan)
    check_equal(got, ref, what)
    outs = [view(kind, B, h, s, D, dtype, cuda, gen, fill=float("nan")) for h, s in
            ((Hq, Sq), (Hq, Sq), (Hkv, Skv), (Hkv, Skv))]
    got = run(q, k, v, do, plan, out=outs[0][0], gout=tuple(x for x, _ in outs[1:]))
    check_equal(got, ref, what + " into NaN views")
    for name, (x, buf) in zip(("o", "dq", "dk", "dv"), outs):
        assert got[("o", "lse", "dq", "dk", "dv").index(name)] is x
        inside = torch.zeros(buf.shape, dtype=torch.bool, device=cuda)
        inside.as_strided(x.shape, x.stride(), x.storage_offset() - buf.storage_offset()).fill_(True)
        assert torch.isnan(buf[~inside]).all(), f"{what}: {name} was written outside its view"
        assert not torch.isnan(x).any(), f"{what}: {name} has unwritten elements"


@pytest.mark.parametrize("kind", VIEWS)
@pytest.mark.parametrize("B", [1, 2, 3])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_views_match_contiguous(cuda, kind, B, D, dtype):
    """Every view kind, batch size, dtype and head dim on a square variable-block plan (a map per head)"""
    gen = torch.Generator().manual_seed(B * 10 + D)
    H, S = 4, 333
    check_views(cuda, kind, B, H, H, S, S, D, dtype, varblock_plan(cuda, B * H, S, S, gen))


PLANS = ["square", "rect_long_kv", "rect_short_kv", "gqa4", "mqa"] + [f"band_{m}" for m in BANDS]


@pytest.mark.parametrize("kind", VIEWS)
@pytest.mark.parametrize("plan_kind", PLANS)
def test_plans_match_contiguous(cuda, plan_kind, kind):
    """Rectangular plans, grouped-query heads (Hkv = Hq / 4 and 1) and the band masks, B = 2, bf16, D = 128"""
    from svgb200 import core

    gen = torch.Generator().manual_seed(PLANS.index(plan_kind))
    B, Hq, Sq, Skv = 2, 8, 344, 344
    Hkv = {"gqa4": 2, "mqa": 1}.get(plan_kind, Hq)
    Skv = {"rect_long_kv": 900, "rect_short_kv": 150}.get(plan_kind, Skv)
    if plan_kind.startswith("band_"):
        plan = core.plan_band(*BANDS[plan_kind[5:]], B * Hkv, Sq, cuda)
    else:
        plan = varblock_plan(cuda, B * Hkv, Sq, Skv, gen)
    check_views(cuda, kind, B, Hq, Hkv, Sq, Skv, 128, torch.bfloat16, plan)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_shd_padded_rows(cuda, dtype):
    """[S, H, D] with a padded row stride (a column slice of a wider projection) in the 'shd' layout"""
    gen = torch.Generator().manual_seed(1)
    S, H, D = 500, 6, 64
    plan = varblock_plan(cuda, H, S, S, gen)
    q, k, v, do = (torch.randn(S, H * D + 128, generator=gen).to(dtype).to(cuda)[:, 64:64 + H * D].view(S, H, D)
                   for _ in range(4))
    assert not q.is_contiguous()
    check_equal(run(q, k, v, do, plan, layout="shd"), run(*(t.contiguous() for t in (q, k, v, do)), plan, layout="shd"),
                "shd padded")


def test_zero_stride_do_and_copies(cuda):
    """A zero-stride dO (the expanded gradient of o.sum()) and a last stride other than 1 go through .contiguous()
    and still give the contiguous call's bits"""
    gen = torch.Generator().manual_seed(2)
    B, H, S, D = 2, 4, 300, 128
    plan = varblock_plan(cuda, B * H, S, S, gen)
    q, k, v = (view("transposed", B, H, S, D, torch.bfloat16, cuda, gen)[0] for _ in range(3))
    do = torch.ones((), dtype=torch.bfloat16, device=cuda).expand(B, H, S, D)
    check_equal(run(q, k, v, do, plan), run(*(t.contiguous() for t in (q, k, v, do)), plan), "zero-stride dO")
    kt = k.contiguous().transpose(2, 3).contiguous().transpose(2, 3)  # last stride S
    assert kt.stride(-1) != 1
    check_equal(run(q, kt, v, do, plan), run(*(t.contiguous() for t in (q, k, v, do)), plan), "last stride S")


def _autograd(q_in, k_in, v_in, plan, do_fn):
    """core.attention under autograd from [B, S, H, D] leaves, with the output gradient do_fn(o)"""
    from svgb200 import core

    leaves = [t.detach().clone().requires_grad_() for t in (q_in, k_in, v_in)]
    o = core.attention(*(t.transpose(1, 2) for t in leaves), plan)
    torch.autograd.backward(o, do_fn(o))
    return [o.detach()] + [t.grad for t in leaves]


def test_autograd_transposed_views(cuda):
    """core.attention on transposed projections: o keeps [B, S, H, D] memory, the gradient of
    o.transpose(1, 2).reshape(B, S, H * D) arrives as a transposed view and is used in place; the results equal the
    contiguous inputs' bit for bit, and two runs give the same bits"""
    from svgb200 import core

    gen = torch.Generator().manual_seed(3)
    B, H, S, D = 2, 8, 700, 128
    plan = varblock_plan(cuda, B * H, S, S, gen)
    q, k, v, g = (torch.randn(B, S, H, D, generator=gen).to(torch.bfloat16).to(cuda) for _ in range(4))
    seen = []

    def do_fn(o):
        assert o.transpose(1, 2).is_contiguous(), "o does not keep the [B, S, H, D] memory of a transposed q"
        d = g.transpose(1, 2)
        seen.append(d)
        return d

    a = _autograd(q, k, v, plan, do_fn)
    b = _autograd(q, k, v, plan, do_fn)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    leaves = [t.transpose(1, 2).contiguous().requires_grad_() for t in (q, k, v)]
    o = core.attention(*leaves, plan)
    torch.autograd.backward(o, g.transpose(1, 2).contiguous())
    assert torch.equal(a[0], o.detach())
    for x, y in zip(a[1:], leaves):
        assert torch.equal(x.transpose(1, 2), y.grad)
    assert a[1].is_contiguous()  # dq reached the [B, S, H, D] leaf without a layout change


def test_launch_count_and_no_copy_kernels(cuda):
    """A strided forward + backward makes the contiguous call's launches and, in a torch.profiler trace, no copy"""
    from svgb200 import core

    gen = torch.Generator().manual_seed(4)
    B, H, S, D = 2, 4, 600, 128
    plan = varblock_plan(cuda, B * H, S, S, gen)
    plan.key_major()  # built before the trace: the key-major planner transposes the map
    q, k, v, g = (torch.randn(B, S, H, D, generator=gen).to(torch.bfloat16).to(cuda) for _ in range(4))
    counts = []
    for inputs, do in (((q, k, v), g), ((t.transpose(1, 2).contiguous().transpose(1, 2) for t in (q, k, v)), g)):
        n0 = core.launch_count
        _autograd(*inputs, plan, lambda o: do.transpose(1, 2) if not o.is_contiguous() else do.transpose(1, 2).contiguous())
        counts.append(core.launch_count - n0)
    assert counts[0] == counts[1] == 4
    leaves = [t.detach().clone().requires_grad_() for t in (q, k, v)]
    d = g.transpose(1, 2)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        o = core.attention(*(t.transpose(1, 2) for t in leaves), plan)
        torch.autograd.backward(o, d)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    assert any("attn_fwd_kernel" in n for n in names) and any("attn_bwd_kernel" in n for n in names), names
    copies = [n for n in names if "copy" in n.lower() or "memcpy" in n.lower() or "elementwise" in n.lower()]
    assert not copies, copies


def test_wan_720p_transposed_projection(cuda):
    """Wan 2.1 720p (40 heads, S = 75 600, D = 128) from transposed [1, S, H, D] projections under a 300 x 1000 map at
    density 0.3: forward and backward bit for bit against the contiguous copies"""
    gen = torch.Generator().manual_seed(5)
    H, S, D = 40, 75600, 128
    plan = varblock_plan(cuda, H, S, S, gen, MB=300, NB=1000, density=0.3)
    g = torch.Generator(device=cuda).manual_seed(5)
    q, k, v, do = (torch.randn(1, S, H, D, device=cuda, generator=g).to(torch.bfloat16).transpose(1, 2)
                   for _ in range(4))
    check_equal(run(q, k, v, do, plan), run(*(t.contiguous() for t in (q, k, v, do)), plan), "Wan 720p")


def test_hunyuan_720p_band_batch2(cuda):
    """HunyuanVideo 720p band (24 heads, S = 119 056, W = 19 072) at B = 2 on transposed projections: forward and
    backward bit for bit against the contiguous copies"""
    from svgb200 import core

    ctx, F, P, plen, W = 256, 33, 3600, 71, 19072
    V = F * P
    B, H, S, D = 2, 24, ctx + V, 128
    plan = core.plan_band(MASK_HY, V, V + plen, W, B * H, S, cuda)
    g = torch.Generator(device=cuda).manual_seed(6)
    q, k, v, do = (torch.randn(B, S, H, D, device=cuda, generator=g).to(torch.bfloat16).transpose(1, 2)
                   for _ in range(4))
    check_equal(run(q, k, v, do, plan), run(*(t.contiguous() for t in (q, k, v, do)), plan), "HunyuanVideo 720p B=2")
