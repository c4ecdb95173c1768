"""The block-causal mask (SVGB_MASK_BLOCK_CAUSAL: chunk-wise causal attention of autoregressive video) on the GPU: the
exact key census of the forward on every row at small and production shapes, the backward's key and gradient censuses
and its key-major plan structure, fp64 autograd with B = 2 and grouped-query heads, block = 1 bit for bit the causal
sliding window, strided views, compiled flex_attention under the same mask, and the KV-cache plans in every cache format,
single and split, against the host mirror, the oracle, the square plan and a renumbered cache."""
import random

import pytest
import torch

import block_causal_mask as bm
from oracle import bwd_census as bc
from oracle import census as oc
from test_attention_bwd_census_gpu import run_grad as _run_grad
from test_attention_bwd_census_gpu import run_key
from test_attention_census_gpu import bound_ok, check_census
from test_attention_gqa_gpu import check_exact, run_both
from test_attention_kvcache_fp8_gpu import FP8_LSE, FP8_TOL, _cache8, _head_scales, _paged8, _q8
from test_attention_kvcache_fp8_rows_gpu import _cache as _cache_rows
from test_attention_kvcache_fp8_rows_gpu import _q8rows
from test_attention_kvcache_gpu import _eq, _paged_from, _rand
from test_attention_kvcache_split_gpu import _lists, _nan_partials

pytestmark = pytest.mark.gpu

DT = {"bf16": torch.bfloat16, "fp16": torch.float16}
S_SMALL = 1100  # = 8 * 128 + 76
# (block C, first_block F, window W (-1: unbounded), sink): C = 1 / 127 / 128 / 129 / 300, a shorter first block, W = C,
# W > C, unbounded, sinks below, across and past a block boundary
SMALL = [(1, 1, -1, 0), (1, 1, 200, 0), (127, 127, -1, 0), (128, 128, -1, 0), (129, 129, -1, 0), (300, 300, -1, 0),
         (300, 300, 300, 0), (300, 300, 450, 0), (129, 40, -1, 0), (129, 1, 129, 0), (300, 77, 600, 37),
         (128, 128, 256, 100), (129, 129, 258, 200), (300, 300, 300, 650), (2000, 2000, -1, 0)]
WAN_S, WAN_C, FRAME = 21 * 1560, 4680, 1560  # Wan: 21 latent frames of 1560 tokens, chunks of 3 frames


def _ids(c):
    return "-".join(map(str, c))


def _plan(cuda, args, H, S):
    from svgb200 import core

    C_, F, W, sink = args
    return core.plan_block_causal(H, S, cuda, block=C_, first_block=F, window=W, sink=sink)


def _mod(args):
    return bm.block_causal_mask_fn(*args)


# --------------------------------------------------------------------------------------------
# forward key census
# --------------------------------------------------------------------------------------------
def run_census(cuda, args, H, S, D, dtype):
    from svgb200 import core

    plan = _plan(cuda, args, H, S)
    cnt, n = oc.band_census(_mod(args), S, D, cuda)
    cnt, n = cnt.cpu(), n.cpu()
    bound_ok([cnt], dtype)
    q = torch.zeros(1, H, S, D, dtype=dtype, device=cuda)
    k = torch.randn(1, H, S, D, device=cuda).to(dtype)
    for enc in oc.ENCODINGS:
        v = oc.identity_values(S, D, enc, H, dtype, cuda)
        o, lse = core.attn_fwd(q, k, v, plan, return_lse=True)
        check_census(o[0], lse, [cnt] * H, [n] * H, enc, f"BLOCK{args} S={S} D={D} {dtype}")


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("args", SMALL, ids=_ids)
def test_census_small(cuda, args, D, dtype):
    run_census(cuda, args, 2, S_SMALL, D, DT[dtype])


FULL = [(WAN_C, WAN_C, -1, 0), (WAN_C, WAN_C, 3 * WAN_C, FRAME), (WAN_C, FRAME, -1, 0)]


@pytest.mark.parametrize("args", FULL, ids=["chunks", "window-sink", "i2v"])
def test_census_wan(cuda, args):
    """S = 21 * 1560 with chunks of three frames: unbounded, a 14 040-key window with a one-frame sink, and the I2V layout
    whose first block is one frame."""
    run_census(cuda, args, 2, WAN_S, 128, torch.float16)


# --------------------------------------------------------------------------------------------
# backward: key census, key-major structure, gradient census
# --------------------------------------------------------------------------------------------
def check_plans(plan, args, S, cuda):
    """Both plans' items against the host mirror's launch order; the key-major lists against the mask."""
    C_, F, W, sink = args
    for p, transposed in ((plan, False), (plan.key_major(), True)):
        (items,), chunks = bc.read_plan(p, 1)
        got = [(int(it[0, 0]), int(it[0, 1]) + int(it[1, 1])) for it in items]
        assert got == bm.band_items(sink, p.desc.m2, S, transposed), f"transposed={transposed}: items"
        if transposed:
            msg = bc.check_band_t_structure(items, chunks, _mod(args), S, cuda)
            assert msg is None, f"key-major band plan: {msg}"


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("args", SMALL, ids=_ids)
def test_key_census_small(cuda, args, D, dtype):
    plan = _plan(cuda, args, 2, S_SMALL)
    check_plans(plan, args, S_SMALL, cuda)
    tab = bc.band_tables(_mod(args), S_SMALL, D, cuda)
    run_key(cuda, plan, [tab] * 2, S_SMALL, D, DT[dtype], f"BLOCK{args} D={D} {dtype}")


@pytest.mark.parametrize("args", FULL[1:], ids=["window-sink", "i2v"])
def test_key_census_wan(cuda, args):
    plan = _plan(cuda, args, 2, WAN_S)
    check_plans(plan, args, WAN_S, cuda)
    tab = bc.band_tables(_mod(args), WAN_S, 128, cuda)
    assert int(tab[0].max()) <= bc.MAX_COUNT[torch.float16] and int(tab[2].max()) <= bc.MAX_COUNT[torch.float16]
    run_key(cuda, plan, [tab] * 2, WAN_S, 128, torch.float16, f"BLOCK{args} S={WAN_S}")


@pytest.mark.parametrize("dtype", ["bf16", "fp16"])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("args,S", [((300, 300, -1, 0), 1025), ((129, 40, 258, 37), 960), ((1, 1, 255, 0), 1089),
                                    ((200, 13, 201, 300), 1151)], ids=["chunks", "first-window", "block1", "sink"])
def test_grad_census(cuda, args, S, D, dtype):
    """Real scores and values with every intermediate exact, all eight backward instantiations."""
    from svgb200 import core

    C_, F, W, sink = args
    W = S + C_ if W == -1 else W
    g = torch.Generator().manual_seed(S)
    case = bc.GradCase(f"BLOCK{args}", S, D, 2, 1.0, *bc._grad_inputs(2, S, D, 1.0, g),
                       band=(core.MASK_BLOCK_CAUSAL, sink, bm.m1_of(C_, F), W), mod=_mod(args))
    _run_grad(cuda, case, DT[dtype], f"BLOCK{args} D={D} {dtype}")


def _rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm())


def test_fp64_autograd_batch_gqa_determinism(cuda):
    """B = 2, Hq = 4 over Hkv = 2, an I2V-like short first block, a window and a sink: o, dq, dk, dv against fp64
    autograd through the oracle's masked attention, and a second backward gives the same bits."""
    from oracle import attention as oa
    from svgb200 import core

    B, Hq, Hkv, S, D, args = 2, 4, 2, 1500, 64, (300, 100, 600, 37)
    g = torch.Generator().manual_seed(11)
    q, do = (torch.randn(B, Hq, S, D, generator=g).to(torch.bfloat16) for _ in range(2))
    k, v = (torch.randn(B, Hkv, S, D, generator=g).to(torch.bfloat16) for _ in range(2))
    ref = [t.reshape(-1, S, D).double().requires_grad_() for t in (q, k, v)]
    rk, rv = (t.view(B, Hkv, S, D).repeat_interleave(Hq // Hkv, 1).reshape(-1, S, D) for t in ref[1:])
    o_ref = oa.masked_attention_bhsd(ref[0], rk, rv, _mod(args), dtype=torch.float64)
    o_ref.backward(do.reshape(-1, S, D).double())
    plan = _plan(cuda, args, B * Hkv, S)
    grads = []
    for _ in range(2):
        x = [t.to(cuda).requires_grad_() for t in (q, k, v)]
        o = core.attention(*x, plan)
        o.backward(do.to(cuda))
        grads.append([o.detach()] + [t.grad for t in x])
    for name, a, a2, b in zip(("o", "dq", "dk", "dv"), grads[0], grads[1], [o_ref.detach()] + [t.grad for t in ref]):
        assert torch.equal(a, a2), f"{name}: not deterministic"
        assert _rel(a.reshape(b.shape).cpu(), b) < 1e-2, f"{name}: relative difference {_rel(a.reshape(b.shape).cpu(), b):.2e}"


# --------------------------------------------------------------------------------------------
# block = 1 is the causal sliding window, bit for bit
# --------------------------------------------------------------------------------------------
def _fwd_bwd(plan, q, k, v, do):
    from svgb200 import core

    o, lse = core.attn_fwd(q, k, v, plan, return_lse=True)
    grads = tuple(torch.full_like(t, float("nan")) for t in (q, k, v))
    core.attn_bwd(q, k, v, o, do, lse, plan, out=grads)
    return (o, lse) + grads


@pytest.mark.parametrize("W,sink", [(-1, 0), (300, 0), (1000, 130)])
def test_block_one_equals_plan_local(cuda, W, sink):
    from svgb200 import core

    S = 4000
    g = torch.Generator().manual_seed(W)
    q, k, v, do = (torch.randn(1, 2, S, 128, generator=g).to(torch.bfloat16).to(cuda) for _ in range(4))
    a = _fwd_bwd(core.plan_block_causal(2, S, cuda, block=1, window=W, sink=sink), q, k, v, do)
    b = _fwd_bwd(core.plan_local(2, S, cuda, causal=True, window_size=(W - 1 if W != -1 else -1, 0), sink=sink),
                 q, k, v, do)
    for name, x, y in zip(("o", "lse", "dq", "dk", "dv"), a, b):
        assert torch.equal(x, y), f"{name}: {int((x != y).sum())} elements differ"


@pytest.mark.parametrize("view", ["bshd-B2", "shd"])
def test_views(cuda, view):
    """Transposed [B, S, H, D] views and the [S, H, D] layout match the contiguous [B, H, S, D] call bit for bit."""
    from svgb200 import core

    B = 2 if view == "bshd-B2" else 1
    H, S, D = 4, 2000, 128
    plan = core.plan_block_causal(B * H, S, cuda, block=300, first_block=100, window=900, sink=130)
    g = torch.Generator().manual_seed(B)
    base = [torch.randn(B, S, H, D, generator=g).to(torch.bfloat16).to(cuda) for _ in range(4)]
    ref = _fwd_bwd(plan, *(t.transpose(1, 2).contiguous() for t in base))
    if view == "shd":
        o, lse = core.attn_fwd(*(t[0].contiguous() for t in base[:3]), plan, layout="shd", return_lse=True)
        dq, dk, dv = core.attn_bwd(*(t[0].contiguous() for t in base[:3]), o, base[3][0].contiguous(), lse, plan,
                                   layout="shd")
        got = [o[None].transpose(1, 2), lse] + [t[None].transpose(1, 2) for t in (dq, dk, dv)]
    else:
        views = [t.transpose(1, 2) for t in base]
        o, lse = core.attn_fwd(*views[:3], plan, return_lse=True)
        got = [o, lse, *core.attn_bwd(*views[:3], o, views[3], lse, plan)]
    for name, a, b in zip(("o", "lse", "dq", "dk", "dv"), got, ref):
        assert torch.equal(a, b), f"{view}: {name}"


def test_gqa_bit_for_bit(cuda):
    """GQA on a block-causal plan: o, lse, dq bit for bit the MHA call on repeated K / V, dk / dv its group sums."""
    from svgb200 import core

    p = core.plan_block_causal(4, 3000, cuda, block=700, window=1400, sink=37)
    check_exact(*run_both(cuda, p, p, 16, 4, 3000, 3000, 128, torch.bfloat16), 4, torch.bfloat16, "bhsd", "block GQA")


def test_e4m3_band_plan(cuda):
    """e4m3 q, k, v through svgb_attn_fwd_strided_e4m3 on a block-causal plan, against the bf16 call."""
    from svgb200 import core

    S, H = 3000, 4
    g = torch.Generator().manual_seed(3)
    q, k, v = (torch.randn(1, H, S, 128, generator=g).to(torch.bfloat16).to(cuda) for _ in range(3))
    plan = core.plan_block_causal(H, S, cuda, block=700, window=1400, sink=100)
    o = core.attn_fwd(q, k, v, plan)
    (q8, sq), (k8, sk), (v8, sv) = (core.quantize_e4m3(t) for t in (q, k, v))
    o8 = core.attn_fwd_fp8(q8, k8, v8, sq, sk, sv, plan)
    torch.testing.assert_close(o8.float(), o.float(), **FP8_TOL)


# --------------------------------------------------------------------------------------------
# compiled flex_attention under the same mask
# --------------------------------------------------------------------------------------------
def test_against_compiled_flex_attention(cuda):
    """The Wan 1.3B shape (12 heads, S = 32 760, chunks of 4 680), a CausVid-style `ends` mask_mod: forward within bf16
    rounding of compiled flex_attention."""
    try:
        from torch.nn.attention.flex_attention import create_block_mask, flex_attention

        flex = torch.compile(flex_attention)
    except Exception as e:  # pragma: no cover
        pytest.skip(f"flex_attention unavailable: {e}")
    from svgb200 import core

    H, S, C_ = 12, WAN_S, WAN_C
    ends = torch.div(torch.arange(S, device=cuda), C_, rounding_mode="floor").add(1).mul(C_).clamp(max=S)

    def mask_mod(b, h, q_idx, kv_idx):
        return kv_idx < ends[q_idx]

    g = torch.Generator().manual_seed(1)
    q, k, v = (torch.randn(1, H, S, 128, generator=g).to(torch.bfloat16).to(cuda) for _ in range(3))
    try:
        bmask = create_block_mask(mask_mod, 1, 1, S, S, device=cuda)
        ref = flex(q, k, v, block_mask=bmask)
    except Exception as e:  # pragma: no cover
        pytest.skip(f"flex_attention compilation unavailable: {e}")
    o = core.attn_fwd(q, k, v, core.plan_block_causal(H, S, cuda, block=C_))
    assert _rel(o, ref) < 1e-2, f"relative difference {_rel(o, ref):.2e}"


# --------------------------------------------------------------------------------------------
# KV cache
# --------------------------------------------------------------------------------------------
def _kplan(lens, Sq, kc, n=1, *, table=None, batch_idx=None, Snew=0, **blk):
    from svgb200 import core

    paged = table is not None
    return core.plan_kvcache(lens, q_len=Sq, num_blocks=kc.shape[0], new_len=Snew,
                             cache_len=None if paged else kc.shape[1], block_table=table,
                             page_size=kc.shape[1] if paged else None, cache_batch_idx=batch_idx, num_splits=n,
                             num_heads=8, **blk)


def _kfwd(q, kc, vc, plan, n=None, **kw):
    from svgb200 import core

    if n is not None and n > 1:
        _nan_partials(plan, q, n)
    out = torch.full(q.shape, float("nan"), dtype=torch.bfloat16 if kc.dtype == torch.float8_e4m3fn else q.dtype,
                     device=q.device)
    return core.attn_fwd(q, kc, vc, plan, return_lse=True, out=out, **kw)


def _blk(C_, F, W, sink):
    return dict(block=C_, first_block=F, window_size=(W, -1), sink=sink)


@pytest.mark.parametrize("kind", ["contiguous", "batch_idx", "paged"])
def test_kv_plan_matches_host_mirror(cuda, kind):
    from svgb200 import core

    seqlens, Sq, Snew = [900, -5, 10 ** 6, 0, 1500], 300, 40
    C_, F, W, sink = 200, 77, 450, 130
    g = random.Random(1)
    tab = bi = None
    if kind == "paged":
        page, nblocks, max_pages = 128, 20, 14
        tab = [[g.randrange(-3, 24) for _ in range(max_pages)] for _ in seqlens]
        table = torch.tensor(tab, dtype=torch.int32, device=cuda)
    else:
        page, nblocks, table = 1792, 6, None
        if kind == "batch_idx":
            bi = [4, 0, 2, 5, 1]
    lens = torch.tensor(seqlens, dtype=torch.int32, device=cuda)
    plan = core.plan_kvcache(lens, q_len=Sq, num_blocks=nblocks, new_len=Snew, block_table=table,
                             page_size=page if table is not None else None, cache_len=None if table is not None else page,
                             cache_batch_idx=None if bi is None else torch.tensor(bi, dtype=torch.int32, device=cuda),
                             **_blk(C_, F, W, sink))
    assert plan.desc.mask_mode == core.MASK_BLOCK_CAUSAL and plan.desc.kind == core.PLAN_KVCACHE
    items, Ls = bm.kv_plan(seqlens, Sq=Sq, new_len=Snew, nblocks=nblocks, block_rows=page, table=tab, batch_idx=bi,
                           sink=sink, block=C_, first_block=F, window=W)
    ws = plan.ws.cpu()
    i32 = ws.view(torch.int32)
    assert i32[0].item() == len(items)
    assert i32[4:4 + 2 + len(seqlens)].tolist() == [len(seqlens), Sq] + Ls
    got = _lists(plan)
    for (b, r0, nr, chunks), (g0, gn, gch) in zip(items, got):
        assert (g0, gn) == (r0, nr)
        want = [(row, ((valid - 1) & 0xff) | (256 if elem else 0) | (j << 10)) for row, valid, elem, j in chunks]
        assert gch == want, (kind, b, r0)


@pytest.mark.parametrize("paged", [False, True])
@pytest.mark.parametrize("blk", [(300, 300, -1, 0), (4680 // 4, 390, 2340, 390), (129, 1, 129, 200)], ids=_ids)
def test_kv_split_lists_concatenate_to_the_single_list(cuda, paged, blk):
    Ls, Sq, page = [2900, 0, 1300, 77], 300, 256
    g = torch.Generator().manual_seed(3)
    kc = _rand((len(Ls), 3072, 1, 64), torch.bfloat16, cuda, g)
    table = None
    if paged:
        kc, table = _paged_from(kc, Ls, page, 5, g, cuda)
    lens = torch.tensor(Ls, dtype=torch.int32, device=cuda)
    single = _lists(_kplan(lens, Sq, kc, 1, table=table, **_blk(*blk)))
    longest = max(len(c) for _, _, c in single)
    for n in (2, 3, 8, longest + 3):
        split = _lists(_kplan(lens, Sq, kc, n, table=table, **_blk(*blk)))
        assert len(split) == n * len(single)
        for i, (r0, nr, chunks) in enumerate(single):
            parts = [split[s * len(single) + i] for s in range(n)]
            assert all(p[:2] == (r0, nr) for p in parts), (n, i)
            assert [c for p in parts for c in p[2]] == chunks, (n, i)


def _ref64(q, ks, vs, Ls, args):
    """fp64 o [B, Sq, Hq, D], lse [B, Hq, Sq] under the block rule, from each stream's logical keys ks[b] [L_b, Hkv, D]"""
    B, Sq, Hq, D = q.shape
    mod = _mod(args)
    os, lses = [], []
    for b in range(B):
        L = Ls[b]
        G = Hq // ks[b].shape[1]
        k = ks[b].double().repeat_interleave(G, 1).transpose(0, 1)
        v = vs[b].double().repeat_interleave(G, 1).transpose(0, 1)
        p = torch.arange(Sq, device=q.device)[:, None] + (L - Sq)
        m = mod(p, torch.arange(L, device=q.device)[None, :])
        s = (q[b].double().transpose(0, 1) @ k.transpose(1, 2)) * D ** -0.5
        s = s.masked_fill(~m, float("-inf"))
        lse = torch.logsumexp(s, -1)
        os.append((torch.exp(s - lse[..., None]).nan_to_num(0.0) @ v).transpose(0, 1))
        lses.append(lse)
    return torch.stack(os), torch.stack(lses)


def _formats(kc_bf, g, cuda):
    """The same shape as a 16-bit cache, a per-head e4m3 cache and a per-row e4m3 cache: {name: (k, v, scale kwargs,
    k values, v values)}"""
    shape = kc_bf.shape
    vc_bf = _rand(shape, kc_bf.dtype, cuda, g)
    k8, ks, kd = _cache8(shape, cuda, g)
    v8, vs, vd = _cache8(shape, cuda, g)
    kr, ksr, krd, _ = _cache_rows(shape, cuda, g)
    vr, vsr, vrd, _ = _cache_rows(shape, cuda, g)
    return {"16": (kc_bf, vc_bf, {}, kc_bf, vc_bf), "e4m3": (k8, v8, dict(k_scale=ks, v_scale=vs), kd, vd),
            "e4m3 rows": (kr, vr, dict(k_scale=ksr, v_scale=vsr), krd, vrd)}


@pytest.mark.parametrize("fmt", ["bf16", "fp16", "e4m3", "e4m3 rows"])
@pytest.mark.parametrize("n", [1, 2, 3, 8, 0])
def test_kv_against_oracle(cuda, fmt, n):
    """Chunks of 300 keys against caches of several lengths (the last chunk mid-block, a stream shorter than q), a
    shorter first block, a window and a sink, GQA: o and lse against fp64 on the cache's values and, for the e4m3
    caches, on q as the call quantises it (per query head over the call's rows, or per row)."""
    Ls, Sq, Hkv, G, D = [2100, 700, 200, 3000], 300, 2, 4, 128
    args = (300, 100, 900, 130)
    g = torch.Generator().manual_seed(hash((fmt, n)) % 1000)
    dt = torch.float16 if fmt == "fp16" else torch.bfloat16
    q = _rand((len(Ls), Sq, G * Hkv, D), dt, cuda, g)
    k, v, kw, kd, vd = _formats(_rand((len(Ls), 3072, Hkv, D), dt, cuda, g), g, cuda)["16" if fmt in DT else fmt]
    lens = torch.tensor(Ls, dtype=torch.int32, device=cuda)
    plan = _kplan(lens, Sq, k, n, **_blk(*args))
    o, lse = _kfwd(q, k, v, plan, n, **kw)
    qd = q
    if fmt == "e4m3":
        sq = _head_scales(q)
        qd = _q8(q, sq).float() * sq[:, None]
    elif fmt == "e4m3 rows":
        q8, sq = _q8rows(q)
        qd = q8.float() * sq[..., None]
    eo, el = _ref64(qd, [kd[b, :L] for b, L in enumerate(Ls)], [vd[b, :L] for b, L in enumerate(Ls)], Ls, args)
    fin = torch.isfinite(el)
    assert torch.equal(fin, torch.isfinite(lse))
    if fmt in DT:
        assert torch.allclose(o.double(), eo, atol=2e-2, rtol=2e-2)
        assert torch.allclose(lse.double()[fin], el[fin], atol=1e-3, rtol=1e-3)
    else:
        # per-head e4m3: a few rows' lse differ from this model of the q quantisation by up to 1.7e-2 (measured on the
        # H100), so that format's lse is held to 2e-2; a dropped or extra 128-key chunk moves lse by 0.1 or more here
        torch.testing.assert_close(o.double(), eo, **FP8_TOL)
        torch.testing.assert_close(lse.double()[fin], el[fin], **(FP8_LSE if fmt == "e4m3 rows" else
                                                                  dict(rtol=0, atol=2e-2)))
    o2, l2 = _kfwd(q, k, v, plan, n, **kw)
    _eq("o", o2, o, "determinism")
    _eq("lse", l2, lse, "determinism")


@pytest.mark.parametrize("Sq", [1, 50])
def test_kv_one_live_split_is_the_single_pass(cuda, Sq):
    """Every stream holds at most 128 keys, so split 0 gets the only chunk: o and lse are the single pass's bits, in
    every cache format."""
    Ls, Hkv, D = [100, 128, 5, 0], 2, 128
    g = torch.Generator().manual_seed(11)
    q = _rand((len(Ls), Sq, 8, D), torch.bfloat16, cuda, g)
    lens = torch.tensor(Ls, dtype=torch.int32, device=cuda)
    for name, (k, v, kw, _, _) in _formats(_rand((len(Ls), 256, Hkv, D), torch.bfloat16, cuda, g), g, cuda).items():
        o1, l1 = _kfwd(q, k, v, _kplan(lens, Sq, k, 1, **_blk(60, 20, 60, 0)), **kw)
        for n in (2, 4):
            on, ln = _kfwd(q, k, v, _kplan(lens, Sq, k, n, **_blk(60, 20, 60, 0)), n, **kw)
            _eq("o", on, o1, f"{name} n={n} Sq={Sq}")
            _eq("lse", ln, l1, f"{name} n={n} Sq={Sq}")


def test_kv_paged_e4m3_against_contiguous(cuda):
    """A shuffled paged per-head e4m3 cache gives the contiguous cache's bits under the block rule."""
    Ls, Sq = [3000, 1234], 700
    g = torch.Generator().manual_seed(4)
    q = _rand((2, Sq, 8, 128), torch.bfloat16, cuda, g)
    k8, ks, _ = _cache8((2, 3072, 2, 128), cuda, g)
    v8, vs, _ = _cache8((2, 3072, 2, 128), cuda, g)
    lens = torch.tensor(Ls, dtype=torch.int32, device=cuda)
    blk = _blk(700, 700, 2100, 256)
    co, cl = _kfwd(q, k8, v8, _kplan(lens, Sq, k8, **blk), k_scale=ks, v_scale=vs)
    g2 = torch.Generator().manual_seed(9)
    kp, table = _paged8(k8, 256, 2, g2)
    g2 = torch.Generator().manual_seed(9)
    vp, _ = _paged8(v8, 256, 2, g2)
    po, pl = _kfwd(q, kp, vp, _kplan(lens, Sq, kp, table=table, **blk), k_scale=ks, v_scale=vs)
    _eq("o", po, co, "paged e4m3")
    _eq("lse", pl, cl, "paged e4m3")


def test_kv_chunk_matches_the_square_plan(cuda):
    """Self-Forcing's inference step: the third chunk of a sequence appended with kvcache_append and attended with the
    block rule equals the square block-causal plan's rows of that chunk on the whole sequence, within bf16 rounding."""
    from svgb200 import core

    C_, H, D = 1024, 4, 128
    S = 4 * C_
    g = torch.Generator().manual_seed(12)
    q, k, v = (torch.randn(1, H, S, D, generator=g).to(torch.bfloat16).to(cuda) for _ in range(3))
    o_sq = core.attn_fwd(q, k, v, core.plan_block_causal(H, S, cuda, block=C_, window=2 * C_, sink=256))
    kc, vc = (torch.zeros(1, S, H, D, dtype=torch.bfloat16, device=cuda) for _ in range(2))
    lens = torch.zeros(1, dtype=torch.int32, device=cuda)
    for c in range(3):  # the first three chunks, one append each
        rows = slice(c * C_, (c + 1) * C_)
        core.kvcache_append(kc, vc, k[:, :, rows].transpose(1, 2), v[:, :, rows].transpose(1, 2), lens)
        lens += C_
    qc = q[:, :, 2 * C_:3 * C_].transpose(1, 2).contiguous()
    plan = core.plan_kvcache(lens, q_len=C_, num_blocks=1, cache_len=S, **_blk(C_, C_, 2 * C_, 256))
    o = core.attn_fwd(qc, kc, vc, plan)
    ref = o_sq[:, :, 2 * C_:3 * C_].transpose(1, 2)
    torch.testing.assert_close(o.float(), ref.float(), atol=2e-2, rtol=2e-2)
    print(f"KV-cache chunk vs square plan: bit-identical={torch.equal(o, ref)}")


def test_kv_renumbered_first_block(cuda):
    """Lowering a rolling stream's positions by one 256-row page (the first page dropped, the table shifted, the sink
    none) with first_block = ((F - 256 - 1) mod C) + 1 gives the same o bit for bit."""
    C_, F, W, page = 700, 700, 1400, 256
    L, Sq = 3500, 300
    g = torch.Generator().manual_seed(13)
    q = _rand((1, Sq, 4, 128), torch.bfloat16, cuda, g)
    kc, vc = (_rand((1, 3584, 2, 128), torch.bfloat16, cuda, g) for _ in range(2))
    g2 = torch.Generator().manual_seed(5)
    kp, table = _paged_from(kc, [L], page, 0, g2, cuda)
    g2 = torch.Generator().manual_seed(5)
    vp, _ = _paged_from(vc, [L], page, 0, g2, cuda)
    lens = torch.tensor([L], dtype=torch.int32, device=cuda)
    a, la = _kfwd(q, kp, vp, _kplan(lens, Sq, kp, table=table, **_blk(C_, F, W, 0)))
    F2 = (F - page - 1) % C_ + 1
    table2 = torch.cat([table[:, 1:], table[:, :1]], 1)
    b, lb = _kfwd(q, kp, vp, _kplan(lens - page, Sq, kp, table=table2, **_blk(C_, F2, W, 0)))
    _eq("o", b, a, "renumbered")
    _eq("lse", lb, la, "renumbered")


def test_launch_counts(cuda):
    """One plan launch; one forward launch per square call (three backward launches once the key-major plan exists,
    one more the first time); a split KV-cache call is one plan, the attention and the merge."""
    from svgb200 import core

    S = 3000
    n0 = core.launch_count
    plan = core.plan_block_causal(2, S, cuda, block=700)
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
    kc = torch.randn(1, 4096, 2, 128, device=cuda).to(torch.bfloat16)
    qk = torch.randn(1, 100, 4, 128, device=cuda).to(torch.bfloat16)
    lens = torch.tensor([3000], dtype=torch.int32, device=cuda)
    for n, launches in ((1, 1), (4, 2)):
        n0 = core.launch_count
        p = core.plan_kvcache(lens, q_len=100, num_blocks=1, cache_len=4096, num_splits=n, **_blk(700, 700, -1, 0))
        assert core.launch_count - n0 == 1
        n0 = core.launch_count
        core.attn_fwd(qk, kc, kc, p)
        assert core.launch_count - n0 == launches
