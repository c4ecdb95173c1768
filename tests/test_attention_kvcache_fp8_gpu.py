"""The FP8 (e4m3) KV cache on the GPU: the quantising append bit for bit against torch's conversion and quantize_e4m3,
saturation, a paged cache bit for bit the contiguous one, grouped-query heads bit for bit MHA on repeated K/V and
scales, rolling eviction with recycled pages and NaN evicted rows, the key census, the exact FP8 online-softmax census
of oracle/softmax.py through a paged KV-cache plan (with its per-head scales, and with grouped-query heads), an fp64
reference on the dequantised inputs, determinism, svgb_attn_fwd_strided_e4m3 on band plans against svgb_attn_fwd and
on a variable-block plan with B = 2 and grouped-query heads, and the drop-in's launches, host synchronisation and
refusal under grad."""
import ctypes as C
import dataclasses

import numpy as np
import pytest
import torch

import kvcache_mask as km
from oracle import softmax as sm
from test_attention_kvcache_gpu import _eq, _rand, _ref64
from test_softmax_census_gpu import check

pytestmark = pytest.mark.gpu

E4M3 = torch.float8_e4m3fn
NAN8 = 0x7F  # an e4m3 NaN byte
FP8_TOL = dict(rtol=8e-2, atol=4e-2)  # tests/test_fp8_gpu.py
FP8_LSE = dict(rtol=1e-3, atol=5e-3)


def _q8(x, scale):
    """torch's conversion of the append: RN-satfinite(x * (1 / scale[h])) over [..., H, D]"""
    return (x.float() * (1 / scale)[:, None]).clamp(-448, 448).to(E4M3)


def _head_scales(x):
    """absmax / 448 per head of a [..., H, D] tensor, as quantize_e4m3 picks it"""
    return (x.float().abs().amax(dim=tuple(range(x.dim() - 2)) + (-1,)) / 448).clamp_min(1e-12)


def _fwd8(q, kc, vc, ks, vs, lens, *, Snew=0, table=None, batch_idx=None, causal=False, window_size=(-1, -1), sink=0):
    from svgb200 import core

    paged = table is not None
    plan = core.plan_kvcache(lens, q_len=q.shape[1], num_blocks=kc.shape[0], new_len=Snew,
                             cache_len=None if paged else kc.shape[1], block_table=table,
                             page_size=kc.shape[1] if paged else None, cache_batch_idx=batch_idx, causal=causal,
                             window_size=window_size, sink=sink)
    out = torch.full_like(q, float("nan"))
    return core.attn_fwd(q, kc, vc, plan, return_lse=True, out=out, k_scale=ks, v_scale=vs)


def _paged8(kc8, page, extra_pages, g):
    """The contiguous e4m3 cache [B, S_cache, H, D] as a zero-filled page pool under a shuffled block table."""
    B, S_cache, H, D = kc8.shape
    max_pages = (S_cache + page - 1) // page
    n = B * max_pages + extra_pages
    perm = torch.randperm(n, generator=g).tolist()
    pool = torch.zeros(n, page, H, D, dtype=torch.uint8, device=kc8.device)
    src = kc8.view(torch.uint8)
    for b in range(B):
        for i in range(max_pages):
            rows = src[b, i * page:(i + 1) * page]
            pool[perm[b * max_pages + i], :rows.shape[0]] = rows
    table = torch.tensor(perm[:B * max_pages], dtype=torch.int32).view(B, max_pages).to(kc8.device)
    return pool.view(E4M3), table


def _cache8(shape, cuda, g):
    """A random bf16 cache quantised per head: (e4m3 cache, scales [H], dequantised fp32 cache)"""
    x = _rand(shape, torch.bfloat16, cuda, g)
    s = _head_scales(x)
    x8 = _q8(x, s)
    return x8, s, x8.float() * s[:, None]


# --------------------------------------------------------------------------------------------
# append
# --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["contiguous", "paged", "batch_idx"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_append_e4m3_writes_exactly_the_quantised_rows(cuda, kind, dtype):
    from svgb200 import core

    B, Snew, H, D = 3, 70, 2, 128
    g = torch.Generator().manual_seed(31)
    k, v = (_rand((B, Snew, H, D), dtype, cuda, g) for _ in range(2))
    seqlens = [0, 300, 186]
    table = bi = None
    if kind == "paged":
        page, max_pages, nblk = 128, 4, 15
        tab = torch.randperm(nblk, generator=g)[:B * max_pages].view(B, max_pages).tolist()
        table = torch.tensor(tab, dtype=torch.int32, device=cuda)
        shape = (nblk, page, H, D)
    else:
        shape = (5, 512, H, D)
        if kind == "batch_idx":
            bi = torch.tensor([4, 0, 2], dtype=torch.int32, device=cuda)
    lens = torch.tensor(seqlens, dtype=torch.int32, device=cuda)
    # quantize_e4m3's bytes and scales per head over all new rows
    k8q, ks = core.quantize_e4m3(k.permute(2, 0, 1, 3).reshape(H, B * Snew, D))
    v8q, vs = core.quantize_e4m3(v.permute(2, 0, 1, 3).reshape(H, B * Snew, D))
    k8q, v8q = (t.view(H, B, Snew, D).permute(1, 2, 0, 3) for t in (k8q, v8q))
    for ks_, vs_, what in ((ks, vs, "quantize_e4m3 scales"), (ks / 4, vs / 8, "saturating")):
        kc, vc = (torch.full(shape, NAN8, dtype=torch.uint8, device=cuda).view(E4M3) for _ in range(2))
        n0 = core.launch_count
        core.kvcache_append(kc, vc, k, v, lens, block_table=table, cache_batch_idx=bi, k_scale=ks_, v_scale=vs_)
        assert core.launch_count - n0 == 1
        kb, vb = kc.view(torch.uint8), vc.view(torch.uint8)
        kref, vref = _q8(k, ks_).view(torch.uint8), _q8(v, vs_).view(torch.uint8)
        written = torch.zeros(shape[:2], dtype=torch.bool, device=cuda)
        for b in range(B):
            for i in range(Snew):
                t = seqlens[b] + i
                if table is not None:
                    blk, row = tab[b][t // 128], t % 128
                else:
                    blk, row = (bi[b].item() if bi is not None else b), t
                assert torch.equal(kb[blk, row], kref[b, i]) and torch.equal(vb[blk, row], vref[b, i]), (what, b, i)
                if what != "saturating":
                    assert torch.equal(kb[blk, row], k8q[b, i]) and torch.equal(vb[blk, row], v8q[b, i]), (what, b, i)
                written[blk, row] = True
        assert bool((kb[~written] == NAN8).all()) and bool((vb[~written] == NAN8).all()), "a row outside the new ones changed"
        if what == "saturating":
            mag = kc.float().abs()[written]
            assert mag.max().item() == 448.0 and int((mag == 448.0).sum()) > 0


# --------------------------------------------------------------------------------------------
# paged == contiguous, GQA == MHA, rolling eviction
# --------------------------------------------------------------------------------------------
# (lengths after the append, Sq, causal, window_size, sink, page): B of 1 and 3, L_b = 0, Sq > L_b
PAGED = [
    ([1000], 300, True, (-1, -1), 0, 256),
    ([1900, 0, 640], 256, False, (333, 0), 200, 128),
    ([90, 2300, 1], 700, False, (500, 70), 300, 384),
]


@pytest.mark.parametrize("case", range(len(PAGED)))
def test_paged_equals_contiguous(cuda, case):
    Ls, Sq, causal, window, sink, page = PAGED[case]
    B, D = len(Ls), 128
    S_cache = ((max(Ls) + page - 1) // page) * page
    g = torch.Generator().manual_seed(40 + case)
    q = _rand((B, Sq, 8, D), torch.bfloat16, cuda, g)
    kc, ks, _ = _cache8((B, S_cache, 2, D), cuda, g)
    vc, vs, _ = _cache8((B, S_cache, 2, D), cuda, g)
    lens = torch.tensor(Ls, dtype=torch.int32, device=cuda)
    o, lse = _fwd8(q, kc, vc, ks, vs, lens, causal=causal, window_size=window, sink=sink)
    kp, table = _paged8(kc, page, 3, torch.Generator().manual_seed(99))
    vp, table_v = _paged8(vc, page, 3, torch.Generator().manual_seed(99))
    assert torch.equal(table, table_v)
    po, plse = _fwd8(q, kp, vp, ks, vs, lens, table=table, causal=causal, window_size=window, sink=sink)
    _eq("o", po, o, PAGED[case])
    _eq("lse", plse, lse, PAGED[case])
    empty = torch.tensor([L == 0 for L in Ls], device=cuda)
    assert bool((o[empty] == 0).all()) and bool((lse[empty] == float("-inf")).all())


def test_gqa_equals_mha_on_repeated_kv(cuda):
    Ls, Sq, D, G = [1500, 129, 900], 200, 128, 3
    g = torch.Generator().manual_seed(50)
    q = _rand((3, Sq, 6, D), torch.bfloat16, cuda, g)
    kc, ks, _ = _cache8((3, 1600, 2, D), cuda, g)
    vc, vs, _ = _cache8((3, 1600, 2, D), cuda, g)
    lens = torch.tensor(Ls, dtype=torch.int32, device=cuda)
    o, lse = _fwd8(q, kc, vc, ks, vs, lens, window_size=(300, 0), sink=70)
    rep = lambda t: t.view(torch.uint8).repeat_interleave(G, 2).view(E4M3)  # noqa: E731
    ro, rlse = _fwd8(q, rep(kc), rep(vc), ks.repeat_interleave(G), vs.repeat_interleave(G), lens, window_size=(300, 0),
                     sink=70)
    _eq("o", o, ro, "gqa")
    _eq("lse", lse, rlse, "gqa")


def test_rolling_eviction_recycled_pages(cuda):
    """Pages behind a sink-plus-window stream's window were evicted and their ids recycled (or set to garbage), and the
    evicted rows of the contiguous cache are NaN bytes: the window never visits them."""
    page, frame, D = 256, 512, 128
    sink, window = frame, 3 * frame
    L, Sq = 12 * frame, frame
    g = torch.Generator().manual_seed(55)
    q = _rand((1, Sq, 4, D), torch.bfloat16, cuda, g)
    kc, ks, kd = _cache8((1, L, 2, D), cuda, g)
    vc, vs, vd = _cache8((1, L, 2, D), cuda, g)
    ev0, ev1 = sink, ((L - Sq - window) // page) * page
    lens = torch.tensor([L], dtype=torch.int32, device=cuda)
    n_pages = L // page
    ids = torch.randperm(n_pages, generator=g).tolist()
    table = list(ids)
    for i in range(ev0 // page, ev1 // page):
        table[i] = ids[n_pages - 1 - (i % 3)] if i % 2 else -7
    kpool, vpool = (torch.full((n_pages, page, 2, D), NAN8, dtype=torch.uint8, device=cuda) for _ in range(2))
    for i in range(n_pages):
        if not ev0 // page <= i < ev1 // page:
            kpool[ids[i]] = kc.view(torch.uint8)[0, i * page:(i + 1) * page]
            vpool[ids[i]] = vc.view(torch.uint8)[0, i * page:(i + 1) * page]
    for c in (kc, vc):
        c.view(torch.uint8)[0, ev0:ev1] = NAN8
    tt = torch.tensor([table], dtype=torch.int32, device=cuda)
    po, plse = _fwd8(q, kpool.view(E4M3), vpool.view(E4M3), ks, vs, lens, table=tt, causal=True,
                     window_size=(window, 0), sink=sink)
    co, clse = _fwd8(q, kc, vc, ks, vs, lens, causal=True, window_size=(window, 0), sink=sink)
    _eq("o", po, co, "rolling")
    _eq("lse", plse, clse, "rolling")
    kd[0, ev0:ev1] = 0
    vd[0, ev0:ev1] = 0
    eo, _ = _ref64(q, [kd[0]], [vd[0]], [L], sink, window, 0)
    torch.testing.assert_close(po.double(), eo, **FP8_TOL)


# --------------------------------------------------------------------------------------------
# census: q = 0, one-hot V codes; every output row the count of its allowed keys
# --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["causal", "sink_window"])
def test_forward_key_census_paged(cuda, case):
    D, page, H = 128, 256, 2
    Ls, Sq = [3000, 1234], 700
    sink, window = (0, (-1, -1)) if case == "causal" else (300, (517, 0))
    B = len(Ls)
    max_pages = (max(Ls) + page - 1) // page
    g = torch.Generator().manual_seed(8)
    table = torch.randperm(B * max_pages, generator=g).view(B, max_pages).to(torch.int32).to(cuda)
    q = torch.zeros(B, Sq, H, D, dtype=torch.bfloat16, device=cuda)
    kpool = torch.zeros(B * max_pages, page, H, D, dtype=E4M3, device=cuda)
    vpool = torch.zeros(B * max_pages, page, H, D, dtype=torch.uint8, device=cuda)
    code = torch.arange(max_pages * page, device=cuda) % D
    onehot = torch.nn.functional.one_hot(code, D).float()
    one8 = onehot.to(E4M3).view(torch.uint8)
    for b in range(B):
        for i in range(max_pages):
            vpool[table[b, i]] = one8[i * page:(i + 1) * page, None, :]
    ones = torch.ones(H, dtype=torch.float32, device=cuda)
    lens = torch.tensor(Ls, dtype=torch.int32, device=cuda)
    o, lse = _fwd8(q, kpool, vpool.view(E4M3), ones, ones, lens, table=table, causal=True, window_size=window,
                   sink=sink)
    left = 10 ** 9 if window[0] == -1 else window[0]
    allowed = np.frompyfunc(km.allowed, 5, 1)  # the plan's predicate on logical positions (tests/kvcache_mask.py)
    for b, L in enumerate(Ls):
        p = np.arange(Sq)[:, None] + (L - Sq)
        m = torch.from_numpy(allowed(p, np.arange(L)[None, :], sink, left, 0).astype(bool)).to(cuda)
        n = m.sum(1)
        inv = torch.where(n > 0, 1.0 / n.float(), torch.zeros_like(n, dtype=torch.float32))
        exp = ((m.float() @ onehot[:L]) * inv[:, None]).to(torch.bfloat16)
        for h in range(H):
            _eq("o", o[b, :, h], exp, (case, b, h))
            got = torch.where(torch.isfinite(lse[b, h]), torch.exp(lse[b, h].double()).round(),
                              torch.zeros_like(n, dtype=torch.float64))
            assert torch.equal(got.long(), n), (case, b, h)


# --------------------------------------------------------------------------------------------
# the exact FP8 online-softmax census (oracle/softmax.py) through a paged KV-cache plan
# --------------------------------------------------------------------------------------------
def _grouped(case, G):
    """The census case with each head repeated G times: query heads G j .. G j + G - 1 share key/value head j (its keys,
    values, c and v_scale), so the kernel must read k_scale and v_scale at the key/value head to match the closed form."""
    idx = torch.arange(case.H).repeat_interleave(G)
    return dataclasses.replace(case, name=f"{case.name}_g{G}", H=case.H * G, c=[case.c[i] for i in idx],
                               kcls=case.kcls[idx], kt=case.kt[idx], rcls=case.rcls[idx], v=case.v[idx],
                               vs=[case.vs[i] for i in idx])


@pytest.mark.parametrize("G", [1, 2])
@pytest.mark.parametrize("name", ["premise_e4m3_qk", "band_none"])
def test_softmax_census_fp8_paged(cuda, name, G):
    """q_scale, k_scale of oracle.softmax (q_scale * k_scale = 2 and 1/2 per key/value head, c = 1 from sm_scale) and
    v_scale 1/2 and 2; one stream of L = Sq keys with no mask, so the plan visits every 128-key chunk in ascending
    order, as the band plan does.  Query i sits at logical position i; the keys live in shuffled pages."""
    from svgb200 import core
    from svgb200._lib import check as lib_check
    from svgb200._lib import lib

    base = sm.premise_case("e4m3_qk") if name == "premise_e4m3_qk" else sm.band_case("none", c=sm.FP8_C, vs=sm.FP8_VS)
    assert base.c == sm.FP8_C and base.vs == sm.FP8_VS
    case = _grouped(base, G) if G > 1 else base
    S, D, Hq, Hkv = case.S, case.D, case.H, base.H
    q, k, v = (t.to(E4M3).view(torch.uint8) for t in case.tensors())  # [H, S, D], plan order = logical order
    k, v = k[::G], v[::G]  # one key/value head per group
    qs = torch.tensor([sm.FP8_QS[h // G] for h in range(Hq)], dtype=torch.float32, device=cuda)
    ks, vs = (torch.tensor(x, dtype=torch.float32, device=cuda) for x in (sm.FP8_KS, sm.FP8_VS))
    page = 256
    npages = (S + page - 1) // page
    g = torch.Generator().manual_seed(90 + G)
    ids = torch.randperm(npages + 3, generator=g)[:npages].tolist()
    pools = []
    for x in (k, v):
        pool = torch.zeros(npages + 3, page, Hkv, D, dtype=torch.uint8)
        rows = x.transpose(0, 1)  # [S, Hkv, D]
        for i, pid in enumerate(ids):
            chunk = rows[i * page:(i + 1) * page]
            pool[pid, :chunk.shape[0]] = chunk
        pools.append(pool.to(cuda))
    table = torch.tensor([ids], dtype=torch.int32, device=cuda)
    plan = core.plan_kvcache(torch.tensor([S], dtype=torch.int32, device=cuda), q_len=S, num_blocks=npages + 3,
                             block_table=table, page_size=page)
    q8 = q[None].contiguous().to(cuda)  # [1, Hq, S, D]
    kf, vf = (p.view(-1, Hkv, D) for p in pools)  # the cache as rows
    o = torch.full((1, Hq, S, D), float("nan"), dtype=torch.bfloat16, device=cuda)
    lse = torch.empty(Hq, S, dtype=torch.float32, device=cuda)
    st = lambda *x: (C.c_longlong * 3)(*x)  # noqa: E731
    lib_check(lib().svgb_attn_fwd_strided_e4m3(
        q8.data_ptr(), kf.data_ptr(), vf.data_ptr(), qs.data_ptr(), ks.data_ptr(), vs.data_ptr(), o.data_ptr(),
        lse.data_ptr(), 1, Hq, Hkv, S, kf.shape[0], D, st(*q8.stride()[:3]), st(Hkv * D, D, Hkv * D),
        st(Hkv * D, D, Hkv * D), st(*o.stride()[:3]), sm.scale_for(1.0), C.byref(plan.desc), plan.ws.data_ptr(),
        torch.cuda.current_stream().cuda_stream), "svgb_attn_fwd_strided_e4m3")
    check(cuda, case, o[0], lse, f"fp8 census {name} G={G} through a paged KV-cache plan")


# --------------------------------------------------------------------------------------------
# accuracy, determinism
# --------------------------------------------------------------------------------------------
def test_fp64_on_dequantised_inputs_and_determinism(cuda):
    from svgb200 import core

    B, Hq, Hkv, D = 3, 12, 4, 128
    Ls, Sq, S_cache = [2100, 513, 3000], 400, 3072
    g = torch.Generator().manual_seed(61)
    q = _rand((B, Sq, Hq, D), torch.bfloat16, cuda, g)
    kc, ks, kd = _cache8((B, S_cache, Hkv, D), cuda, g)
    vc, vs, vd = _cache8((B, S_cache, Hkv, D), cuda, g)
    lens = torch.tensor(Ls, dtype=torch.int32, device=cuda)
    o1, l1 = _fwd8(q, kc, vc, ks, vs, lens, window_size=(700, 50), sink=100)
    o2, l2 = _fwd8(q, kc, vc, ks, vs, lens, window_size=(700, 50), sink=100)
    _eq("o", o1, o2, "determinism")
    _eq("lse", l1, l2, "determinism")
    assert o1.dtype == torch.bfloat16 and l1.shape == (B, Hq, Sq)
    q8, qs = core.quantize_e4m3(q.reshape(B * Sq, Hq, D).transpose(0, 1).contiguous())  # what the call quantised
    qd = (q8.view(E4M3).float() * qs[:, None, None]).transpose(0, 1).reshape(B, Sq, Hq, D)
    eo, el = _ref64(qd, [kd[b, :L] for b, L in enumerate(Ls)], [vd[b, :L] for b, L in enumerate(Ls)], Ls, 100, 700, 50)
    torch.testing.assert_close(o1.double(), eo, **FP8_TOL)
    torch.testing.assert_close(l1.double(), el, **FP8_LSE)


# --------------------------------------------------------------------------------------------
# svgb_attn_fwd_strided_e4m3 on band plans
# --------------------------------------------------------------------------------------------
def _strided_e4m3(q8, k8, v8, qs, ks, vs, plan, sm_scale):
    from svgb200 import core
    from svgb200._lib import check, lib

    B, Hq, S, D = q8.shape
    o = torch.full((B, Hq, S, D), float("nan"), dtype=torch.bfloat16, device=q8.device)
    lse = torch.empty(B * Hq, S, dtype=torch.float32, device=q8.device)
    st = lambda t: (C.c_longlong * 3)(*t.stride()[:3])  # noqa: E731
    check(lib().svgb_attn_fwd_strided_e4m3(q8.data_ptr(), k8.data_ptr(), v8.data_ptr(), qs.data_ptr(), ks.data_ptr(),
                                           vs.data_ptr(), o.data_ptr(), lse.data_ptr(), B, Hq, k8.shape[1], S,
                                           k8.shape[2], D, st(q8), st(k8), st(v8), st(o), sm_scale,
                                           C.byref(plan.desc), plan.ws.data_ptr(),
                                           torch.cuda.current_stream().cuda_stream), "svgb_attn_fwd_strided_e4m3")
    return o, lse.view(B, Hq, S)


@pytest.mark.parametrize("G", [1, 3])
def test_strided_e4m3_band_plan(cuda, G):
    from svgb200 import core

    H, S, D = 6, 1300, 128
    Hkv = H // G
    g = torch.Generator().manual_seed(70 + G)
    q, k, v = (_rand((1, h, S, D), torch.bfloat16, cuda, g) for h in (H, Hkv, Hkv))
    (q8, qs), (k8, ks), (v8, vs) = (core.quantize_e4m3(t) for t in (q, k, v))
    plan = core.plan_local(H, S, cuda, window_size=(400, 90), sink=130)
    o, lse = _strided_e4m3(q8, k8, v8, qs, ks, vs, plan, 0.09)
    rep = lambda t: t.repeat_interleave(G, 1).contiguous()  # noqa: E731
    ro, rlse = core.attn_fwd_fp8(q8, rep(k8), rep(v8), qs, ks.repeat_interleave(G), vs.repeat_interleave(G), plan,
                                 return_lse=True, sm_scale=0.09)
    _eq("o", o, ro, ("band", G))
    _eq("lse", lse, rlse.view(1, H, S), ("band", G))


def test_strided_e4m3_varblock_batched_gqa(cuda):
    """A variable-block plan over the B * Hkv key/value heads with B = 2 and G = 3: q_scale is read at b Hq + hq and
    k_scale, v_scale at b Hkv + hq / G.  Equals attn_fwd_fp8 (svgb_attn_fwd) on K, V, their scales and the map repeated
    per group, bit for bit."""
    from svgb200 import core

    B, Hq, Hkv, S, D, blk = 2, 6, 2, 1024, 128, 64
    G, nb = Hq // Hkv, S // blk
    g = torch.Generator().manual_seed(80)
    q, k, v = (_rand((B, h, S, D), torch.bfloat16, cuda, g) for h in (Hq, Hkv, Hkv))
    (q8, qs), (k8, ks), (v8, vs) = (core.quantize_e4m3(t) for t in (q, k, v))
    bm = torch.rand(B * Hkv, nb, nb, generator=g) < 0.4
    bm |= torch.eye(nb, dtype=torch.bool)
    sizes = torch.full((B * Hkv, nb), blk, dtype=torch.int32)
    plan = core.plan_varblock(bm.to(cuda), sizes.to(cuda), sizes.to(cuda), S)
    o, lse = _strided_e4m3(q8, k8, v8, qs, ks, vs, plan, 0.07)
    rep = lambda t: t.repeat_interleave(G, 1).contiguous()  # noqa: E731
    rplan = core.plan_varblock(bm.repeat_interleave(G, 0).to(cuda), sizes.repeat_interleave(G, 0).to(cuda),
                               sizes.repeat_interleave(G, 0).to(cuda), S)
    ro, rlse = core.attn_fwd_fp8(q8, rep(k8), rep(v8), qs, ks.repeat_interleave(G), vs.repeat_interleave(G), rplan,
                                 return_lse=True, sm_scale=0.07)
    _eq("o", o, ro, "varblock B=2 G=3")
    _eq("lse", lse, rlse.view(B, Hq, S), "varblock B=2 G=3")


# --------------------------------------------------------------------------------------------
# the drop-in: launches, no host sync, grad
# --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seqlens", ["int", "tensor"])
def test_dropin_no_host_sync_and_launch_counts(cuda, seqlens):
    from svgb200 import core, patch

    B, page, H, D = 2, 256, 2, 128
    g = torch.Generator().manual_seed(66)
    kc, vc = (torch.zeros(8, page, H, D, dtype=E4M3, device=cuda) for _ in range(2))
    table = torch.tensor([[3, 1, 6], [0, 7, 2]], dtype=torch.int32, device=cuda)
    q = _rand((B, 50, 4, D), torch.bfloat16, cuda, g)
    k, v = (_rand((B, 50, H, D), torch.bfloat16, cuda, g) for _ in range(2))
    ks = vs = torch.full((H,), 1 / 64, dtype=torch.float32, device=cuda)
    lens = 200 if seqlens == "int" else torch.tensor([200, 500], dtype=torch.int32, device=cuda)
    torch.cuda.synchronize()
    n0 = core.launch_count
    torch.cuda.set_sync_debug_mode("error")
    try:
        o, lse = patch.flash_attn_with_kvcache(q, kc, vc, k, v, cache_seqlens=lens, block_table=table, causal=True,
                                               num_splits=4, return_softmax_lse=True, k_descale=ks, v_descale=vs)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    # append, plan, the three of quantize_e4m3 on q (absmax, scale, quantise), forward
    assert core.launch_count - n0 == 6
    assert o.shape == q.shape and o.dtype == torch.bfloat16 and lse.shape == (B, 4, 50)
    assert bool(torch.isfinite(o).all())


def test_grad_raises_before_any_launch(cuda):
    from svgb200 import core, patch
    from svgb200._lib import SvgbError

    kc = vc = torch.zeros(1, 256, 2, 128, dtype=E4M3, device=cuda)
    s = torch.ones(2, dtype=torch.float32, device=cuda)
    q = torch.zeros(1, 8, 2, 128, dtype=torch.bfloat16, device=cuda, requires_grad=True)
    n0 = core.launch_count
    with pytest.raises(SvgbError, match="no backward"):
        patch.flash_attn_with_kvcache(q, kc, vc, cache_seqlens=100, causal=True, k_descale=s, v_descale=s)
    assert core.launch_count == n0
