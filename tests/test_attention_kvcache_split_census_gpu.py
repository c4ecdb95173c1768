"""Split KV-cache attention (svgb_attn_fwd_kvcache_split) against the closed forms of oracle/kvsplit_census.py, on the
cases of tests/kvsplit_cases.py: the split lists read back from the plan against the host mirror piece by piece, every
fp32 partial o_s bit for bit and every partial lse inside its bounds (read from the test's own NaN-filled workspace),
the merged o and lse within the merge bound of the kernel's own partials and of the closed form's, the key census
counts exact, core.attn_fwd bit-identical to the direct call, and two calls giving the same bits."""
import ctypes as C

import numpy as np
import pytest
import torch

import kvsplit_cases as kc
from oracle import kvsplit_census as ks

pytestmark = pytest.mark.gpu

E4M3 = torch.float8_e4m3fn
NAN8 = 0x7F
DT = {"bf16": torch.bfloat16, "fp16": torch.float16, "e4m3": torch.bfloat16, "e4m3_rows": torch.bfloat16}
CHUNK_ELEM, LOGICAL_SHIFT = 1 << 8, 10  # attn_common.cuh: kChunkElem, kChunkLogicalShift


def _logical(case, cap, cuda, g):
    """K, V [B, cap, Hkv, D] by logical key (fp32 values) and per-row scale exponents [B, Hkv, cap]; rows past the
    last chunk a stream's plan can load are NaN"""
    B, Hkv, D = case.B, case.Hkv, case.D
    k = torch.where(torch.rand(B, cap, Hkv, D, generator=g) < 0.5, -1.0, 1.0)
    v = torch.zeros(B, cap, Hkv, D)
    for hk in range(Hkv):
        v[:, torch.arange(cap), hk, torch.from_numpy(ks.key_codes(cap, D, hk))] = 1.0
    dk = torch.randint(-2, 7, (B, Hkv, cap), generator=g).float()
    dv = torch.randint(-2, 7, (B, Hkv, cap), generator=g).float()
    for b, L in enumerate(case.Ls):
        end = -(-L // 128) * 128
        k[b, end:], v[b, end:] = float("nan"), float("nan")
    return k, v, dk, dv


def _encode(case, x, d):
    """logical fp32 rows -> the cache's element type: 16-bit, e4m3 (per-head scale 1) or e4m3 bytes x 2^-d (row scale
    2^d); NaN rows stay NaN"""
    if case.fmt in ("bf16", "fp16"):
        return x.to(DT[case.fmt])
    if case.fmt == "e4m3":
        y = x.to(E4M3).view(torch.uint8)
    else:
        y = (x * torch.exp2(-d).transpose(1, 2)[..., None]).to(E4M3).view(torch.uint8)
    return torch.where(torch.isnan(x), torch.full_like(y, NAN8), y)


def _place(case, cuda, g):
    """(q, k cache, v cache, scale kwargs, plan kwargs, (block of stream b, physical row of logical key t))"""
    B, Hkv, D, page = case.B, case.Hkv, case.D, case.page
    cap = 3072 if max(case.Ls) <= 3072 else -(-max(case.Ls) // page) * page
    k, v, dk, dv = _logical(case, cap, cuda, g)
    k8, v8 = _encode(case, k, dk), _encode(case, v, dv)
    nanval = NAN8 if case.fmt.startswith("e4m3") else float("nan")
    sk, sv = torch.exp2(dk), torch.exp2(dv)  # [B, Hkv, cap]
    if case.layout == "paged":
        mp = cap // page
        nb = B * mp + 3
        perm = torch.randperm(nb, generator=g)
        table = perm[:B * mp].view(B, mp).to(torch.int32)
        pools = [torch.full((nb, page, Hkv, D), nanval, dtype=k8.dtype) for _ in range(2)]
        spools = [torch.full((nb, Hkv, page), float("nan")) for _ in range(2)]
        for b in range(B):
            for i in range(mp):
                for pool, x in zip(pools, (k8, v8)):
                    pool[table[b, i]] = x[b, i * page:(i + 1) * page]
                for sp, s in zip(spools, (sk, sv)):
                    sp[table[b, i]] = s[b, :, i * page:(i + 1) * page]
        kw = dict(block_table=table.to(cuda), page_size=page)
        rows = page
        phys = lambda b, t: int(table[b, t // page]) * page + t % page  # noqa: E731
        kc_, vc_, ksr, vsr = pools + spools
    else:
        bi = None
        nb = B
        if case.layout == "batch_idx":
            nb = B + 2
            bi = torch.randperm(nb, generator=g)[:B].to(torch.int32)
        blocks = bi.tolist() if bi is not None else list(range(B))
        kc_, vc_ = (torch.full((nb, cap, Hkv, D), nanval, dtype=k8.dtype) for _ in range(2))
        ksr, vsr = (torch.full((nb, Hkv, cap), float("nan")) for _ in range(2))
        for b, blk in enumerate(blocks):
            kc_[blk], vc_[blk], ksr[blk], vsr[blk] = k8[b], v8[b], sk[b], sv[b]
        kw = dict(cache_len=cap, cache_batch_idx=bi.to(cuda) if bi is not None else None)
        rows = cap
        phys = lambda b, t: blocks[b] * cap + t  # noqa: E731
    if case.fmt.startswith("e4m3"):
        kc_, vc_ = kc_.view(E4M3), vc_.view(E4M3)
    scales = {}
    if case.fmt == "e4m3":
        one = torch.ones(Hkv, dtype=torch.float32, device=cuda)
        scales = dict(k_scale=one, v_scale=one.clone())
    elif case.fmt == "e4m3_rows":
        scales = dict(k_scale=ksr.contiguous().to(cuda), v_scale=vsr.contiguous().to(cuda))
    q = torch.zeros(B, case.Sq, case.Hq, D, dtype=DT[case.fmt], device=cuda)
    return q, kc_.to(cuda), vc_.to(cuda), scales, kw, rows, phys


def _plan(case, kcache, kw, n, cuda):
    from svgb200 import core

    lens = torch.tensor(case.Ls, dtype=torch.int32, device=cuda)
    return core.plan_kvcache(lens, q_len=case.Sq, num_blocks=kcache.shape[0], num_splits=n,
                             num_heads=case.Hq if n == 0 else None, **kw, **case.mask.plan_kwargs())


def _split_direct(fmt, q, kcache, vcache, scales, plan, n, sm_scale=None):
    """svgb_attn_fwd_kvcache_split on the test's own NaN-filled workspace, q quantised as core.attn_fwd does:
    (o [R, Hq, D], lse [Hq, R], o_part [n, R, Hq, D], lse_part [n, Hq, R])"""
    from svgb200 import core
    from svgb200._lib import check, lib

    B, Sq, Hq, D = q.shape
    R = B * Sq
    nb, rows, Hkv = kcache.shape[:3]
    nbytes = C.c_size_t()
    check(lib().svgb_attn_fwd_kvcache_split_bytes(n, R, Hq, D, C.byref(nbytes)), "svgb_attn_fwd_kvcache_split_bytes")
    ws = torch.full((nbytes.value // 4,), float("nan"), dtype=torch.float32, device=q.device)
    o = torch.full((R, Hq, D), float("nan"), dtype=DT[fmt], device=q.device)
    lse = torch.full((Hq, R), float("nan"), dtype=torch.float32, device=q.device)
    qf = q.reshape(R, Hq, D)
    if fmt in ("bf16", "fp16"):
        qx, qst, sc, dt, row, fill = qf, core._st(qf, "shd"), (None,) * 3, core._dt(q), 0, 8
        kf, vf = kcache.flatten(0, 1), vcache.flatten(0, 1)
    else:
        if fmt == "e4m3":
            qx, qs = core.quantize_e4m3(qf.transpose(0, 1).contiguous())
            qst, row = core._st(qx[None], "bhsd", 16), 0
        else:
            qx, qs = core.quantize_e4m3_rows(qf)
            qst, row = core._st(qx, "shd", 16), 1
        sc, dt, fill = (qs, scales["k_scale"], scales["v_scale"]), core._E4M3, 16
        kf, vf = (c.flatten(0, 1).view(torch.uint8) for c in (kcache, vcache))
    check(lib().svgb_attn_fwd_kvcache_split(
        qx.data_ptr(), kf.data_ptr(), vf.data_ptr(), *map(core._p, sc), o.data_ptr(), lse.data_ptr(), dt, row, B, Hq,
        Hkv, Sq, nb, rows, D, qst, core._st(kf, "shd", fill), core._st(vf, "shd", fill), core._st(o, "shd"),
        float(D) ** -0.5 if sm_scale is None else sm_scale, C.byref(plan.desc), plan.ws.data_ptr(), ws.data_ptr(), ws.numel() * 4,
        torch.cuda.current_stream().cuda_stream), "svgb_attn_fwd_kvcache_split")
    n_o = n * R * Hq * D
    return o, lse, ws[:n_o].view(n, R, Hq, D), ws[n_o:n_o + n * Hq * R].view(n, Hq, R)


def _lists(plan):
    ws = plan.ws.cpu()
    count = ws.view(torch.int32)[0].item()
    it = ws[plan.desc.items_off:].view(torch.int32)
    ch = ws[plan.desc.chunks_off:].view(torch.int32)
    out = []
    for i in range(count):
        d = it[8 * i:8 * i + 8].tolist()
        out.append((d[0], d[1] + d[5], [tuple(ch[2 * (d[2] + c):2 * (d[2] + c) + 2].tolist()) for c in range(d[3])]))
    return out


def _same(name, a, b, what):
    bad = ~(a == b)  # NaN never matches
    assert not bool(bad.any()), f"{what}: {name} differs in {int(bad.sum())} of {a.numel()} elements"


def _check(case, cuda):
    from svgb200 import core

    g = torch.Generator().manual_seed(1000 + case.seed)
    q, kcache, vcache, scales, kw, rows, phys = _place(case, cuda, g)
    plan = _plan(case, kcache, kw, case.n, cuda)
    B, Sq, Hq, D = q.shape
    n = plan.desc.max_items // (B * case.items_per_stream)
    assert n > 1, case.name  # the automatic count splits the production shapes
    if case.n == 0 and core.device_check()[2] == 132:
        assert n == kc.splits(case), (case.name, n)  # the count the CPU tests assume for this case
    what = f"{case.name} (n={n})"

    # the split lists, piece by piece
    want = ks.plan_lists(case, n)
    got = _lists(plan)
    assert len(got) == len(want), what
    for i, ((r0, nr, chunks), (wr0, wnr, wch)) in enumerate(zip(got, want)):
        b = wr0 // Sq
        assert (r0, nr) == (wr0, wnr), (what, i)
        exp = [(phys(b, 128 * j), min(128, case.Ls[b] - 128 * j) - 1 | (CHUNK_ELEM if e else 0) | j << LOGICAL_SHIFT)
               for j, e in wch]
        assert chunks == exp, (what, i)

    # partials: written everywhere, o_s bit for bit, lse_s inside its bounds
    o, lse, o_p, l_p = _split_direct(case.fmt, q, kcache, vcache, scales, plan, n)
    ns_, cnt, N = ks.key_census(case, n)
    eo, _ = ks.partials_fp32(ns_, cnt, case.G)
    lo, hi = ks.lse_partial_bounds(ns_, Hq)
    op, lp = o_p.cpu().numpy(), l_p.cpu().numpy()
    assert not np.isnan(op).any() and not np.isnan(lp).any(), f"{what}: a partial left unwritten"
    bad = op != eo
    assert not bad.any(), f"{what}: o_s differs in {int(bad.sum())} elements, first at {np.argwhere(bad)[0]}"
    fin = np.isfinite(lo)
    assert np.array_equal(np.isfinite(lp), fin), what
    assert bool(((lp[fin] >= lo[fin]) & (lp[fin] <= hi[fin])).all()), f"{what}: a partial lse outside its bounds"

    # the merge: within the bound of the kernel's partials and of the closed form's
    on, ln = o.double().cpu().numpy(), lse.cpu().numpy()
    dt = DT[case.fmt]
    y, beta, el, bl = ks.bound(op, lp)
    assert bool(ks.admissible(on, y, beta, dt).all()), f"{what}: merged o outside the bound of its partials"
    f = np.isfinite(el)
    assert np.array_equal(np.isfinite(ln), f), what
    assert bool((np.abs(ln[f] - el[f]) <= bl[f]).all()), f"{what}: merged lse outside the bound of its partials"
    assert bool((on[~f.T] == 0).all()), f"{what}: a row without keys is not 0"
    lo0, hi0 = np.where(fin, lo, 0), np.where(fin, hi, 0)
    yc, bc, elc, blc = ks.bound(eo, np.where(fin, (lo0 + hi0) / 2, -np.inf), (hi0 - lo0) / 2)
    assert bool(ks.admissible(on, yc, bc, dt).all()), f"{what}: merged o outside the closed form's bound"
    assert bool((np.abs(ln[f] - elc[f]) <= blc[f]).all()), f"{what}: merged lse outside the closed form's bound"
    # the key census: exp(lse) is the mask's count N
    got_n = np.where(np.isfinite(ln), np.rint(np.exp(ln.astype(np.float64))), 0).astype(np.int64)
    assert np.array_equal(got_n, np.broadcast_to(N[None], got_n.shape)), f"{what}: exp(lse) is not the key count"

    # core.attn_fwd on the same plan, and a second call: the same bits
    co, cl = core.attn_fwd(q, kcache, vcache, plan, return_lse=True, **scales)
    _same("o", co.reshape(B * Sq, Hq, D), o, f"{what}: core.attn_fwd")
    _same("lse", cl.transpose(0, 1).reshape(Hq, B * Sq), lse, f"{what}: core.attn_fwd")
    o2, l2, op2, lp2 = _split_direct(case.fmt, q, kcache, vcache, scales, plan, n)
    for name, a, b in (("o", o2, o), ("lse", l2, lse), ("o_part", op2, o_p), ("lse_part", lp2, l_p)):
        _same(name, a, b, f"{what}: determinism")


@pytest.mark.parametrize("case", kc.SMALL, ids=lambda c: c.name)
def test_split_census(cuda, case):
    _check(case, cuda)


@pytest.mark.parametrize("case", kc.PRODUCTION, ids=lambda c: c.name)
def test_split_census_production(cuda, case):
    _check(case, cuda)


def _merge_checks(what, dt, on, ln, op, lp, eo, lo, hi):
    """the merged o [R, Hq, D] (float64) and lse [Hq, R] within the bound of the kernel's partials (op, lp) and of the
    closed form's (eo, lse in [lo, hi])"""
    y, beta, el, bl = ks.bound(op, lp)
    assert bool(ks.admissible(on, y, beta, dt).all()), f"{what}: merged o outside the bound of its partials"
    f = np.isfinite(el)
    assert np.array_equal(np.isfinite(ln), f), what
    assert bool((np.abs(ln[f] - el[f]) <= bl[f]).all()), f"{what}: merged lse outside the bound of its partials"
    fin = np.isfinite(lo)
    lo0, hi0 = np.where(fin, lo, 0), np.where(fin, hi, 0)
    yc, bc, elc, blc = ks.bound(eo, np.where(fin, (lo0 + hi0) / 2, -np.inf), (hi0 - lo0) / 2)
    assert bool(ks.admissible(on, yc, bc, dt).all()), f"{what}: merged o outside the closed form's bound"
    assert bool((np.abs(ln[f] - elc[f]) <= blc[f]).all()), f"{what}: merged lse outside the closed form's bound"


@pytest.mark.parametrize("i", range(len(kc.SOFTMAX)), ids=lambda i: "{}_n{}_{}{}".format(*kc.SOFTMAX[i]))
def test_split_softmax_census(cuda, i):
    """oracle.softmax's census on one contiguous stream of S = 1 000 queries over its 1 000 keys: every split's partial
    o bit for bit and lse inside lse_bounds, where a row's hot split and its cold splits lie over 100 nats apart, and
    the merge within its bound: a merge without the max, or with m from any split but the top one, overflows here."""
    from svgb200 import core
    from oracle import softmax as sm

    base, mask, n, fmt = kc.softmax_case(i)
    S, H, D = base.S, base.H, base.D
    dt = DT[fmt]
    q, k, v = base.tensors()  # [H, S, D] integers, logical order
    cap = -(-S // 128) * 128
    kcache, vcache = (torch.zeros(1, cap, H, D, dtype=dt) for _ in range(2))
    kcache[0, :S], vcache[0, :S] = k.transpose(0, 1).to(dt), v.transpose(0, 1).to(dt)
    kcache, vcache = kcache.to(cuda), vcache.to(cuda)
    qg = q.transpose(0, 1)[None].to(dt).to(cuda)
    assert torch.equal(qg.float().cpu()[0], q.transpose(0, 1)) and torch.equal(vcache[0, :S].float().cpu(), v.transpose(0, 1))
    plan = core.plan_kvcache(torch.tensor([S], dtype=torch.int32, device=cuda), q_len=S, num_blocks=1, cache_len=cap,
                             num_splits=n, **mask.plan_kwargs())
    what = f"softmax census {kc.SOFTMAX[i]}"
    mirror = ks.Case("softmax", [S], S, H, 1, D, fmt, "contig", mask, n)
    got = _lists(plan)
    for (r0, nr, chunks), (wr0, wnr, wch) in zip(got, ks.plan_lists(mirror, n)):
        assert (r0, nr) == (wr0, wnr) and [c[1] >> LOGICAL_SHIFT for c in chunks] == [j for j, _ in wch], what
    scale = sm.scale_for(base.c[0])
    o, lse, o_p, l_p = _split_direct(fmt, qg, kcache, vcache, {}, plan, n, scale)
    eo, lo, hi, _, budget = ks.softmax_partials(base, mask, n)
    assert budget < sm.BUDGET, what
    op, lp = o_p.cpu().numpy(), l_p.cpu().numpy()
    assert not np.isnan(op).any() and not np.isnan(lp).any(), f"{what}: a partial left unwritten"
    bad = op != eo
    assert not bad.any(), f"{what}: o_s differs in {int(bad.sum())} elements, first at {np.argwhere(bad)[0]}"
    fin = np.isfinite(lo)
    assert np.array_equal(np.isfinite(lp), fin), what
    assert bool(((lp[fin] >= lo[fin]) & (lp[fin] <= hi[fin])).all()), f"{what}: a partial lse outside its bounds"
    assert float(lp[fin].max()) > 100, what  # the hot splits are live
    _merge_checks(what, dt, o.double().cpu().numpy(), lse.cpu().numpy(), op, lp, eo, lo, hi)
    co, cl = core.attn_fwd(qg, kcache, vcache, plan, return_lse=True, sm_scale=scale)
    _same("o", co.reshape(S, H, D), o, f"{what}: core.attn_fwd")
    _same("lse", cl[0], lse, f"{what}: core.attn_fwd")
    o2, l2, op2, lp2 = _split_direct(fmt, qg, kcache, vcache, {}, plan, n, scale)
    for name, a, b in (("o", o2, o), ("lse", l2, lse), ("o_part", op2, o_p), ("lse_part", lp2, l_p)):
        _same(name, a, b, f"{what}: determinism")
