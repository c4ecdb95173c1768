"""Variable-length KV-cache attention (svgb_attn_plan_kvcache_varlen, svgb_kvcache_append_varlen, plan_kvcache(
cu_seqlens_q=), flash_attn_with_kvcache(cu_seqlens_q=)) on the GPU: each stream's o and lse bit for bit a uniform plan
on that stream alone, uniform lengths bit for bit the uniform plan in every format, the plan's lists against the
per-stream lists, the varlen append against a per-stream loop, fp64, determinism, launch counts, no host
synchronisation and production sizes."""
import pytest
import torch

pytestmark = pytest.mark.gpu

DT = {"bf16": torch.bfloat16, "fp16": torch.float16}
PAGE = 256


def _cu(lens, cuda):
    out = [0]
    for n in lens:
        out.append(out[-1] + n)
    return torch.tensor(out, dtype=torch.int32, device=cuda)


def _rand(shape, dtype, cuda, g):
    return torch.randn(*shape, generator=g).clamp(-4, 4).to(dtype).to(cuda)


def _eq(name, a, b, what):
    bad = ~(a == b)  # NaN (an unwritten element) never matches
    assert not bool(bad.any()), f"{what}: {name} differs in {int(bad.sum())} of {a.numel()} elements"


class Cache:
    """B streams' caches in one layout: 'contig' (stream b in block b), 'batch_idx' (a permutation of blocks) or
    'paged' (256-row pages, shuffled table); per-stream geometry arguments for plan_kvcache and kvcache_append."""

    def __init__(self, layout, B, cap, Hkv, D, dtype, cuda, g, fill=None):
        self.layout, self.B, self.cap = layout, B, cap
        if layout == "paged":
            mp = -(-cap // PAGE)
            self.cap = mp * PAGE
            self.table = torch.randperm(B * mp, generator=g or torch.Generator().manual_seed(0)).to(torch.int32)
            self.table = self.table.view(B, mp).to(cuda)
            shape = (B * mp, PAGE, Hkv, D)
        else:
            shape = (B + 1, cap, Hkv, D)  # one spare block, so batch_idx is no identity
        self.bi = (torch.randperm(B + 1, generator=g)[:B].to(torch.int32).to(cuda) if layout == "batch_idx" else None)
        if fill is None and g is None:  # production sizes: drawn on the device (torch.manual_seed)
            self.k, self.v = (torch.randn(shape, device=cuda).clamp(-4, 4).to(dtype) for _ in range(2))
        elif fill is None:
            self.k, self.v = (_rand(shape, dtype, cuda, g) for _ in range(2))
        else:
            self.k, self.v = (torch.full(shape, fill, dtype=dtype, device=cuda) for _ in range(2))

    def geo(self, b=None):
        """geometry keywords for all streams (b None) or stream b alone"""
        s = slice(None) if b is None else slice(b, b + 1)
        if self.layout == "paged":
            return dict(block_table=self.table[s])
        bi = self.bi if self.bi is not None else torch.arange(self.B, dtype=torch.int32, device=self.k.device)
        return dict(cache_batch_idx=None if (b is None and self.bi is None) else bi[s])

    def plan_geo(self, b=None):
        paged = self.layout == "paged"
        return dict(num_blocks=self.k.shape[0], cache_len=None if paged else self.k.shape[1],
                    page_size=PAGE if paged else None, **self.geo(b))


MASKS = {
    "causal": dict(causal=True),
    "window": dict(window_size=(300, 0), sink=70),
    "block": dict(block=96, first_block=40, window_size=(320, -1), sink=30),
}
# (Lq_b, cache_seqlens_b, capacity): 0, 1, 255, 256, 257 queries, Lq_b > L_b, L_b = 0, a length clamped at capacity
CASES = [
    ([257, 0, 1, 256, 255], [1000, 300, 0, 2000, 40], 1300),
    ([3, 700, 0, 129], [1900, 10, 64, 0], 2000),
]
FORMATS = [("bf16", 128, 1), ("fp16", 64, 4), ("bf16", 64, 4), ("fp16", 128, 1)]


def _plan(core, lens, lq, cache, mask, n, Hq, b=None, **kw):
    """the varlen plan of every stream (b None), or the uniform plan of stream b alone"""
    if b is None:
        cu = _cu(lq, lens.device)
        return core.plan_kvcache(lens, cu_seqlens_q=cu, total_q=sum(lq), **cache.plan_geo(), **MASKS[mask],
                                 num_splits=n, num_heads=Hq, **kw)
    return core.plan_kvcache(lens[b:b + 1], q_len=lq[b], **cache.plan_geo(b), **MASKS[mask], num_splits=n,
                             num_heads=Hq)


def _splits(plan):
    return plan.desc.max_items // plan.desc.varlen_items


@pytest.mark.parametrize("n", [1, 2, 4, 0])
@pytest.mark.parametrize("mask", list(MASKS))
@pytest.mark.parametrize("layout", ["contig", "batch_idx", "paged"])
@pytest.mark.parametrize("fmt", range(len(FORMATS)))
@pytest.mark.parametrize("case", range(len(CASES)))
def test_per_stream_bit_for_bit(cuda, case, fmt, layout, mask, n):
    """Each stream's rows of one varlen call equal plan_kvcache(q_len=Lq_b) on that stream alone, with the split count
    the varlen plan used; outputs go into NaN-filled buffers."""
    from svgb200 import core

    lq, ls, cap = CASES[case]
    dtype, D, G = FORMATS[fmt]
    Hkv, B = 2, len(lq)
    Hq = G * Hkv
    g = torch.Generator().manual_seed(100 * case + fmt)
    cache = Cache(layout, B, cap, Hkv, D, DT[dtype], cuda, g)
    lens = torch.tensor(ls, dtype=torch.int32, device=cuda)
    q = _rand((sum(lq), Hq, D), DT[dtype], cuda, g)
    plan = _plan(core, lens, lq, cache, mask, n, Hq)
    assert plan.desc.varlen_items > 0 and (n == 0 or _splits(plan) == n)
    o = torch.full_like(q, float("nan"))
    o_, lse = core.attn_fwd(q, cache.k, cache.v, plan, return_lse=True, out=o)
    assert o_ is o and lse.shape == (Hq, sum(lq))
    cu = [0]
    for x in lq:
        cu.append(cu[-1] + x)
    for b in range(B):
        if lq[b] == 0:
            continue
        p = _plan(core, lens, lq, cache, mask, _splits(plan), Hq, b=b)
        ro, rlse = core.attn_fwd(q[None, cu[b]:cu[b + 1]], cache.k, cache.v, p, return_lse=True)
        what = (CASES[case], FORMATS[fmt], layout, mask, n, b)
        _eq("o", o[cu[b]:cu[b + 1]], ro[0], what)
        _eq("lse", lse[:, cu[b]:cu[b + 1]], rlse[0], what)


def _fp8_cache(cache, rows, g, cuda):
    """e4m3 copies of cache.k / cache.v and their scales: per head [Hkv] or per row [blocks, Hkv, block_rows]"""
    nb, br, Hkv, _ = cache.k.shape
    k8, v8 = (t.float().clamp(-448, 448).to(torch.float8_e4m3fn) for t in (cache.k, cache.v))
    if rows:
        ks, vs = (torch.exp2(torch.randint(-3, 3, (nb, Hkv, br), generator=g).float()).to(cuda) for _ in range(2))
    else:
        ks, vs = (torch.rand(Hkv, generator=g).add(0.25).to(cuda) for _ in range(2))
    return k8, v8, ks, vs


@pytest.mark.parametrize("n", [1, 3])
@pytest.mark.parametrize("fmt", ["bf16", "e4m3_head", "e4m3_rows"])
def test_uniform_lengths_equal_uniform_plan(cuda, fmt, n):
    """With every Lq_b = Sq the varlen plan's whole output equals plan_kvcache(q_len=Sq)'s, in every format."""
    from svgb200 import core

    B, Sq, Hq, Hkv, D = 3, 300, 4, 2, 128
    g = torch.Generator().manual_seed(7)
    cache = Cache("paged", B, 1500, Hkv, D, torch.bfloat16, cuda, g)
    lens = torch.tensor([900, 0, 1400], dtype=torch.int32, device=cuda)
    q = _rand((B, Sq, Hq, D), torch.bfloat16, cuda, g)
    kw, k, v = {}, cache.k, cache.v
    if fmt != "bf16":
        k, v, ks, vs = _fp8_cache(cache, fmt == "e4m3_rows", g, cuda)
        kw = dict(k_scale=ks, v_scale=vs)
    for mask in MASKS:
        pu = core.plan_kvcache(lens, q_len=Sq, **cache.plan_geo(), **MASKS[mask], num_splits=n)
        pv = _plan(core, lens, [Sq] * B, cache, mask, n, Hq)
        uo, ulse = core.attn_fwd(q, k, v, pu, return_lse=True, **kw)
        vo, vlse = core.attn_fwd(q.reshape(B * Sq, Hq, D), k, v, pv, return_lse=True, **kw)
        _eq("o", vo, uo.reshape(B * Sq, Hq, D), (fmt, n, mask))
        _eq("lse", vlse, ulse.transpose(0, 1).reshape(Hq, B * Sq), (fmt, n, mask))


@pytest.mark.parametrize("n", [1, 2])
@pytest.mark.parametrize("fmt", ["e4m3_head", "e4m3_rows"])
def test_fp8_per_stream(cuda, fmt, n):
    """e4m3 caches, per stream.  Per-head: q gets the same per-head absmax in every stream (a row of 8.0 at each
    stream's first row, |q| <= 4 elsewhere), so the per-stream calls quantise q with the same scales."""
    from svgb200 import core

    lq, ls, cap = CASES[0]
    Hq, Hkv, D, B = 4, 2, 128, len(lq)
    g = torch.Generator().manual_seed(11)
    cache = Cache("paged", B, cap, Hkv, D, torch.bfloat16, cuda, g)
    k8, v8, ks, vs = _fp8_cache(cache, fmt == "e4m3_rows", g, cuda)
    lens = torch.tensor(ls, dtype=torch.int32, device=cuda)
    q = _rand((sum(lq), Hq, D), torch.bfloat16, cuda, g)
    cu = [0]
    for x in lq:
        cu.append(cu[-1] + x)
    for b in range(B):
        if lq[b]:
            q[cu[b], :, 0] = 8.0
    for mask in MASKS:
        plan = _plan(core, lens, lq, cache, mask, n, Hq)
        o = torch.full_like(q, float("nan"))
        _, lse = core.attn_fwd(q, k8, v8, plan, return_lse=True, out=o, k_scale=ks, v_scale=vs)
        for b in range(B):
            if lq[b] == 0:
                continue
            p = _plan(core, lens, lq, cache, mask, n, Hq, b=b)
            ro, rlse = core.attn_fwd(q[None, cu[b]:cu[b + 1]], k8, v8, p, return_lse=True, k_scale=ks, v_scale=vs)
            _eq("o", o[cu[b]:cu[b + 1]], ro[0], (fmt, n, mask, b))
            _eq("lse", lse[:, cu[b]:cu[b + 1]], rlse[0], (fmt, n, mask, b))


def _lists(plan):
    """{item: (q0, nr, [chunks])} of stream 0 of every item with rows, read back from the plan's workspace"""
    d, ws = plan.desc, plan.ws
    items = ws[d.items_off:d.items_off + 32 * d.max_items].view(torch.int32).view(d.max_items, 2, 4).cpu()
    chunks = ws[d.chunks_off:].view(torch.int32).view(-1, 2).cpu()
    out = []
    for i in range(d.max_items):
        q0, nr, off, ln = (int(x) for x in items[i, 0])
        nr1 = int(items[i, 1, 1])
        out.append((q0, nr + nr1, [tuple(c) for c in chunks[off:off + ln].tolist()]))
    return out


@pytest.mark.parametrize("mask", list(MASKS))
@pytest.mark.parametrize("layout", ["contig", "paged"])
def test_plan_lists_concatenate(cuda, layout, mask):
    """The varlen plan's items are the per-stream uniform lists in stream order, rows offset by cu_q[b], then empty
    items; every split's lists concatenate to the single list."""
    from svgb200 import core

    lq, ls, cap = CASES[0]
    B = len(lq)
    g = torch.Generator().manual_seed(3)
    cache = Cache(layout, B, cap, 2, 64, torch.bfloat16, cuda, g)
    lens = torch.tensor(ls, dtype=torch.int32, device=cuda)
    single = _lists(_plan(core, lens, lq, cache, mask, 1, 2))
    want, cu = [], 0
    for b in range(B):
        if lq[b]:
            for q0, nr, ch in _lists(_plan(core, lens, lq, cache, mask, 1, 2, b=b)):
                want.append((q0 + cu, nr, ch))
        cu += lq[b]
    assert single[:len(want)] == want
    assert all(nr == 0 and not ch for _, nr, ch in single[len(want):])
    for n in (2, 3):
        sp = _lists(_plan(core, lens, lq, cache, mask, n, 2))
        I = len(single)
        for i, (q0, nr, ch) in enumerate(single):
            parts = [sp[s * I + i] for s in range(n)]
            assert all(p[:2] == (q0, nr) for p in parts)
            assert sum((p[2] for p in parts), []) == ch


@pytest.mark.parametrize("fmt", ["bf16", "fp16", "e4m3_head", "e4m3_rows"])
@pytest.mark.parametrize("layout", ["contig", "batch_idx", "paged"])
def test_append_equals_per_stream_loop(cuda, layout, fmt):
    """The varlen append writes exactly the new rows (and, per row, their scales) into sentinel-filled caches, bit for
    bit a per-stream loop of kvcache_append; a stream past its capacity is skipped as the uniform append skips it."""
    from svgb200 import core

    lnew, ls, cap = [5, 0, 300, 1, 400], [10, 7, 1000, 1299, 1200], 1300  # the last stream runs past capacity
    B, Hkv, D = len(lnew), 2, 128
    g = torch.Generator().manual_seed(5)
    dt = torch.float16 if fmt == "fp16" else torch.bfloat16
    fp8 = fmt.startswith("e4m3")
    c1 = Cache(layout, B, cap, Hkv, D, dt, cuda, g, fill=float("nan") if not fp8 else 0.0)
    if fp8:
        c1.k = torch.full(c1.k.shape, 0x7F, dtype=torch.uint8, device=cuda).view(torch.float8_e4m3fn)
        c1.v = c1.k.clone()
    kw = {}
    if fmt == "e4m3_head":
        kw = dict(k_scale=torch.full((Hkv,), 0.5, device=cuda), v_scale=torch.full((Hkv,), 0.25, device=cuda))
    elif fmt == "e4m3_rows":
        nb, br = c1.k.shape[:2]
        kw = dict(k_scale=torch.full((nb, Hkv, br), -7.0, device=cuda), v_scale=torch.full((nb, Hkv, br), -7.0, device=cuda))
    k, v = (_rand((sum(lnew), Hkv, D), dt, cuda, g) for _ in range(2))
    lens = torch.tensor(ls, dtype=torch.int32, device=cuda)
    ref_k, ref_v = c1.k.clone(), c1.v.clone()
    ref_kw = {n: t.clone() for n, t in kw.items()}
    core.kvcache_append(c1.k, c1.v, k, v, lens, cu_seqlens=_cu(lnew, cuda), **c1.geo(), **kw)
    cu = 0
    for b in range(B):
        if lnew[b]:
            core.kvcache_append(ref_k, ref_v, k[None, cu:cu + lnew[b]], v[None, cu:cu + lnew[b]], lens[b:b + 1],
                                **c1.geo(b), **ref_kw)
        cu += lnew[b]
    bits = (lambda t: t.view(torch.uint8)) if fp8 else (lambda t: t.view(torch.int16))  # NaN sentinels compare too
    _eq("k_cache", bits(c1.k), bits(ref_k), (layout, fmt))
    _eq("v_cache", bits(c1.v), bits(ref_v), (layout, fmt))
    for n in kw if fmt == "e4m3_rows" else ():
        _eq(n, kw[n], ref_kw[n], (layout, fmt))
    # exactly the new rows inside the capacity were written, and per row their scales
    for c in (c1.k, c1.v):
        sentinel = (torch.isnan(c) if not fp8 else c.view(torch.uint8) == 0x7F).all(-1).all(-1)
        assert int((~sentinel).sum()) == sum(min(n, max(c1.cap - s, 0)) for n, s in zip(lnew, ls))
    if fmt == "e4m3_rows":
        assert int((kw["k_scale"] != -7.0).sum()) == Hkv * sum(min(n, max(c1.cap - s, 0)) for n, s in zip(lnew, ls))


def _ref64(q, cache, lens, lq, sink, left, right):
    """fp64 o [total_q, Hq, D], lse [Hq, total_q] of the local mask from each stream's logical keys"""
    Hq, D = q.shape[1:]
    os, lses, cu = [], [], 0
    for b in range(len(lq)):
        L = min(int(lens[b]), cache.cap)
        if cache.layout == "paged":
            idx = cache.table[b].long()
            kb, vb = (t[idx].flatten(0, 1)[:L] for t in (cache.k, cache.v))
        else:
            blk = b if cache.bi is None else int(cache.bi[b])
            kb, vb = cache.k[blk, :L], cache.v[blk, :L]
        G = Hq // kb.shape[1]
        k = kb.double().repeat_interleave(G, 1).transpose(0, 1)
        v = vb.double().repeat_interleave(G, 1).transpose(0, 1)
        qq = q[cu:cu + lq[b]].double().transpose(0, 1)
        p = torch.arange(lq[b], device=q.device)[:, None] + (L - lq[b])
        kv = torch.arange(L, device=q.device)[None, :]
        m = (kv < sink) | ((p - kv <= left) & (kv - p <= right))
        s = (qq @ k.transpose(1, 2) * D ** -0.5).masked_fill(~m, float("-inf"))
        lse = torch.logsumexp(s, -1)
        os.append((torch.exp(s - lse[..., None]).nan_to_num(0.0) @ v).transpose(0, 1))
        lses.append(lse)
        cu += lq[b]
    return torch.cat(os), torch.cat(lses, 1)


@pytest.mark.parametrize("n", [1, 4])
@pytest.mark.parametrize("layout", ["contig", "paged"])
def test_fp64_and_determinism(cuda, layout, n):
    from svgb200 import core

    lq, ls, cap = CASES[1]
    Hq, Hkv, D = 4, 2, 128
    g = torch.Generator().manual_seed(9)
    cache = Cache(layout, len(lq), cap, Hkv, D, torch.bfloat16, cuda, g)
    lens = torch.tensor(ls, dtype=torch.int32, device=cuda)
    q = _rand((sum(lq), Hq, D), torch.bfloat16, cuda, g)
    plan = _plan(core, lens, lq, cache, "window", n, Hq)
    o, lse = core.attn_fwd(q, cache.k, cache.v, plan, return_lse=True)
    o2, lse2 = core.attn_fwd(q, cache.k, cache.v, plan, return_lse=True)
    _eq("o", o, o2, "determinism")
    _eq("lse", lse, lse2, "determinism")
    eo, else_ = _ref64(q, cache, lens, lq, 70, 300, 0)
    assert torch.allclose(o.double(), eo, atol=2e-2, rtol=2e-2)
    fin = torch.isfinite(else_)
    assert torch.equal(torch.isfinite(lse), fin)
    assert torch.allclose(lse.double()[fin], else_[fin], atol=1e-3, rtol=1e-3)
    assert bool((o[(~fin).transpose(0, 1)] == 0).all())  # rows without an allowed key: o = 0


@pytest.mark.parametrize("fp8", [False, True])
def test_dropin_launches_no_host_sync(cuda, fp8):
    """flash_attn_with_kvcache(cu_seqlens_q=, cu_seqlens_k_new=): append, plan and forward (3 launches, plus the per-head
    q quantisation of an FP8 cache), no host synchronisation, and each stream equal to the uniform drop-in on it."""
    from svgb200 import core
    from svgb200.patch import flash_attn_with_kvcache

    lq, lnew, ls = [1, 300, 0, 4], [1, 300, 0, 2], [0, 500, 64, 1000]
    B, Hq, Hkv, D, cap = len(lq), 4, 2, 128, 1536
    g = torch.Generator().manual_seed(13)
    cache = Cache("paged", B, cap, Hkv, D, torch.bfloat16, cuda, g)
    kw = {}
    if fp8:
        cache.k, cache.v, ks, vs = _fp8_cache(cache, False, g, cuda)
        kw = dict(k_descale=ks, v_descale=vs)
    ref_k, ref_v = cache.k.clone(), cache.v.clone()
    q = _rand((sum(lq), Hq, D), torch.bfloat16, cuda, g)
    for b, x in enumerate(lq):
        if x:
            q[sum(lq[:b]), :, 0] = 8.0  # one per-head absmax in every stream (FP8: same q scales per stream)
    k, v = (_rand((sum(lnew), Hkv, D), torch.bfloat16, cuda, g) for _ in range(2))
    lens = torch.tensor(ls, dtype=torch.int32, device=cuda)
    cu_q, cu_k = _cu(lq, cuda), _cu(lnew, cuda)
    torch.cuda.synchronize()
    n0 = core.launch_count
    torch.cuda.set_sync_debug_mode("error")
    try:
        o, lse = flash_attn_with_kvcache(q, cache.k, cache.v, k, v, cache_seqlens=lens, block_table=cache.table,
                                         causal=True, return_softmax_lse=True, cu_seqlens_q=cu_q,
                                         cu_seqlens_k_new=cu_k, max_seqlen_q=max(lq), **kw)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert core.launch_count - n0 == (6 if fp8 else 3)
    assert o.shape == q.shape and lse.shape == (Hq, sum(lq))
    cq = ck = 0
    for b in range(B):
        if lq[b]:
            ro, rlse = flash_attn_with_kvcache(q[None, cq:cq + lq[b]], ref_k, ref_v, k[None, ck:ck + lnew[b]],
                                               v[None, ck:ck + lnew[b]], cache_seqlens=lens[b:b + 1],
                                               block_table=cache.table[b:b + 1], causal=True,
                                               return_softmax_lse=True, **kw)
            _eq("o", o[cq:cq + lq[b]], ro[0], (fp8, b))
            _eq("lse", lse[:, cq:cq + lq[b]], rlse[0], (fp8, b))
        cq += lq[b]
        ck += lnew[b]


@pytest.mark.parametrize("n", [1, 0])
@pytest.mark.parametrize("Hq", [12, 40])
def test_production_wan_mixed_batch(cuda, Hq, n):
    """A Wan-480p batch (1 560 tokens per frame) on shuffled 256-row pages with a 1-frame sink and a 9-frame window: a
    1-frame first chunk into an empty cache, 3-frame chunks against 9 and 21 frames, a 1-frame chunk against 21 frames;
    each stream bit for bit the uniform plan on it."""
    from svgb200 import core

    P = 1560
    lq = [P, 3 * P, 3 * P, P]
    ls = [P, 12 * P, 24 * P, 22 * P]  # after the append
    B, D = len(lq), 128
    torch.manual_seed(21)
    cache = Cache("paged", B, 24 * P, Hq, D, torch.bfloat16, cuda, None)
    lens = torch.tensor(ls, dtype=torch.int32, device=cuda)
    q = torch.randn(sum(lq), Hq, D, device=cuda).clamp(-4, 4).to(torch.bfloat16)
    win = dict(window_size=(9 * P, 0), sink=P)
    plan = core.plan_kvcache(lens, cu_seqlens_q=_cu(lq, cuda), total_q=sum(lq), max_seqlen_q=max(lq),
                             **cache.plan_geo(), **win, num_splits=n, num_heads=Hq)
    o = torch.full_like(q, float("nan"))
    _, lse = core.attn_fwd(q, cache.k, cache.v, plan, return_lse=True, out=o)
    cu = 0
    for b in range(B):
        p = core.plan_kvcache(lens[b:b + 1], q_len=lq[b], **cache.plan_geo(b), **win, num_splits=_splits(plan))
        ro, rlse = core.attn_fwd(q[None, cu:cu + lq[b]], cache.k, cache.v, p, return_lse=True)
        _eq("o", o[cu:cu + lq[b]], ro[0], (Hq, n, b))
        _eq("lse", lse[:, cu:cu + lq[b]], rlse[0], (Hq, n, b))
        cu += lq[b]
