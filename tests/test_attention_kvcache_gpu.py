"""Attention into a KV cache (svgb_kvcache_append, svgb_attn_plan_kvcache, flash_attn_with_kvcache) on the GPU: a
contiguous cache bit for bit plan_local_varlen on each stream's valid rows, a paged cache with a shuffled block table
bit for bit the contiguous one, rolling eviction with recycled pages, the append into NaN-filled caches, the forward
key census on paged caches, fp64 references, determinism, the plan read back against the host mirror, launch counts,
no host synchronisation, and the refusal under grad."""
import random

import pytest
import torch

import kvcache_mask as km

pytestmark = pytest.mark.gpu

DT = {"bf16": torch.bfloat16, "fp16": torch.float16}


def _cu(lens):
    out = [0]
    for n in lens:
        out.append(out[-1] + n)
    return out


def _rand(shape, dtype, cuda, g):
    return torch.randn(*shape, generator=g).to(dtype).to(cuda)


def _window(causal, window_size, sink):
    return dict(causal=causal, window_size=window_size, sink=sink)


def _fwd(q, kc, vc, lens, *, Snew=0, table=None, batch_idx=None, causal=False, window_size=(-1, -1), sink=0):
    from svgb200 import core

    paged = table is not None
    plan = core.plan_kvcache(lens, q_len=q.shape[1], num_blocks=kc.shape[0], new_len=Snew,
                             cache_len=None if paged else kc.shape[1], block_table=table,
                             page_size=kc.shape[1] if paged else None, cache_batch_idx=batch_idx,
                             **_window(causal, window_size, sink))
    out = torch.full_like(q, float("nan"))
    return core.attn_fwd(q, kc, vc, plan, return_lse=True, out=out)


def _eq(name, a, b, what):
    bad = ~(a == b)  # NaN (an unwritten element) never matches
    assert not bool(bad.any()), f"{what}: {name} differs in {int(bad.sum())} of {a.numel()} elements"


def _ref64(q, ks, vs, Ls, sink, left, right, scale=None):
    """fp64 o [B, Sq, Hq, D], lse [B, Hq, Sq] from each stream's logical keys ks[b] [L_b, Hkv, D]"""
    B, Sq, Hq, D = q.shape
    scale = D ** -0.5 if scale is None else scale
    os, lses = [], []
    for b in range(B):
        L = Ls[b]
        G = Hq // ks[b].shape[1]
        k = ks[b].double().repeat_interleave(G, 1).transpose(0, 1)  # [Hq, L, D]
        v = vs[b].double().repeat_interleave(G, 1).transpose(0, 1)
        qq = q[b].double().transpose(0, 1)
        p = torch.arange(Sq, device=q.device)[:, None] + (L - Sq)
        kv = torch.arange(L, device=q.device)[None, :]
        m = (kv < sink) | ((p - kv <= left) & (kv - p <= right))
        s = (qq @ k.transpose(1, 2)) * scale
        s = s.masked_fill(~m, float("-inf"))
        lse = torch.logsumexp(s, -1)
        w = torch.exp(s - lse[..., None]).nan_to_num(0.0)
        os.append((w @ v).transpose(0, 1))
        lses.append(lse)
    return torch.stack(os), torch.stack(lses)


# --------------------------------------------------------------------------------------------
# contiguous cache == plan_local_varlen on the valid rows, bit for bit
# --------------------------------------------------------------------------------------------
# (lengths after the append, Sq, causal, window_size, sink): causal, windows with edges inside chunks, sinks ending
# mid-chunk, L_b = 0, Sq > L_b, decode Sq = 1
CONTIG = [
    ([1000], 300, True, (-1, -1), 0),
    ([777, 0, 1300], 260, True, (-1, -1), 0),
    ([1500, 129, 900], 200, False, (300, 0), 70),
    ([640, 2000, 5], 130, False, (255, 17), 0),
    ([100, 600, 1], 1, True, (-1, -1), 0),
    ([50, 400, 901], 120, False, (-1, -1), 0),
]


@pytest.mark.parametrize("Hq,Hkv", [(4, 4), (6, 2)])
@pytest.mark.parametrize("D,dtype", [(128, "bf16"), (64, "fp16")])
@pytest.mark.parametrize("case", range(len(CONTIG)))
def test_contiguous_equals_varlen(cuda, case, D, dtype, Hq, Hkv):
    from svgb200 import core

    Ls, Sq, causal, window, sink = CONTIG[case]
    B, S_cache, dt = len(Ls), max(Ls) + 77, DT[dtype]
    g = torch.Generator().manual_seed(case)
    q = _rand((B, Sq, Hq, D), dt, cuda, g)
    kc, vc = (_rand((B, S_cache, Hkv, D), dt, cuda, g) for _ in range(2))
    lens = torch.tensor(Ls, dtype=torch.int32, device=cuda)
    o, lse = _fwd(q, kc, vc, lens, causal=causal, window_size=window, sink=sink)
    # the same streams packed: query segment b = its Sq rows, key segment b = its L_b valid rows
    kp = torch.cat([kc[b, :Ls[b]] for b in range(B)])
    vp = torch.cat([vc[b, :Ls[b]] for b in range(B)])
    t = lambda c: torch.tensor(c, dtype=torch.int32, device=cuda)  # noqa: E731
    plan = core.plan_local_varlen(t(_cu([Sq] * B)), t(_cu(Ls)), total_q=B * Sq, total_k=sum(Ls), causal=causal,
                                  window_size=window, sink=sink)
    ro, rlse = core.attn_fwd(q.reshape(B * Sq, Hq, D), kp, vp, plan, layout="shd", return_lse=True)
    _eq("o", o, ro.view(B, Sq, Hq, D), CONTIG[case])
    _eq("lse", lse, rlse.view(Hq, B, Sq).transpose(0, 1), CONTIG[case])
    left, right = window
    left = 10 ** 9 if left == -1 else left
    right = 0 if causal else (10 ** 9 if right == -1 else right)
    eo, else_ = _ref64(q, [kc[b, :Ls[b]] for b in range(B)], [vc[b, :Ls[b]] for b in range(B)], Ls, sink, left, right)
    assert torch.allclose(o.double(), eo, atol=2e-2, rtol=2e-2)
    fin = torch.isfinite(else_)
    assert torch.equal(fin, torch.isfinite(lse))
    assert torch.allclose(lse.double()[fin], else_[fin], atol=1e-3, rtol=1e-3)
    assert bool((o[~torch.isfinite(lse).transpose(1, 2)] == 0).all())  # rows without keys: o = 0


def _paged_from(kc, Ls, page, extra_pages, g, cuda):
    """The contiguous cache kc [B, S_cache, H, D] as a page pool with a shuffled block table, and the rest of the pool
    filled with other finite values."""
    B, S_cache, H, D = kc.shape
    max_pages = (S_cache + page - 1) // page
    n = B * max_pages + extra_pages
    perm = torch.randperm(n, generator=g).tolist()
    pool = torch.randn(n, page, H, D, generator=g).to(kc.dtype).to(cuda)
    table = torch.tensor(perm[:B * max_pages], dtype=torch.int32).view(B, max_pages).to(cuda)
    for b in range(B):
        for i in range(max_pages):
            rows = kc[b, i * page:(i + 1) * page]
            pool[perm[b * max_pages + i], :rows.shape[0]] = rows
    return pool, table


# paged == contiguous: causal, a window edge and a sink edge inside non-identity pages
PAGED = [
    ([1000, 1700], 300, True, (-1, -1), 0, 256),
    ([1900, 0, 640], 256, False, (333, 0), 200, 128),
    ([2300], 700, False, (500, 70), 300, 384),
    ([1, 1024], 1, True, (-1, -1), 129, 256),
]


@pytest.mark.parametrize("D,dtype", [(128, "bf16"), (64, "fp16")])
@pytest.mark.parametrize("case", range(len(PAGED)))
def test_paged_equals_contiguous(cuda, case, D, dtype):
    Ls, Sq, causal, window, sink, page = PAGED[case]
    B, dt = len(Ls), DT[dtype]
    S_cache = ((max(Ls) + page - 1) // page) * page
    g = torch.Generator().manual_seed(10 + case)
    q = _rand((B, Sq, 8, D), dt, cuda, g)
    kc, vc = (_rand((B, S_cache, 2, D), dt, cuda, g) for _ in range(2))
    lens = torch.tensor(Ls, dtype=torch.int32, device=cuda)
    o, lse = _fwd(q, kc, vc, lens, causal=causal, window_size=window, sink=sink)
    g2 = torch.Generator().manual_seed(99)
    kp, table = _paged_from(kc, Ls, page, 3, g2, cuda)
    g2 = torch.Generator().manual_seed(99)
    vp, table_v = _paged_from(vc, Ls, page, 3, g2, cuda)
    assert torch.equal(table, table_v)
    po, plse = _fwd(q, kp, vp, lens, table=table, causal=causal, window_size=window, sink=sink)
    _eq("o", po, o, PAGED[case])
    _eq("lse", plse, lse, PAGED[case])


def test_rolling_eviction_recycled_pages(cuda):
    """A sink-plus-window stream over pages: the pages behind the window were evicted and their ids recycled for the
    newest frames (or set to garbage), and the evicted rows of the contiguous reference are NaN.  The window never
    visits them, so the paged result equals the contiguous one bit for bit and the fp64 reference."""
    page, frame, D, dt = 256, 512, 128, torch.bfloat16
    sink, window = frame, 3 * frame  # one-frame sink, three frames back
    L, Sq = 12 * frame, frame         # 12 frames, the last one queries
    g = torch.Generator().manual_seed(5)
    q = _rand((1, Sq, 4, D), dt, cuda, g)
    kc, vc = (_rand((1, L, 2, D), dt, cuda, g) for _ in range(2))
    # keys behind every query's window and past the sink: whole pages [sink, L - Sq - window) rounded inwards
    ev0, ev1 = sink, ((L - Sq - window) // page) * page
    assert ev1 - ev0 >= 4 * page
    lens = torch.tensor([L], dtype=torch.int32, device=cuda)
    # paged: the logical pages of the evicted range hold recycled ids (also in use by the newest pages) or garbage
    n_pages = L // page
    ids = torch.randperm(n_pages, generator=g).tolist()
    table = list(ids)
    for i in range(ev0 // page, ev1 // page):
        table[i] = ids[n_pages - 1 - (i % 3)] if i % 2 else -7
    kpool, vpool = (torch.full((n_pages, page, 2, D), float("nan"), dtype=dt, device=cuda) for _ in range(2))
    for i in range(n_pages):
        if ev0 // page <= i < ev1 // page:
            continue
        kpool[ids[i]] = kc[0, i * page:(i + 1) * page]
        vpool[ids[i]] = vc[0, i * page:(i + 1) * page]
    kc[0, ev0:ev1] = float("nan")
    vc[0, ev0:ev1] = float("nan")
    tt = torch.tensor([table], dtype=torch.int32, device=cuda)
    po, plse = _fwd(q, kpool, vpool, lens, table=tt, causal=True, window_size=(window, 0), sink=sink)
    co, clse = _fwd(q, kc, vc, lens, causal=True, window_size=(window, 0), sink=sink)
    _eq("o", po, co, "rolling")
    _eq("lse", plse, clse, "rolling")
    kref, vref = kc[0].clone(), vc[0].clone()
    kref[ev0:ev1] = 0
    vref[ev0:ev1] = 0
    eo, _ = _ref64(q, [kref], [vref], [L], sink, window, 0)
    assert torch.allclose(po.double(), eo, atol=2e-2, rtol=2e-2)


# --------------------------------------------------------------------------------------------
# append
# --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["contiguous", "paged", "batch_idx"])
@pytest.mark.parametrize("D,dtype", [(128, "bf16"), (64, "fp16")])
def test_append_writes_exactly_the_new_rows(cuda, kind, D, dtype):
    from svgb200 import core

    dt, B, Snew, H = DT[dtype], 3, 70, 2
    g = torch.Generator().manual_seed(3)
    k, v = (_rand((B, Snew, H, D), dt, cuda, g) for _ in range(2))
    seqlens = [0, 300, 186]
    table = bi = None
    if kind == "paged":
        page, max_pages = 128, 4
        kc, vc = (torch.full((15, page, H, D), float("nan"), dtype=dt, device=cuda) for _ in range(2))
        tab = torch.randperm(15, generator=g)[:B * max_pages].view(B, max_pages).tolist()
        table = torch.tensor(tab, dtype=torch.int32, device=cuda)
    else:
        kc, vc = (torch.full((5, 512, H, D), float("nan"), dtype=dt, device=cuda) for _ in range(2))
        if kind == "batch_idx":
            bi = torch.tensor([4, 0, 2], dtype=torch.int32, device=cuda)
    lens = torch.tensor(seqlens, dtype=torch.int32, device=cuda)
    n0 = core.launch_count
    core.kvcache_append(kc, vc, k, v, lens, block_table=table, cache_batch_idx=bi)
    assert core.launch_count - n0 == 1
    written = torch.zeros(kc.shape[:2], dtype=torch.bool, device=cuda)
    for b in range(B):
        for i in range(Snew):
            t = seqlens[b] + i
            if table is not None:
                blk, row = tab[b][t // 128], t % 128
            else:
                blk, row = (bi[b].item() if bi is not None else b), t
            assert torch.equal(kc[blk, row], k[b, i]) and torch.equal(vc[blk, row], v[b, i]), (kind, b, i)
            written[blk, row] = True
    assert bool(kc[~written].isnan().all()) and bool(vc[~written].isnan().all()), "a row outside the new ones changed"


def test_append_then_attend_strided_new_rows(cuda):
    """The drop-in: k, v given as views of a packed projection, appended and attended in one call."""
    from svgb200 import patch

    dt, B, S_cache, H, D, Snew = torch.bfloat16, 2, 1024, 2, 128, 100
    g = torch.Generator().manual_seed(4)
    kc, vc = (_rand((B, S_cache, H, D), dt, cuda, g) for _ in range(2))
    kv = _rand((B, Snew, 2, H, D), dt, cuda, g)
    k, v = kv.unbind(2)
    q = _rand((B, Snew, 4, D), dt, cuda, g)
    lens = torch.tensor([300, 700], dtype=torch.int32, device=cuda)
    kref, vref = kc.clone(), vc.clone()
    o = patch.flash_attn_with_kvcache(q, kc, vc, k, v, cache_seqlens=lens, causal=True)
    for b, s in enumerate([300, 700]):
        kref[b, s:s + Snew], vref[b, s:s + Snew] = k[b], v[b]
    assert torch.equal(kc, kref) and torch.equal(vc, vref)
    ro, _ = _fwd(q, kref, vref, lens + Snew, causal=True)
    _eq("o", o, ro, "drop-in")


# --------------------------------------------------------------------------------------------
# census: q = 0 and one-hot key codes, every output row the count of its allowed keys
# --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["causal", "sink_window"])
def test_forward_key_census_paged(cuda, case):
    dt, D, page, H = torch.float16, 128, 256, 2
    Ls, Sq = [3000, 1234], 700
    sink, window = (0, (-1, -1)) if case == "causal" else (300, (517, 0))
    B = len(Ls)
    max_pages = (max(Ls) + page - 1) // page
    g = torch.Generator().manual_seed(8)
    ids = torch.randperm(B * max_pages, generator=g)
    table = ids.view(B, max_pages).to(torch.int32).to(cuda)
    q = torch.zeros(B, Sq, H, D, dtype=dt, device=cuda)
    kpool = torch.zeros(B * max_pages, page, H, D, dtype=dt, device=cuda)
    vpool = torch.zeros_like(kpool)
    code = torch.arange(max_pages * page, device=cuda) % D  # logical key j -> one-hot column j mod D
    onehot = torch.nn.functional.one_hot(code, D).to(dt)
    for b in range(B):
        for i in range(max_pages):
            vpool[table[b, i]] = onehot[i * page:(i + 1) * page, None, :]
    lens = torch.tensor(Ls, dtype=torch.int32, device=cuda)
    o, lse = _fwd(q, kpool, vpool, lens, table=table, causal=True, window_size=window, sink=sink)
    left = 10 ** 9 if window[0] == -1 else window[0]
    for b, L in enumerate(Ls):
        p = torch.arange(Sq, device=cuda)[:, None] + (L - Sq)
        kv = torch.arange(L, device=cuda)[None, :]
        m = (kv < sink) | ((p - kv <= left) & (kv - p <= 0))
        n = m.sum(1)
        cnt = (m.to(torch.float32) @ onehot[:L].float())  # [Sq, D]
        inv = torch.where(n > 0, 1.0 / n.float(), torch.zeros_like(n, dtype=torch.float32))
        exp = (cnt * inv[:, None]).to(dt)
        for h in range(H):
            _eq("o", o[b, :, h], exp, (case, b, h))
            got_n = torch.where(torch.isfinite(lse[b, h]), torch.exp(lse[b, h].double()).round(), torch.zeros_like(n, dtype=torch.float64))
            assert torch.equal(got_n.long(), n), (case, b, h)


# --------------------------------------------------------------------------------------------
# plan read-back, determinism, launches, host syncs, grad
# --------------------------------------------------------------------------------------------
def test_plan_matches_host_mirror(cuda):
    from svgb200 import core

    seqlens, Sq, Snew, page = [900, -5, 10 ** 6, 0], 300, 40, 128
    g = random.Random(1)
    nblocks, max_pages = 20, 9
    tab = [[g.randrange(-3, 24) for _ in range(max_pages)] for _ in seqlens]
    table = torch.tensor(tab, dtype=torch.int32, device=cuda)
    lens = torch.tensor(seqlens, dtype=torch.int32, device=cuda)
    kw = dict(sink=130, left=250, right=0)
    plan = core.plan_kvcache(lens, q_len=Sq, num_blocks=nblocks, new_len=Snew, block_table=table, page_size=page,
                             causal=True, window_size=(kw["left"], 0), sink=kw["sink"])
    items, Ls = km.plan(seqlens, Sq=Sq, new_len=Snew, nblocks=nblocks, block_rows=page, table=tab, **kw)
    ws = plan.ws.cpu()
    i32 = ws.view(torch.int32)
    assert i32[0].item() == len(items)
    kvt = i32[4:4 + 2 + len(seqlens)].tolist()
    assert kvt == [len(seqlens), Sq] + Ls
    desc = plan.desc
    it = ws[desc.items_off:].view(torch.int32)
    ch = ws[desc.chunks_off:].view(torch.int32)
    for n, (b, r0, nr, chunks) in enumerate(items):
        s0 = it[8 * n:8 * n + 8].tolist()
        assert s0[0] == r0 and s0[1] == min(nr, 128) and s0[5] == max(nr - 128, 0) and s0[4] == r0 + 128
        off, cnt = s0[2], s0[3]
        got = [tuple(ch[2 * (off + c):2 * (off + c) + 2].tolist()) for c in range(cnt)]
        want = [(row, ((valid - 1) & 0xff) | (256 if elem else 0) | (j << 10)) for row, valid, elem, j in chunks]
        assert got == want, (b, r0)


def test_fp64_random_and_determinism(cuda):
    dt, B, Hq, Hkv, D = torch.bfloat16, 3, 12, 4, 128
    Ls, Sq, S_cache = [2100, 513, 3000], 400, 3072
    g = torch.Generator().manual_seed(21)
    q = _rand((B, Sq, Hq, D), dt, cuda, g)
    kc, vc = (_rand((B, S_cache, Hkv, D), dt, cuda, g) for _ in range(2))
    lens = torch.tensor(Ls, dtype=torch.int32, device=cuda)
    o1, l1 = _fwd(q, kc, vc, lens, window_size=(700, 50), sink=100)
    o2, l2 = _fwd(q, kc, vc, lens, window_size=(700, 50), sink=100)
    _eq("o", o1, o2, "determinism")
    _eq("lse", l1, l2, "determinism")
    eo, el = _ref64(q, [kc[b, :L] for b, L in enumerate(Ls)], [vc[b, :L] for b, L in enumerate(Ls)], Ls, 100, 700, 50)
    assert (o1.double() - eo).abs().max().item() < 2e-2
    assert (l1.double() - el).abs().max().item() < 1e-3


@pytest.mark.parametrize("seqlens", ["int", "tensor"])
def test_dropin_no_host_sync_and_launch_counts(cuda, seqlens):
    from svgb200 import core, patch

    dt, B, page, H, D = torch.bfloat16, 2, 256, 2, 64
    g = torch.Generator().manual_seed(6)
    kc, vc = (_rand((8, page, H, D), dt, cuda, g) for _ in range(2))
    table = torch.tensor([[3, 1, 6], [0, 7, 2]], dtype=torch.int32, device=cuda)
    q = _rand((B, 50, 4, D), dt, cuda, g)
    k, v = (_rand((B, 50, H, D), dt, cuda, g) for _ in range(2))
    lens = 200 if seqlens == "int" else torch.tensor([200, 500], dtype=torch.int32, device=cuda)
    torch.cuda.synchronize()
    n0 = core.launch_count
    torch.cuda.set_sync_debug_mode("error")
    try:
        o, lse = patch.flash_attn_with_kvcache(q, kc, vc, k, v, cache_seqlens=lens, block_table=table, causal=True,
                                               num_splits=4, return_softmax_lse=True)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert core.launch_count - n0 == 3  # append, plan, forward
    assert o.shape == q.shape and lse.shape == (B, 4, 50)
    assert bool(torch.isfinite(o).all())


def test_grad_raises_before_any_launch(cuda):
    from svgb200 import core, patch
    from svgb200._lib import SvgbError

    dt = torch.bfloat16
    kc = vc = torch.zeros(1, 256, 2, 64, dtype=dt, device=cuda)
    q = torch.zeros(1, 8, 2, 64, dtype=dt, device=cuda, requires_grad=True)
    n0 = core.launch_count
    with pytest.raises(SvgbError, match="no backward"):
        patch.flash_attn_with_kvcache(q, kc, vc, cache_seqlens=100, causal=True)
    assert core.launch_count == n0
    plan = core.plan_kvcache(100, q_len=8, num_blocks=1, cache_len=256,
                             cache_batch_idx=torch.zeros(1, dtype=torch.int32, device=cuda))
    n0 = core.launch_count
    with pytest.raises(SvgbError, match="KV-cache plan"):
        core.attention(q, kc, vc, plan)
    with pytest.raises(SvgbError, match="KV-cache plan"):
        plan.key_major()
    assert core.launch_count == n0
