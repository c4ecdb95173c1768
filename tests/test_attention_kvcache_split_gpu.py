"""Split KV-cache attention (plan_kvcache(num_splits=), svgb_attn_fwd_kvcache_split) on the GPU: the split lists read back
from the plan against the single plan's, one live split bit for bit the single pass in all three cache formats, fp64
references with NaN-filled outputs and partials, determinism, the launches without host synchronisation, and the
production shapes under the automatic split count."""
import ctypes as C

import pytest
import torch

from test_attention_kvcache_fp8_gpu import FP8_LSE, FP8_TOL, _cache8, _paged8
from test_attention_kvcache_fp8_rows_gpu import _cache as _cache_rows
from test_attention_kvcache_gpu import _eq, _paged_from, _rand, _ref64

pytestmark = pytest.mark.gpu

DT = {"bf16": torch.bfloat16, "fp16": torch.float16}


def _plan(lens, Sq, kc, n, *, table=None, **win):
    from svgb200 import core

    paged = table is not None
    return core.plan_kvcache(lens, q_len=Sq, num_blocks=kc.shape[0], cache_len=None if paged else kc.shape[1],
                             block_table=table, page_size=kc.shape[1] if paged else None, num_splits=n, **win)


def _nan_partials(plan, q, n):
    """fill the workspace the split forward will use with NaN bytes"""
    from svgb200 import core
    from svgb200._lib import lib

    B, Sq, Hq, D = q.shape
    nbytes = C.c_size_t()
    assert lib().svgb_attn_fwd_kvcache_split_bytes(n, B * Sq, Hq, D, C.byref(nbytes)) == 0
    core.workspace("kvcache_split", nbytes.value, q.device).fill_(255)


def _fwd(q, kc, vc, plan, n=None, **kw):
    from svgb200 import core

    if n is not None:
        _nan_partials(plan, q, n)
    out = torch.full(q.shape, float("nan"), dtype=torch.bfloat16 if kc.dtype == torch.float8_e4m3fn else q.dtype,
                     device=q.device)
    return core.attn_fwd(q, kc, vc, plan, return_lse=True, out=out, **kw)


def _lists(plan):
    """per item of the plan: (first row, rows, [(row, meta)]) read back from its workspace"""
    ws = plan.ws.cpu()
    count = ws.view(torch.int32)[0].item()
    it = ws[plan.desc.items_off:].view(torch.int32)
    ch = ws[plan.desc.chunks_off:].view(torch.int32)
    out = []
    for i in range(count):
        d = it[8 * i:8 * i + 8].tolist()
        chunks = [tuple(ch[2 * (d[2] + c):2 * (d[2] + c) + 2].tolist()) for c in range(d[3])]
        assert d[6:8] == d[2:4]  # both streams walk one list
        out.append((d[0], d[1] + d[5], chunks))
    return out


@pytest.mark.parametrize("paged", [False, True])
@pytest.mark.parametrize("win", [dict(causal=True), dict(causal=True, window_size=(700, 0), sink=300),
                                 dict(window_size=(255, 130), sink=129)])
def test_split_lists_concatenate_to_the_single_list(cuda, paged, win):
    Ls, Sq, page = [2900, 0, 1300, 77], 300, 256
    g = torch.Generator().manual_seed(3)
    kc = _rand((len(Ls), 3072, 1, 64), torch.bfloat16, cuda, g)
    table = None
    if paged:
        kc, table = _paged_from(kc, Ls, page, 5, g, cuda)
    lens = torch.tensor(Ls, dtype=torch.int32, device=cuda)
    single = _lists(_plan(lens, Sq, kc, 1, table=table, **win))
    longest = max(len(c) for _, _, c in single)
    for n in (2, 3, 5, longest + 3):
        split = _lists(_plan(lens, Sq, kc, n, table=table, **win))
        assert len(split) == n * len(single)
        for i, (r0, nr, chunks) in enumerate(single):
            parts = [split[s * len(single) + i] for s in range(n)]
            assert all(p[:2] == (r0, nr) for p in parts), (n, i)
            assert [c for p in parts for c in p[2]] == chunks, (n, i)


def _formats(q, kc_bf, g, cuda):
    """The same keys as a bf16 cache, a per-head e4m3 cache and a per-row e4m3 cache: [(k, v, scale kwargs)]"""
    shape = kc_bf.shape
    vc_bf = _rand(shape, torch.bfloat16, cuda, g)
    k8, ks, _ = _cache8(shape, cuda, g)
    v8, vs, _ = _cache8(shape, cuda, g)
    kr, ksr, _, _ = _cache_rows(shape, cuda, g)
    vr, vsr, _, _ = _cache_rows(shape, cuda, g)
    return {"bf16": (kc_bf, vc_bf, {}), "e4m3": (k8, v8, dict(k_scale=ks, v_scale=vs)),
            "e4m3 rows": (kr, vr, dict(k_scale=ksr, v_scale=vsr))}


@pytest.mark.parametrize("Sq", [1, 50])
def test_one_live_split_is_the_single_pass_bit_for_bit(cuda, Sq):
    """Every stream holds at most 128 keys, so each item visits one chunk and split 0 gets it: the merge multiplies by
    w = 1 and adds log 1, and o and lse are the single pass's bits, in every cache format."""
    Ls, Hq, Hkv, D = [100, 128, 5, 0], 8, 2, 128
    g = torch.Generator().manual_seed(11)
    q = _rand((len(Ls), Sq, Hq, D), torch.bfloat16, cuda, g)
    kc = _rand((len(Ls), 256, Hkv, D), torch.bfloat16, cuda, g)
    lens = torch.tensor(Ls, dtype=torch.int32, device=cuda)
    for name, (k, v, kw) in _formats(q, kc, g, cuda).items():
        o1, l1 = _fwd(q, k, v, _plan(lens, Sq, k, 1, causal=True), **kw)
        for n in (2, 4):
            on, ln = _fwd(q, k, v, _plan(lens, Sq, k, n, causal=True), n, **kw)
            _eq("o", on, o1, f"{name} n={n} Sq={Sq}")
            _eq("lse", ln, l1, f"{name} n={n} Sq={Sq}")
        assert bool((l1[3] == float("-inf")).all()) and bool((o1[3] == 0).all())  # the stream without keys


# (n, Sq): every n at every Sq; dtype / D / G / paged cycle over the cases so that each value meets several n and Sq
FP64 = [(n, Sq) for n in (2, 3, 4, 7, 32) for Sq in (1, 50, 256, 300)]


@pytest.mark.parametrize("case", range(len(FP64)))
def test_fp64_reference(cuda, case):
    n, Sq = FP64[case]
    dtype, D = [("bf16", 128), ("fp16", 64), ("bf16", 64), ("fp16", 128)][case % 4]
    G = (1, 4)[(case // 2) % 2]
    paged = case % 3 != 0
    Ls, Hkv = [2100, 0, 700, 3000], 2
    win = dict(causal=True, window_size=(1500, 0), sink=130) if case % 2 else dict(causal=True)
    left = win.get("window_size", (10 ** 9, 0))[0]
    g = torch.Generator().manual_seed(100 + case)
    dt = DT[dtype]
    q = _rand((len(Ls), Sq, G * Hkv, D), dt, cuda, g)
    kc, vc = (_rand((len(Ls), 3072, Hkv, D), dt, cuda, g) for _ in range(2))
    ks, vs = [kc[b, :L] for b, L in enumerate(Ls)], [vc[b, :L] for b, L in enumerate(Ls)]
    table = None
    if paged:
        g2 = torch.Generator().manual_seed(case)
        kc, table = _paged_from(kc, Ls, 256, 3, g2, cuda)
        g2 = torch.Generator().manual_seed(case)
        vc, _ = _paged_from(vc, Ls, 256, 3, g2, cuda)
    lens = torch.tensor(Ls, dtype=torch.int32, device=cuda)
    plan = _plan(lens, Sq, kc, n, table=table, **win)
    o, lse = _fwd(q, kc, vc, plan, n)
    eo, el = _ref64(q, ks, vs, Ls, win.get("sink", 0), left, 0)
    fin = torch.isfinite(el)
    assert torch.equal(fin, torch.isfinite(lse)), FP64[case]
    assert bool((lse[~fin] == float("-inf")).all())
    assert torch.allclose(o.double(), eo, atol=2e-2, rtol=2e-2), FP64[case]
    assert torch.allclose(lse.double()[fin], el[fin], atol=1e-3, rtol=1e-3), FP64[case]
    assert bool((o[~fin.transpose(1, 2)] == 0).all())  # rows without keys: o = 0
    o2, l2 = _fwd(q, kc, vc, plan, n)
    _eq("o", o2, o, "determinism")
    _eq("lse", l2, lse, "determinism")


@pytest.mark.parametrize("fmt", ["e4m3", "e4m3 rows"])
@pytest.mark.parametrize("n", [2, 3, 4, 7, 32])
def test_fp8_against_the_single_pass(cuda, fmt, n):
    """Per-head and per-row e4m3 caches, paged, G = 4, D = 128: split against the single-pass e4m3 result."""
    Ls, Sq, Hkv, D = [2100, 0, 3000], 300, 2, 128
    g = torch.Generator().manual_seed(200 + n)
    q = _rand((len(Ls), Sq, 4 * Hkv, D), torch.bfloat16, cuda, g)
    k, v, kw = _formats(q, _rand((len(Ls), 3072, Hkv, D), torch.bfloat16, cuda, g), g, cuda)[fmt]
    if fmt == "e4m3":
        g2 = torch.Generator().manual_seed(n)
        k, table = _paged8(k, 256, 2, g2)
        g2 = torch.Generator().manual_seed(n)
        v, _ = _paged8(v, 256, 2, g2)
    else:
        table = None  # per-row scales sit at the rows' places: the contiguous cache
    lens = torch.tensor(Ls, dtype=torch.int32, device=cuda)
    win = dict(causal=True, window_size=(1200, 0), sink=200)
    o1, l1 = _fwd(q, k, v, _plan(lens, Sq, k, 1, table=table, **win), **kw)
    on, ln = _fwd(q, k, v, _plan(lens, Sq, k, n, table=table, **win), n, **kw)
    assert on.dtype == torch.bfloat16 and bool(torch.isfinite(on).all())
    torch.testing.assert_close(on.double(), o1.double(), **FP8_TOL)
    fin = torch.isfinite(l1)
    assert torch.equal(fin, torch.isfinite(ln))
    torch.testing.assert_close(ln.double()[fin], l1.double()[fin], **FP8_LSE)
    o2, l2 = _fwd(q, k, v, _plan(lens, Sq, k, n, table=table, **win), n, **kw)
    _eq("o", o2, on, "determinism")
    _eq("lse", l2, ln, "determinism")


def test_launches_without_host_sync(cuda):
    """plan, attention, merge: three launches, no host synchronisation."""
    from svgb200 import core

    B, page, H, D = 2, 256, 2, 128
    g = torch.Generator().manual_seed(7)
    kc, vc = (_rand((8, page, H, D), torch.bfloat16, cuda, g) for _ in range(2))
    table = torch.tensor([[3, 1, 6], [0, 7, 2]], dtype=torch.int32, device=cuda)
    q = _rand((B, 1, 4, D), torch.bfloat16, cuda, g)
    lens = torch.tensor([200, 700], dtype=torch.int32, device=cuda)
    core.attn_fwd(q, kc, vc, _plan(lens, 1, kc, 3, table=table, causal=True))  # sizes the cached workspace
    torch.cuda.synchronize()
    n0 = core.launch_count
    torch.cuda.set_sync_debug_mode("error")
    try:
        plan = _plan(lens, 1, kc, 3, table=table, causal=True)
        o, lse = core.attn_fwd(q, kc, vc, plan, return_lse=True)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert core.launch_count - n0 == 3
    assert o.shape == q.shape and lse.shape == (B, 4, 1) and bool(torch.isfinite(o).all())


def _ref64_per_head(q, k, v, L, sink, left):
    """_ref64 one head at a time (bounded memory at production shapes): o [1, Sq, Hq, D], lse [1, Hq, Sq]"""
    G = q.shape[2] // k.shape[1]
    os, ls = [], []
    for h in range(q.shape[2]):
        o, lse = _ref64(q[:, :, h:h + 1], [k[:, h // G:h // G + 1]], [v[:, h // G:h // G + 1]], [L], sink, left, 0)
        os.append(o)
        ls.append(lse)
    return torch.cat(os, 2), torch.cat(ls, 1)


@pytest.mark.parametrize("Sq,H", [(1560, 12), (1, 40)])
def test_production_shapes_automatic(cuda, Sq, H):
    """Wan 1.3B one-frame chunk (1 560 queries, 12 heads) and decode at 40 heads against a 21-frame cache of 256-row
    pages, sink 1 560, 14 040 back, with the automatic split count."""
    from svgb200 import core

    L, page, sink, left, D = 21 * 1560, 256, 1560, 9 * 1560, 128
    g = torch.Generator().manual_seed(Sq + H)
    cap = -(-L // page) * page
    q = _rand((1, Sq, H, D), torch.bfloat16, cuda, g)
    kc, vc = (_rand((1, cap, H, D), torch.bfloat16, cuda, g) for _ in range(2))
    g2 = torch.Generator().manual_seed(1)
    kp, table = _paged_from(kc, [L], page, 4, g2, cuda)
    g2 = torch.Generator().manual_seed(1)
    vp, _ = _paged_from(vc, [L], page, 4, g2, cuda)
    lens = torch.tensor([L], dtype=torch.int32, device=cuda)
    plan = core.plan_kvcache(lens, q_len=Sq, num_blocks=kp.shape[0], block_table=table, page_size=page, causal=True,
                             window_size=(left, 0), sink=sink, num_splits=0, num_heads=H)
    n = plan.desc.max_items // -(-Sq // 256)
    assert n == core.kvcache_num_splits(-(-Sq // 256) * H, 126, core.device_check()[2]) and n > 1
    o, lse = _fwd(q, kp, vp, plan, n)
    eo, el = _ref64_per_head(q, kc[0, :L], vc[0, :L], L, sink, left)
    assert (o.double() - eo).abs().max().item() < 2e-2
    assert (lse.double() - el).abs().max().item() < 1e-3
