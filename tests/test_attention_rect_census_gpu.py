"""Exact censuses of attention where the query and key lengths differ (tests/rect_census_cases.py), on every row of
every head: rectangular variable-block plans, the local and block-causal masks inside packed segments of unequal
totals, the 16-bit KV cache at Sq < L in one pass, and the Wan 480p chunk-against-cache shape.

  forward key census      q = 0, one-hot key-identity V: o = round16(cnt / n) bit for bit, exp(lse) = n
  forward softmax census  integer log2 scores that move the running max (oracle/softmax.py): o bit for bit, lse
                          within log2f's one ulp
  backward key census     every dQ / dK / dV value a count of allowed pairs times a power of two (oracle/bwd_census.py)
  backward gradient census  small integers on real scores, every intermediate exact: dQ, dK, dV bit for bit

Everything is written into NaN-filled out= buffers, so an element no stream stores fails.  The KV cache has no
backward.  Every case runs bf16 and fp16 at D = 64 and 128 (the production shapes run one format), so each forward and
backward instantiation the square censuses run also runs rectangular.  The premises of every case (exactness, budgets,
coverage, and the oracle mutants it catches) are shown on the CPU in tests/test_attention_rect_census_cpu.py."""
import pytest
import torch

import rect_census_cases as rc
from oracle import bwd_census as bc
from oracle import census as oc
from oracle import softmax as sm
from test_attention_census_gpu import bound_ok, check_census
from test_softmax_census_gpu import check as check_softmax

pytestmark = pytest.mark.gpu

DT = {"bf16": torch.bfloat16, "fp16": torch.float16}
NAMES = ("dq", "dk", "dv")
FMTS = [(64, "bf16"), (64, "fp16"), (128, "bf16"), (128, "fp16")]
FMT_IDS = [f"D{d}-{t}" for d, t in FMTS]


# --------------------------------------------------------------------------------------------
# plans and launches
# --------------------------------------------------------------------------------------------
def plan_of(cuda, case):
    """The plan of a packed-segment or variable-block case."""
    from svgb200 import core

    if case.kind == "varblock":
        return core.plan_varblock(case.bm.to(cuda), case.rows.to(cuda), case.cols.to(cuda), case.Sq, S_kv=case.Skv)
    t = lambda c: torch.tensor(c, dtype=torch.int32, device=cuda)  # noqa: E731
    kw = dict(total_q=case.Sq, total_k=case.Skv)
    if case.kind == "local":
        sink, left, right = case.args
        return core.plan_local_varlen(t(case.cu_q), t(case.cu_k), sink=sink, window_size=(left, right), **kw)
    sink, C_, F, W = case.args
    return core.plan_local_varlen(t(case.cu_q), t(case.cu_k), block=C_, first_block=F, window_size=(W, -1), sink=sink,
                                  **kw)


def fwd(cuda, case, q, k, v, dtype, sm_scale=None):
    """o [H, Sq, D], lse [H, Sq] of q [H, Sq, D] against k, v [H, Skv, D] (float32 values exact in dtype), into a
    NaN-filled out= buffer: through the segment / variable-block plan, or through a KV cache (contiguous or paged,
    the keys in logical order, every other cache row finite noise) under a single-pass plan."""
    from svgb200 import core

    H, Sq, D = q.shape
    kw = dict(return_lse=True, sm_scale=sm_scale)
    if case.kind != "kvcache":
        qd, kd, vd = (t.to(dtype)[None].to(cuda) for t in (q, k, v))
        o, lse = core.attn_fwd(qd, kd, vd, plan_of(cuda, case), out=torch.full_like(qd, float("nan")), **kw)
        return o[0].cpu(), lse.cpu()
    kv, L = case.kv, case.Skv
    g = torch.Generator().manual_seed(L)
    page = kv["page"]
    if page:
        npg = -(-L // page)
        ids = torch.randperm(npg + 3, generator=g)
        table = ids[:npg].view(1, npg).int()
        caches = []
        for x in (k, v):
            pool = torch.randn(npg + 3, page, H, D, generator=g)
            for i in range(npg):
                rows = x[:, i * page:(i + 1) * page].transpose(0, 1)
                pool[int(ids[i]), :rows.shape[0]] = rows
            caches.append(pool.to(dtype).to(cuda))
        geo = dict(num_blocks=npg + 3, block_table=table.to(cuda), page_size=page)
    else:
        cap = L + 77
        caches = []
        for x in (k, v):
            c = torch.randn(1, cap, H, D, generator=g)
            c[0, :L] = x.transpose(0, 1)
            caches.append(c.to(dtype).to(cuda))
        geo = dict(num_blocks=1, cache_len=cap)
    if kv["mask"] == "block":
        mk = dict(block=kv["C"], first_block=kv["F"], window_size=(kv["W"], -1))
    elif kv["mask"] == "causal":
        mk = dict(causal=True)
    else:
        mk = dict(window_size=(kv["left"], 0))
    plan = core.plan_kvcache(torch.tensor([L], dtype=torch.int32, device=cuda), q_len=Sq, sink=kv["sink"],
                             num_splits=1, **geo, **mk)
    qd = q.transpose(0, 1)[None].to(dtype).to(cuda)
    o, lse = core.attn_fwd(qd, *caches, plan, out=torch.full_like(qd, float("nan")), **kw)
    return o[0].transpose(0, 1).cpu(), lse[0].cpu()


def bwd(cuda, case, tensors, lse, dtype, sm_scale):
    """dq [H, Sq, D], dk, dv [H, Skv, D] of attn_bwd into NaN-filled out= buffers; tensors q, k, v, o, do [H, ., D]."""
    from svgb200 import core

    q, k, v, o, do = (t.to(dtype)[None].to(cuda) for t in tensors)
    out = (torch.full_like(q, float("nan")), torch.full_like(k, float("nan")), torch.full_like(v, float("nan")))
    got = core.attn_bwd(q, k, v, o, do, lse.to(cuda), plan_of(cuda, case), sm_scale=sm_scale, out=out)
    assert all(a is b for a, b in zip(got, out))
    return [x[0].cpu() for x in got]


def first_bad(got, exp):
    """(row, column, rows differing) of the first element where got != exp by value (NaN never matches), or None"""
    bad = ~(got.float() == exp.float())
    if not bool(bad.any()):
        return None
    r, c = (int(x) for x in bad.nonzero()[0])
    return r, c, int(bad.any(1).sum())


def report(what, name, h, b, exp, got):
    r, c, nr = b
    raise AssertionError(f"{what}: {name} first differs at (head {h}, row {r}, column {c}) of {nr} rows: expected "
                         f"{float(exp[r, c])!r}, kernel {float(got[r, c])!r}")


# --------------------------------------------------------------------------------------------
# the four censuses
# --------------------------------------------------------------------------------------------
def key_census_fwd(cuda, case, D, dtype, what):
    tabs = [oc.band_census(case.mod(h), case.Sq, D, cuda, Skv=case.Skv) for h in range(case.H)]
    tabs = [(c.cpu(), n.cpu()) for c, n in tabs]
    bound_ok([c for c, _ in tabs], dtype)
    q = torch.zeros(case.H, case.Sq, D)
    k = torch.randn(case.H, case.Skv, D, generator=torch.Generator().manual_seed(D))
    for enc in oc.ENCODINGS:
        v = oc.identity_values(case.Skv, D, enc, case.H, torch.float32, "cpu")[0]
        o, lse = fwd(cuda, case, q, k, v, dtype)
        check_census(o, lse, [c for c, _ in tabs], [n for _, n in tabs], enc, what)


def softmax_census(cuda, scase, case, dtype, what):
    q, k, v = scase.tensors()
    o, lse = fwd(cuda, case, q, k, v, dtype, sm_scale=sm.scale_for(1.0))
    check_softmax(cuda, scase, o, lse, what)


def key_census_bwd(cuda, case, D, dtype, what):
    tabs = [bc.band_tables(case.mod(h), case.Sq, D, cuda, Skv=case.Skv) for h in range(case.H)]
    n_rows = torch.stack([t[1] for t in tabs])
    for enc in oc.ENCODINGS:
        q, _, _, o, do, lse = (t[: case.H] for t in bc.key_inputs(case.Sq, D, enc, n_rows))
        _, k, v, _, _, _ = bc.key_inputs(case.Skv, D, enc, torch.ones(case.H, case.Skv, dtype=torch.long))
        got = bwd(cuda, case, (q, k[: case.H], v[: case.H], o, do), lse, dtype, bc.KEY_SCALE)
        for h, (cnt, _, cnt_t) in enumerate(tabs):
            assert int(cnt[enc].max()) <= bc.MAX_COUNT[dtype] and int(cnt_t[enc].max()) <= bc.MAX_COUNT[dtype]
            exp = bc.key_expected(cnt[enc], cnt_t[enc], case.Sq, D, enc, Skv=case.Skv)
            for name, g, e in zip(NAMES, got, exp):
                b = first_bad(g[h], e.to(dtype))
                if b is not None:
                    report(f"{what}, encoding {enc}", name, h, b, e, g[h])


def grad_census(cuda, case, D, dtype, what):
    gc = case.grad_case(D)
    got = bwd(cuda, case, (gc.q, gc.k, gc.v, gc.o, gc.do), gc.lse(), dtype, gc.sm_scale)
    for h in range(gc.H):
        _, budget, stats = bc.grad_exact(gc, h, cuda)
        assert max(budget) < bc.BUDGET and stats["ds_exact"] and stats["ds_max"] <= 8, f"{what}: head {h} not exact"
        for name, g, e in zip(NAMES, got, bc.grad_expected(gc, h, dtype, cuda)):
            b = first_bad(g[h], e.cpu())
            if b is not None:
                report(what, name, h, b, e, g[h])


# --------------------------------------------------------------------------------------------
# tests
# --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", FMTS, ids=FMT_IDS)
@pytest.mark.parametrize("name", [c.name for c in rc.CASES])
def test_forward_census(cuda, name, fmt):
    """The forward key census and the online-softmax census of every case: which keys each row kept, how often, its
    lse, and the chunk loop's wipes and rescales on real scores."""
    D, dt = fmt
    case = rc.BY_NAME[name]
    what = f"{name} ({case.Sq} x {case.Skv}) D={D} {dt}"
    key_census_fwd(cuda, case, D, DT[dt], f"key census {what}")
    softmax_census(cuda, case.softmax_case(D), case, DT[dt], f"softmax census {what}")


@pytest.mark.parametrize("fmt", FMTS, ids=FMT_IDS)
@pytest.mark.parametrize("name", rc.BACKWARD)
def test_backward_census(cuda, name, fmt):
    """The backward key census (both launches count exactly the allowed pairs of every row and key) and the integer
    gradient census of every case with a backward."""
    D, dt = fmt
    case = rc.BY_NAME[name]
    what = f"{name} ({case.Sq} x {case.Skv}) D={D} {dt}"
    key_census_bwd(cuda, case, D, DT[dt], f"bwd key census {what}")
    grad_census(cuda, case, D, DT[dt], f"gradient census {what}")


def test_softmax_census_wan720_text(cuda):
    """Wan 720p text cross-attention, 75 600 queries against 512 keys, one head, dense, bf16, D = 128."""
    case = rc.WAN720_TEXT
    softmax_census(cuda, case.softmax_case(), case, torch.bfloat16, "softmax census Wan 720p text")


def test_wan480_chunk_against_cache(cuda):
    """Wan 480p: one 3-frame chunk (4 680 queries) against 22 frames (34 320 keys) as one block-causal segment with a
    one-frame sink and a 9-frame window: the forward softmax census (bf16) and the backward key census (fp16, where
    every count of 34 320 keys stays exact), D = 128."""
    case = rc.WAN480_CHUNK
    softmax_census(cuda, case.softmax_case(device=cuda), case, torch.bfloat16, "softmax census Wan 480p chunk")
    key_census_bwd(cuda, case, 128, torch.float16, "bwd key census Wan 480p chunk")
