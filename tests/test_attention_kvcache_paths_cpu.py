"""Which C entries the KV-cache front end reaches, without a GPU: for every cache format (16-bit, per-head e4m3, per-row
e4m3), uniform or variable-length queries and a single or split plan, the append, planner and forward entries in order
with their key sizes; and the refusal of a uniform plan under grad on 16-bit and per-head caches, before any launch."""
import pytest
import torch

from svgb200 import core
from svgb200._lib import SvgbError

E4M3 = torch.float8_e4m3fn
B, Hq, Hkv, D, NB, ROWS = 2, 4, 2, 128, 3, 512


class _Lib:
    """The C library, recorded: each call's entry name and arguments.  A planner call fills the plan as the real one
    would for what the forward reads (kind, S, BH, max_items, varlen_items)."""

    def __init__(self):
        self.seen = []

    def __getattr__(self, name):
        def call(*a):
            self.seen.append((name, a))
            if name.startswith("svgb_attn_plan_kvcache") and not name.endswith("_bytes"):
                _fill(name, a)
            return 0
        return call


def _fill(name, a):
    d = next(x for x in a if type(x).__name__ == "CArgObject")._obj
    if name == "svgb_attn_plan_kvcache_varlen":
        nb, rows, n = a[8], a[9], a[17]
        items = min(a[5] * -(-a[7] // 256), (a[6] + 255 * a[5]) // 256)
        d.S, d.varlen_items = a[6], items
    else:
        nb, rows = a[6], a[7]
        n = a[12] if name == "svgb_attn_plan_kvcache_split" else 1
        items = a[3] * -(-a[4] // 256)
        d.S = a[3] * a[4]
    d.kind = core.PLAN_KVCACHE if n == 1 else core.PLAN_KVCACHE_SPLIT
    d.BH, d.max_items = nb * rows, n * items


@pytest.fixture
def rec(monkeypatch):
    lib_ = _Lib()
    monkeypatch.setattr(core, "lib", lambda: lib_)
    monkeypatch.setattr(core, "_need_cuda", lambda *ts: None)
    monkeypatch.setattr(core, "_stream", lambda t: 0)
    monkeypatch.setattr(core, "_cu_seqlens", lambda who, name, cu, B_, dev: cu)
    monkeypatch.setattr(core.torch.cuda, "current_stream", lambda d: type("S", (), {"cuda_stream": 0})())
    return lib_.seen


def _cache(fmt):
    dt = {"bf16": torch.bfloat16, "head": E4M3, "row": E4M3}[fmt]
    kc, vc = (torch.zeros(NB, ROWS, Hkv, D, dtype=dt) for _ in range(2))
    scales = {"bf16": {}, "head": dict(k_scale=torch.ones(Hkv), v_scale=torch.ones(Hkv)),
              "row": dict(k_scale=torch.ones(NB, Hkv, ROWS), v_scale=torch.ones(NB, Hkv, ROWS))}[fmt]
    return kc, vc, scales


APPEND = {"bf16": "svgb_kvcache_append", "head": "svgb_kvcache_append_e4m3", "row": "svgb_kvcache_append_e4m3_rows"}
QUANT = {"bf16": [], "head": ["svgb_quantize_e4m3"], "row": ["svgb_quantize_e4m3_rows"]}
SINGLE = {"bf16": "svgb_attn_fwd_strided", "head": "svgb_attn_fwd_strided_e4m3",
          "row": "svgb_attn_fwd_kvcache_e4m3_rows"}


@pytest.mark.parametrize("n", [1, 3])
@pytest.mark.parametrize("varlen", [False, True])
@pytest.mark.parametrize("fmt", ["bf16", "head", "row"])
def test_entries_and_sizes(rec, fmt, varlen, n):
    kc, vc, scales = _cache(fmt)
    lens = torch.tensor([100, 300], dtype=torch.int32)
    bi = torch.tensor([2, 0], dtype=torch.int32)
    if varlen:  # streams of 3 and 4 queries, 1 and 3 appended rows
        cu_q, cu_new = torch.tensor([0, 3, 7], dtype=torch.int32), torch.tensor([0, 1, 4], dtype=torch.int32)
        q, k = torch.randn(7, Hq, D).bfloat16(), torch.randn(4, Hkv, D).bfloat16()
        core.kvcache_append(kc, vc, k, k, lens, cache_batch_idx=bi, cu_seqlens=cu_new, **scales)
        plan = core.plan_kvcache(lens, cu_seqlens_q=cu_q, total_q=7, max_seqlen_q=4, cu_seqlens_new=cu_new,
                                 num_blocks=NB, cache_len=ROWS, cache_batch_idx=bi, causal=True, num_splits=n)
    else:
        q, k = torch.randn(B, 5, Hq, D).bfloat16(), torch.randn(B, 3, Hkv, D).bfloat16()
        core.kvcache_append(kc, vc, k, k, lens, cache_batch_idx=bi, **scales)
        plan = core.plan_kvcache(lens, q_len=5, new_len=3, num_blocks=NB, cache_len=ROWS, cache_batch_idx=bi,
                                 causal=True, num_splits=n)
    o, lse = core.attn_fwd(q, kc, vc, plan, return_lse=True, **scales)
    R = q.shape[0] if varlen else B * 5
    planner = "svgb_attn_plan_kvcache" + ("_varlen" if varlen else "_split" if n > 1 else "")
    fwd = ["svgb_attn_fwd_kvcache_split_bytes", "svgb_attn_fwd_kvcache_split"] if n > 1 else [SINGLE[fmt]]
    want = ["svgb_kvcache_append_varlen" if varlen else APPEND[fmt], planner + "_bytes", planner] + QUANT[fmt] + fwd
    assert [name for name, _ in rec] == want
    args = dict(rec)
    # the append: B streams of 3 new rows, or 4 packed rows and the varlen entry's per-row flag
    a = args[want[0]]
    if varlen:
        assert a[8:16] == (0, B, 4, Hkv, D, NB, ROWS, 0) and a[-2] == (1 if fmt == "row" else 0)
    else:
        assert a[7:15] == (0, B, 3, Hkv, D, NB, ROWS, 0)
    # the planner: B streams, the query rows (and their longest stream), the cache, the split count
    p = args[planner]
    if varlen:
        assert p[5:11] == (B, 7, 4, NB, ROWS, 0) and p[17] == n
    else:
        assert p[3:9] == (B, 5, 3, NB, ROWS, 0) and (n == 1 or p[12] == n)
    # the forward: R packed query rows against NB * ROWS cache rows
    f = args[fwd[-1]]
    if n > 1:
        row_flag, dt = (1 if fmt == "row" else 0), (0 if fmt == "bf16" else 2)
        assert f[8:17] == (dt, row_flag, 1 if varlen else B, Hq, Hkv, R if varlen else 5, NB, ROWS, D)
        assert args["svgb_attn_fwd_kvcache_split_bytes"][:4] == (n, R, Hq, D)
    elif fmt == "bf16":
        assert f[5:12] == (0, 1, Hq, Hkv, R, NB * ROWS, D)
    elif fmt == "head":
        assert f[8:14] == (1, Hq, Hkv, R, NB * ROWS, D)
    else:
        assert f[8:14] == (Hq, Hkv, R, NB, ROWS, D)
    assert o.shape == q.shape and o.dtype == torch.bfloat16
    assert lse.shape == ((Hq, 7) if varlen else (B, Hq, 5))


@pytest.mark.parametrize("fmt", ["bf16", "head"])
def test_uniform_plan_under_grad_refused_before_any_launch(rec, fmt):
    """attention into a KV cache has no backward: a uniform plan on a 16-bit or a per-head e4m3 cache refuses q that
    requires grad, as the variable-length and per-row forms do, instead of returning a detached o."""
    kc, vc, scales = _cache(fmt)
    plan = core.plan_kvcache(torch.tensor([100, 300], dtype=torch.int32), q_len=5, num_blocks=NB, cache_len=ROWS,
                             causal=True)
    rec.clear()
    n0 = core.launch_count
    q = torch.zeros(B, 5, Hq, D, dtype=torch.bfloat16, requires_grad=True)
    with pytest.raises(SvgbError, match="attention into a KV cache has no backward"):
        core.attn_fwd(q, kc, vc, plan, **scales)
    assert rec == [] and core.launch_count == n0
