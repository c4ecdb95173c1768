"""The FP8 (e4m3) KV cache without a GPU: the refusals of svgb_attn_fwd_strided_e4m3 and svgb_kvcache_append_e4m3, each
naming its reason, and the argument mapping and refusals of core.kvcache_append, core.attn_fwd under a KV-cache plan and
flash_attn_with_kvcache, including that calls without scales reach exactly the 16-bit entries."""
import ctypes as C

import pytest
import torch

from test_attention_kvcache_cpu import _T, _kv_plan, dropin  # noqa: F401  (dropin: the drop-in's recording fixture)
from test_attention_local_cpu import PTR, lib  # noqa: F401  (lib: the module-scoped library fixture)

E4M3 = torch.float8_e4m3fn


# --------------------------------------------------------------------------------------------
# C ABI refusals
# --------------------------------------------------------------------------------------------
def _plan(kind):
    p = _kv_plan(Sq=100, rows=200)
    p.kind = kind
    return p


def _fwd8(lib, *, D=128, scales=(PTR, PTR, PTR), plan=None, st=(16 * 200 * 128, 200 * 128, 128), Hq=4, Hkv=2):
    plan = plan or _plan(7)
    s = (C.c_longlong * 3)(*st)
    o = (C.c_longlong * 3)(8 * 200 * 128, 200 * 128, 128)
    return lib.svgb_attn_fwd_strided_e4m3(PTR, PTR, PTR, *scales, PTR, None, 1, Hq, Hkv, 200, 200, D, s, s, s, o, 0.1,
                                          C.byref(plan), PTR, None)


@pytest.mark.parametrize("kw,needle", [
    (dict(D=64), b"head_dim 128 (got 64)"),
    (dict(scales=(PTR, None, PTR)), b"needs the three scale vectors"),
    (dict(scales=(None, PTR, PTR)), b"needs the three scale vectors"),
    (dict(plan=_plan(5)), b"segment plans"),
    (dict(plan=_plan(3)), b"gather plans"),
    (dict(plan=_plan(4)), b"variable-block, band or KV-cache plans"),
    (dict(st=(16 * 200 * 128, 200 * 128, 136)), b"multiple of 16 bytes"),
    (dict(st=(16 * 200 * 128, 200 * 128 + 8, 128)), b"multiple of 16 bytes"),
    (dict(Hq=3), b"multiple of the key/value heads"),
])
def test_strided_e4m3_refusals(lib, kw, needle):
    assert _fwd8(lib, **kw) < 0, kw
    assert needle in lib.svgb_last_error(), (kw, lib.svgb_last_error())


def test_strided_e4m3_reaches_the_plan_check(lib):
    """A well-formed call goes past every refusal above to the plan's length check (the plan was built for 200 rows)."""
    plan = _plan(7)
    plan.S = 300
    assert _fwd8(lib, plan=plan) < 0
    assert b"plan was built for" in lib.svgb_last_error()


def _append8(lib, *, dtype=0, D=128, scales=(PTR, PTR), st=(16, 16, 16), table=None, rows=512, max_pages=0):
    s8 = (C.c_longlong * 3)(*st)
    s = (C.c_longlong * 3)(8, 8, 8)
    return lib.svgb_kvcache_append_e4m3(PTR, PTR, PTR, PTR, PTR, None, table, dtype, 2, 4, 2, D, 4, rows, max_pages,
                                        s8, s8, s, s, *scales, None)


@pytest.mark.parametrize("kw,needle", [
    (dict(scales=(PTR, None)), b"needs both scale vectors"), (dict(scales=(None, PTR)), b"needs both scale vectors"),
    (dict(dtype=2), b"bf16 or fp16 new rows"), (dict(D=96), b"head_dim 96"),
    (dict(st=(16, 16, 8)), b"multiple of 16 bytes"), (dict(st=(24, 16, 16)), b"multiple of 16 bytes"),
    (dict(table=PTR, rows=200, max_pages=2), b"multiple of 128"),
])
def test_append_e4m3_refusals(lib, kw, needle):
    assert _append8(lib, **kw) < 0, kw
    assert needle in lib.svgb_last_error(), (kw, lib.svgb_last_error())


def test_svgb_attn_fwd_still_refuses_e4m3_on_a_kvcache_plan(lib):
    """The flat entry's scales are by query head: it names the strided e4m3 entry instead."""
    plan = _plan(7)
    assert lib.svgb_attn_fwd(PTR, PTR, PTR, PTR, PTR, PTR, PTR, None, None, None, None, 2, 2, 200, 128, 128, 200 * 128,
                             128, 200 * 128, 0.1, C.byref(plan), PTR, None) < 0
    assert b"svgb_attn_fwd_strided_e4m3" in lib.svgb_last_error()


# --------------------------------------------------------------------------------------------
# Python: core refusals before any device work
# --------------------------------------------------------------------------------------------
class _Plan:
    """A KV-cache plan stand-in: B = 2 streams of Sq = 5 queries into 2 x 512 cache rows."""
    source = (2, 5)
    S_kv = 1024
    desc = type("D", (), {"kind": 7})()


def _kv(dtype=E4M3, D=128, H=2):
    return torch.zeros(2, 512, H, D, dtype=dtype), torch.zeros(2, 512, H, D, dtype=dtype)


@pytest.mark.parametrize("kw,needle", [
    (dict(q=torch.zeros(2, 5, 4, 128, dtype=torch.float16)), "bf16 q"),
    (dict(q=torch.zeros(2, 5, 4, 64, dtype=torch.bfloat16), cache=_kv(D=64)), "head_dim 128"),
    (dict(k_scale=None), "needs k_scale and v_scale"),
    (dict(k_scale=torch.ones(2, 2)), r"k_scale must be a float32 tensor \[Hkv=2\]"),
    (dict(v_scale=torch.ones(2, dtype=torch.float64)), "v_scale must be a float32"),
    (dict(out=torch.zeros(2, 5, 4, 128, dtype=torch.float16)), "dtype bf16"),
    (dict(q=torch.zeros(2, 5, 3, 128, dtype=torch.bfloat16)), "multiple of the cache's 2"),
])
def test_attn_fwd_fp8_cache_refusals(kw, needle):
    from svgb200 import core
    from svgb200._lib import SvgbError

    q = kw.get("q", torch.zeros(2, 5, 4, 128, dtype=torch.bfloat16))
    kc, vc = kw.get("cache", _kv())
    ks = kw.get("k_scale", torch.ones(2)) if "k_scale" in kw else torch.ones(2)
    vs = kw.get("v_scale", torch.ones(2))
    with pytest.raises(SvgbError, match=needle):
        core._attn_kvcache(q, kc, vc, _Plan(), False, None, kw.get("out"), ks, vs)


def test_attn_fwd_16bit_cache_refuses_scales():
    from svgb200 import core
    from svgb200._lib import SvgbError

    kc, vc = _kv(torch.bfloat16)
    with pytest.raises(SvgbError, match="takes none"):
        core._attn_kvcache(torch.zeros(2, 5, 4, 128, dtype=torch.bfloat16), kc, vc, _Plan(), False, None, None,
                           torch.ones(2), torch.ones(2))


def test_attn_fwd_scales_need_a_kvcache_plan(monkeypatch):
    from svgb200 import core
    from svgb200._lib import SvgbError

    monkeypatch.setattr(core, "_need_cuda", lambda *ts: None)
    plan = type("P", (), {"desc": type("D", (), {"kind": 2})()})()
    t = torch.zeros(1, 2, 128, 128, dtype=torch.bfloat16)
    with pytest.raises(SvgbError, match="attn_fwd_fp8"):
        core.attn_fwd(t, t, t, plan, k_scale=torch.ones(2), v_scale=torch.ones(2))


@pytest.mark.parametrize("kw,needle", [
    (dict(k_scale=torch.ones(2)), "are for float8_e4m3fn caches"),
])
def test_append_16bit_cache_refuses_scales(monkeypatch, kw, needle):
    from svgb200 import core
    from svgb200._lib import SvgbError

    monkeypatch.setattr(core, "_need_cuda", lambda *ts: None)
    kc, vc = _kv(torch.bfloat16)
    k = torch.zeros(2, 4, 2, 128, dtype=torch.bfloat16)
    with pytest.raises(SvgbError, match=needle):
        core.kvcache_append(kc, vc, k, k, 0, **kw)


@pytest.mark.parametrize("kw,needle", [
    (dict(), "needs k_scale and v_scale"), (dict(k_scale=torch.ones(2)), "needs k_scale and v_scale"),
    (dict(k_scale=torch.ones(3), v_scale=torch.ones(2)), r"\[Hkv=2\]"),
])
def test_append_e4m3_cache_needs_scales(monkeypatch, kw, needle):
    from svgb200 import core
    from svgb200._lib import SvgbError

    monkeypatch.setattr(core, "_need_cuda", lambda *ts: None)
    kc, vc = _kv()
    k = torch.zeros(2, 4, 2, 128, dtype=torch.bfloat16)
    with pytest.raises(SvgbError, match=needle):
        core.kvcache_append(kc, vc, k, k, 0, **kw)


# --------------------------------------------------------------------------------------------
# Python: the drop-in's mapping and refusals
# --------------------------------------------------------------------------------------------
class _T8(_T):
    """A shape-only stand-in for an e4m3 tensor."""
    dtype = E4M3


def test_dropin_fp8_mapping(dropin):
    patch, calls = dropin
    q, kc, vc, k, v = _T(2, 5, 8, 128), _T8(3, 1000, 2, 128), _T8(3, 1000, 2, 128), _T(2, 5, 2, 128), _T(2, 5, 2, 128)
    ks, vs = torch.ones(2), torch.full((2,), 0.5)
    assert patch.flash_attn_with_kvcache(q, kc, vc, k, v, cache_seqlens=7, causal=True, return_softmax_lse=True,
                                         k_descale=ks, v_descale=vs) == "out"
    ap, pp, fp = calls
    assert ap[0] == "append" and ap[1] == (kc, vc, k, v, ("lens", 7, 2))
    assert ap[2] == dict(block_table=None, cache_batch_idx=None, k_scale=ks, v_scale=vs)
    assert pp[0] == "plan" and pp[2]["new_len"] == 5 and pp[2]["cache_len"] == 1000
    assert fp[1] == (q, kc, vc, "plan") and fp[2] == dict(return_lse=True, sm_scale=None, k_scale=ks, v_scale=vs)


def test_dropin_without_scales_reaches_the_16bit_calls(dropin):
    """No keyword: exactly the 16-bit calls and keywords."""
    patch, calls = dropin
    q, kc, vc, k, v = _T(2, 5, 8, 128), _T(3, 1000, 2, 128), _T(3, 1000, 2, 128), _T(2, 5, 2, 128), _T(2, 5, 2, 128)
    patch.flash_attn_with_kvcache(q, kc, vc, k, v, cache_seqlens=7, causal=True)
    ap, pp, fp = calls
    assert ap[2] == dict(block_table=None, cache_batch_idx=None)
    assert fp[2] == dict(return_lse=False, sm_scale=None)


def test_core_without_scales_reaches_the_16bit_entries(monkeypatch):
    """core.kvcache_append and the KV-cache forward on 16-bit caches call svgb_kvcache_append and svgb_attn_fwd_strided,
    never the e4m3 entries."""
    from svgb200 import core

    seen = []

    class _Lib:
        def __getattr__(self, name):
            return lambda *a: seen.append(name) or 0

    monkeypatch.setattr(core, "lib", lambda: _Lib())
    monkeypatch.setattr(core, "_need_cuda", lambda *ts: None)
    monkeypatch.setattr(core, "_stream", lambda t: 0)
    monkeypatch.setattr(core, "_seqlens", lambda s, B, dev: torch.zeros(B, dtype=torch.int32))
    kc, vc = _kv(torch.bfloat16)
    k = torch.zeros(2, 4, 2, 128, dtype=torch.bfloat16)
    core.kvcache_append(kc, vc, k, k, 0)
    plan = _Plan()
    plan.ws = torch.zeros(16, dtype=torch.uint8)
    plan.desc = core.Plan()
    plan.desc.kind = core.PLAN_KVCACHE
    core._attn_kvcache(torch.zeros(2, 5, 4, 128, dtype=torch.bfloat16), kc, vc, plan, False, None, None)
    assert seen == ["svgb_kvcache_append", "svgb_attn_fwd_strided"]


@pytest.mark.parametrize("kw,needle", [
    (dict(q_descale=torch.ones(2)), "q_descale is not supported"),
    (dict(k_descale=torch.ones(2, 2), v_descale=torch.ones(2)), r"k_descale must be \[Hkv\].*\[B, Hkv\]"),
    (dict(k_descale=torch.ones(2)), "go together"),
    (dict(), "go together"),
    (dict(q=torch.zeros(2, 5, 8, 128, dtype=E4M3)), "q is torch.float8_e4m3fn"),
    (dict(k=torch.zeros(2, 5, 2, 128, dtype=E4M3), v=torch.zeros(2, 5, 2, 128, dtype=E4M3)), "k is torch.float8"),
])
def test_dropin_fp8_refusals(dropin, kw, needle):
    from svgb200._lib import SvgbError

    patch, calls = dropin
    q = kw.pop("q", _T(2, 5, 8, 128))
    scales = {} if any(n in kw for n in ("k_descale", "q_descale")) or not kw else dict(k_descale=torch.ones(2),
                                                                                        v_descale=torch.ones(2))
    with pytest.raises(SvgbError, match=needle):
        patch.flash_attn_with_kvcache(q, _T8(2, 512, 2, 128), _T8(2, 512, 2, 128), **scales, **kw)
    assert calls == []


def test_dropin_16bit_cache_refuses_descales(dropin):
    from svgb200._lib import SvgbError

    patch, calls = dropin
    with pytest.raises(SvgbError, match="go together"):
        patch.flash_attn_with_kvcache(_T(2, 5, 8, 128), _T(2, 512, 2, 128), _T(2, 512, 2, 128),
                                      k_descale=torch.ones(2), v_descale=torch.ones(2))
    assert calls == []


def test_e4m3_strides_fill_extent_one_dimensions_with_16():
    """A one-KV-head e4m3 cache view whose (never stepped) head stride is odd: the e4m3 calls pass 16 bytes there,
    which their 16-byte stride check takes, where the 16-bit calls pass 8 elements."""
    from svgb200 import core

    base = torch.zeros(2 * 512 * 128 + 7, dtype=torch.uint8)
    cache = base.as_strided((2, 512, 1, 128), (512 * 128, 128, 7, 1))
    rows = base.as_strided((1024, 1, 128), (128, 7, 1))  # the cache as rows [1024, 1, 128], as the forward reads it
    assert core._strides(rows, "shd", 16) == (16, 16, 128)
    assert core._strides(rows, "shd") == (8, 8, 128)
    assert core._strides(cache.transpose(1, 2), "bhsd", 16) == (512 * 128, 16, 128)
    assert tuple(core._st(rows, "shd", 16)) == (16, 16, 128)
