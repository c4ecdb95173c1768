"""The per-row FP8 (e4m3) KV cache without a GPU: the scale rule's exponent built for the host from the device function
(fp8_rows.cuh) against frexp, the ABI refusals of svgb_kvcache_append_e4m3_rows, svgb_attn_fwd_kvcache_e4m3_rows and
svgb_quantize_e4m3_rows, each naming its reason, and core's choice of format from the scale tensors' shape: the
refusals, and that [Hkv] scales or no scales still reach exactly the existing entries."""
import ctypes as C
import math
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest
import torch

from test_attention_kvcache_cpu import _kv_plan
from test_attention_local_cpu import CSRC, PTR, lib  # noqa: F401  (lib: the module-scoped library fixture)

E4M3 = torch.float8_e4m3fn

PROBE = r"""
#include <cstdio>
#include "fp8_rows.cuh"
int main() {
  unsigned b;
  while (std::scanf("%x", &b) == 1) {
    float a;
    memcpy(&a, &b, 4);
    std::printf("%d\n", svgb::e4m3_row_exp(a));
  }
  return 0;
}
"""


@pytest.fixture(scope="module")
def row_exp(tmp_path_factory):
    nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    d = tmp_path_factory.mktemp("fp8_rows_probe")
    (d / "probe.cu").write_text(PROBE)
    subprocess.run([nvcc, "-std=c++17", "-I", str(CSRC), str(d / "probe.cu"), "-o", str(d / "probe")], check=True,
                   capture_output=True)

    def run(values):
        text = "\n".join(f"{struct.unpack('<I', struct.pack('<f', v))[0]:x}" for v in values) + "\n"
        out = subprocess.run([str(d / "probe")], input=text.encode(), capture_output=True, check=True).stdout
        return [int(x) for x in out.split()]

    return run


def _rule(a):
    """The issue's definition: the smallest integer e with a <= 448 * 2^e, clamped to [-126, 127]; a = 0 gives 0."""
    if a == 0:
        return 0
    m, k = math.frexp(a)
    e = k - 9 if m <= 0.875 else k - 8
    return min(max(e, -126), 127)


def test_row_exponent_against_frexp(row_exp):
    f32 = lambda x: float(np.float32(x))  # noqa: E731
    vals = [0.0, 2.0 ** -149, 3 * 2.0 ** -149, 2.0 ** -133, 2.0 ** -126, 2.0 ** -24, 2.0 ** -14, 1023 * 2.0 ** -24,
            float(torch.finfo(torch.bfloat16).max), 65504.0, float(torch.finfo(torch.float32).max), 1.0, 0.875, 0.5]
    for k in range(-140, 128, 7):
        x = 448 * 2.0 ** k
        if x < 3.4e38:
            vals += [f32(x), float(np.nextafter(np.float32(x), np.float32(0))),
                     float(np.nextafter(np.float32(x), np.float32(np.inf)))]
    vals += [f32(v) for v in np.random.default_rng(0).lognormal(0, 20, 200)]
    vals = [v for v in vals if math.isfinite(v)]
    got = row_exp(vals)
    for v, e in zip(vals, got):
        assert e == _rule(v), (v, e, _rule(v))
        if v and -126 < e < 127:  # the smallest: 448 * 2^e covers v and 448 * 2^(e-1) does not
            assert v <= 448 * 2.0 ** e and v > 448 * 2.0 ** (e - 1), v


# --------------------------------------------------------------------------------------------
# C ABI refusals
# --------------------------------------------------------------------------------------------
def _append(lib, *, D=128, scales=(PTR, PTR), rows=512, dtype=0):
    s8 = (C.c_longlong * 3)(16, 16, 16)
    s = (C.c_longlong * 3)(8, 8, 8)
    return lib.svgb_kvcache_append_e4m3_rows(PTR, PTR, PTR, PTR, PTR, None, None, dtype, 2, 4, 2, D, 4, rows, 0, s8,
                                             s8, s, s, *scales, None)


@pytest.mark.parametrize("kw,needle", [
    (dict(scales=(PTR, None)), b"needs both per-row scale tensors"),
    (dict(scales=(None, PTR)), b"needs both per-row scale tensors"),
    (dict(scales=(PTR + 4, PTR)), b"16-byte aligned"),
    (dict(rows=510), b"multiple of 4"),
    (dict(D=64), b"head_dim 128 (got 64)"),
    (dict(dtype=2), b"bf16 or fp16 new rows"),
])
def test_append_rows_refusals(lib, kw, needle):
    assert _append(lib, **kw) < 0, kw
    assert needle in lib.svgb_last_error(), (kw, lib.svgb_last_error())


def _plan(kind):
    p = _kv_plan(Sq=100, rows=200)
    p.kind = kind
    return p


def _fwd(lib, *, D=128, scales=(PTR, PTR, PTR), plan=None, st=(200 * 2 * 128, 128, 2 * 128), rows=200, Hq=4):
    plan = plan or _plan(7)
    s = (C.c_longlong * 3)(*st)
    o = (C.c_longlong * 3)(100 * 4 * 128, 128, 4 * 128)
    return lib.svgb_attn_fwd_kvcache_e4m3_rows(PTR, PTR, PTR, *scales, PTR, None, Hq, 2, 100, 1, rows, D, s, s, s, o,
                                               0.1, C.byref(plan), PTR, None)


@pytest.mark.parametrize("kw,needle", [
    (dict(plan=_plan(1)), b"KV-cache plans (svgb_attn_plan_kvcache) only (kind 1)"),
    (dict(plan=_plan(2)), b"KV-cache plans (svgb_attn_plan_kvcache) only (kind 2)"),
    (dict(plan=_plan(3)), b"KV-cache plans (svgb_attn_plan_kvcache) only (kind 3)"),
    (dict(plan=_plan(5)), b"KV-cache plans (svgb_attn_plan_kvcache) only (kind 5)"),
    (dict(D=64), b"head_dim 128 (got 64)"),
    (dict(scales=(None, PTR, PTR)), b"query row scales q_scale"),
    (dict(scales=(PTR, None, PTR)), b"needs both per-row scale tensors"),
    (dict(scales=(PTR, PTR, None)), b"needs both per-row scale tensors"),
    (dict(rows=202), b"multiple of 4"),
    (dict(st=(200 * 2 * 128, 128, 2 * 128 + 8)), b"multiple of 16 bytes"),
    (dict(st=(200 * 2 * 128, 136, 2 * 128)), b"multiple of 16 bytes"),
    (dict(Hq=3), b"multiple of the key/value heads"),
])
def test_attention_rows_refusals(lib, kw, needle):
    assert _fwd(lib, **kw) < 0, kw
    assert needle in lib.svgb_last_error(), (kw, lib.svgb_last_error())


def test_attention_rows_reaches_the_plan_check(lib):
    plan = _plan(7)
    plan.S = 300
    assert _fwd(lib, plan=plan) < 0
    assert b"plan was built for" in lib.svgb_last_error()


@pytest.mark.parametrize("args,needle", [
    ((PTR, 0, PTR, PTR, 10, 2, 64, 256, 128), b"head_dim 128 (got 64)"),
    ((PTR, 2, PTR, PTR, 10, 2, 128, 256, 128), b"bf16 or fp16 input"),
    ((PTR, 0, PTR, PTR, 10, 2, 128, 260, 128), b"multiples of 8 elements"),
    ((PTR + 8, 0, PTR, PTR, 10, 2, 128, 256, 128), b"16-byte"),
    ((PTR, 0, PTR, PTR, 0, 2, 128, 256, 128), b"bad sizes"),
])
def test_quantize_rows_refusals(lib, args, needle):
    assert lib.svgb_quantize_e4m3_rows(*args, None) < 0
    assert needle in lib.svgb_last_error(), lib.svgb_last_error()


# --------------------------------------------------------------------------------------------
# Python: the format from the scale tensors' shape
# --------------------------------------------------------------------------------------------
class _Plan:
    """A KV-cache plan stand-in: B = 2 streams of Sq = 5 queries into 2 x 512 cache rows."""
    source = (2, 5)
    S_kv = 1024
    desc = type("D", (), {"kind": 7})()


def _kv(dtype=E4M3, D=128, rows=512):
    return torch.zeros(2, rows, 2, D, dtype=dtype), torch.zeros(2, rows, 2, D, dtype=dtype)


def _rows(shape=(2, 2, 512), dtype=torch.float32):
    return torch.ones(shape, dtype=dtype)


@pytest.mark.parametrize("ks,vs,needle", [
    (_rows(), torch.ones(2), "mix formats"),
    (torch.ones(2), _rows(), "mix formats"),
    (torch.ones(2, 2), torch.ones(2), r"k_scale must be a float32 tensor \[Hkv=2\]"),
    (_rows(), None, "mix formats"),
    (_rows((2, 2, 256)), _rows(), r"per-row k_scale must be a contiguous float32 tensor"),
    (_rows(), _rows(dtype=torch.float64), r"per-row v_scale must be a contiguous float32"),
    (_rows((2, 512, 2)).transpose(1, 2), _rows(), r"per-row k_scale must be a contiguous"),
])
def test_attn_fwd_format_refusals(monkeypatch, ks, vs, needle):
    from svgb200 import core
    from svgb200._lib import SvgbError

    monkeypatch.setattr(core, "lib", lambda: pytest.fail("a launch"))
    kc, vc = _kv()
    with pytest.raises(SvgbError, match=needle):
        core._attn_kvcache(torch.zeros(2, 5, 4, 128, dtype=torch.bfloat16), kc, vc, _Plan(), False, None, None, ks, vs)


def test_per_row_scales_need_d128_and_rows_multiple_of_4(monkeypatch):
    from svgb200 import core
    from svgb200._lib import SvgbError

    kc, vc = _kv(rows=510)
    with pytest.raises(SvgbError, match="multiple of 4"):
        core._row_scales("x", _rows((2, 2, 510)), _rows((2, 2, 510)), kc)
    kc, vc = _kv(D=64)
    with pytest.raises(SvgbError, match="head_dim 128"):
        core._row_scales("x", _rows(), _rows(), kc)


def test_append_format_refusals(monkeypatch):
    from svgb200 import core
    from svgb200._lib import SvgbError

    monkeypatch.setattr(core, "_need_cuda", lambda *ts: None)
    monkeypatch.setattr(core, "lib", lambda: pytest.fail("a launch"))
    kc, vc = _kv()
    k = torch.zeros(2, 4, 2, 128, dtype=torch.bfloat16)
    with pytest.raises(SvgbError, match="mix formats"):
        core.kvcache_append(kc, vc, k, k, 0, k_scale=torch.ones(2), v_scale=_rows())
    with pytest.raises(SvgbError, match=r"\[num_blocks, Hkv, block_rows\]=\[2, 2, 512\]"):
        core.kvcache_append(kc, vc, k, k, 0, k_scale=_rows((2, 2, 500)), v_scale=_rows())
    kb, vb = _kv(torch.bfloat16)
    with pytest.raises(SvgbError, match="are for float8_e4m3fn caches"):
        core.kvcache_append(kb, vb, k, k, 0, k_scale=_rows(), v_scale=_rows())


def _recording(monkeypatch):
    from svgb200 import core

    seen = []

    class _Lib:
        def __getattr__(self, name):
            return lambda *a: seen.append(name) or 0

    monkeypatch.setattr(core, "lib", lambda: _Lib())
    monkeypatch.setattr(core, "_need_cuda", lambda *ts: None)
    monkeypatch.setattr(core, "_stream", lambda t: 0)
    monkeypatch.setattr(core, "_seqlens", lambda s, B, dev: torch.zeros(B, dtype=torch.int32))
    plan = _Plan()
    plan.ws = torch.zeros(16, dtype=torch.uint8)
    plan.desc = core.Plan()
    plan.desc.kind = core.PLAN_KVCACHE
    return core, seen, plan


def test_formats_reach_their_entries(monkeypatch):
    """[Hkv] scales reach the per-head entries (and their q quantisation, svgb_quantize_e4m3), no scales the 16-bit ones,
    and [num_blocks, Hkv, block_rows] scales the per-row append, the per-row quantiser and the per-row forward."""
    core, seen, plan = _recording(monkeypatch)
    q = torch.zeros(2, 5, 4, 128, dtype=torch.bfloat16)
    k = torch.zeros(2, 4, 2, 128, dtype=torch.bfloat16)
    kb, vb = _kv(torch.bfloat16)
    core.kvcache_append(kb, vb, k, k, 0)
    core._attn_kvcache(q, kb, vb, plan, False, None, None)
    assert seen == ["svgb_kvcache_append", "svgb_attn_fwd_strided"]
    seen.clear()
    kc, vc = _kv()
    core.kvcache_append(kc, vc, k, k, 0, k_scale=torch.ones(2), v_scale=torch.ones(2))
    core._attn_kvcache(q, kc, vc, plan, False, None, None, torch.ones(2), torch.ones(2))
    assert seen == ["svgb_kvcache_append_e4m3", "svgb_quantize_e4m3", "svgb_attn_fwd_strided_e4m3"]
    seen.clear()
    core.kvcache_append(kc, vc, k, k, 0, k_scale=_rows(), v_scale=_rows())
    core._attn_kvcache(q, kc, vc, plan, False, None, None, _rows(), _rows())
    assert seen == ["svgb_kvcache_append_e4m3_rows", "svgb_quantize_e4m3_rows", "svgb_attn_fwd_kvcache_e4m3_rows"]
