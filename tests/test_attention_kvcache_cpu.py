"""KV-cache attention (svgb_kvcache_append, svgb_attn_plan_kvcache, flash_attn_with_kvcache) without a GPU: the
kernels' origin and chunk classification compiled for the host against the logical-position predicate, the host mirror
and its clamping, the workspace bound, the ABI refusals, and the drop-in's argument mapping and refusals."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

import kvcache_mask as km
from test_attention_local_cpu import CSRC, PTR, lib  # noqa: F401  (lib: the module-scoped library fixture)

# Input per case: "B Sq sink left right" then L_0 .. L_B-1.  Output: per stream the Sq x L grid of mask_allowed on the
# positions the kernel derives (kv_origin of the query row, logical key positions), then, per item and logical chunk,
# seg_chunk_kind with that origin.
PROBE = r"""
#include <cstdio>
#include <vector>
#include "attn_common.cuh"
using namespace svgb;
int main() {
  int B, Sq, sink, left, right;
  while (std::scanf("%d %d %d %d %d", &B, &Sq, &sink, &left, &right) == 5) {
    std::vector<int> kv(B + 2);
    kv[0] = B; kv[1] = Sq;
    for (int b = 0; b < B; ++b) std::scanf("%d", &kv[2 + b]);
    for (int b = 0; b < B; ++b) {
      const int L = kv[2 + b];
      std::vector<unsigned char> out(static_cast<size_t>(Sq) * L);
      for (int i = 0; i < Sq; ++i) {
        const SegOrigin o = kv_origin(kv.data(), b * Sq + i, sink);
        for (int t = 0; t < L; ++t)
          out[static_cast<size_t>(i) * L + t] = mask_allowed(MASK_LOCAL, b * Sq + i - o.shift, t, o.sink_end, left, right);
      }
      std::fwrite(out.data(), 1, out.size(), stdout);
      for (int r0 = 0; r0 < Sq; r0 += kItemRows) {
        const int row = b * Sq + r0, nr = Sq - r0 < kItemRows ? Sq - r0 : kItemRows;
        for (int c0 = 0; c0 < L; c0 += kChunkCols) {
          const int c1 = (c0 + kChunkCols < L ? c0 + kChunkCols : L) - 1;
          const unsigned char k = seg_chunk_kind(false, row, row + nr - 1, c0, c1, kv_origin(kv.data(), row, sink), left, right);
          std::fwrite(&k, 1, 1, stdout);
        }
      }
    }
  }
  return 0;
}
"""

BIG = 10 ** 6
# (L_b, Sq, sink, left, right): causal, windows whose edges fall inside chunks and pages, sinks ending mid-chunk,
# L_b = 0, Sq > L_b, decode Sq = 1
CASES = [
    ([1000, 0, 300], 300, 0, BIG, 0),
    ([777, 1300], 260, 70, 300, 0),
    ([640, 2000, 5], 130, 0, 255, 17),
    ([100, 600, 1], 1, 0, BIG, 0),
    ([50, 400, 901], 520, 129, 0, 0),
    ([3000], 700, 300, 517, 0),
]


@pytest.fixture(scope="module")
def probe(tmp_path_factory):
    nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not found")
    d = tmp_path_factory.mktemp("kvcache_probe")
    (d / "probe.cu").write_text(PROBE)
    subprocess.run([nvcc, "-std=c++17", "-I", str(CSRC), str(d / "probe.cu"), "-o", str(d / "probe")], check=True,
                   capture_output=True)

    def run(Ls, Sq, sink, left, right):
        text = f"{len(Ls)} {Sq} {sink} {left} {right}\n{' '.join(map(str, Ls))}\n"
        return subprocess.run([str(d / "probe")], input=text.encode(), capture_output=True, check=True).stdout

    return run


@pytest.mark.parametrize("case", range(len(CASES)))
def test_kernel_origin_and_chunk_kinds(probe, case):
    """Query i of stream b at logical position L_b - Sq + i: the kernel's predicate on every pair, and the planner's
    FULL / ELEM / omitted on every (item, chunk), equal the semantics."""
    Ls, Sq, sink, left, right = CASES[case]
    out = memoryview(probe(Ls, Sq, sink, left, right))
    at = 0
    for L in Ls:
        grid = np.frombuffer(out[at:at + Sq * L], np.uint8).reshape(Sq, L).astype(bool)
        at += Sq * L
        p = np.arange(Sq)[:, None] + (L - Sq)
        kv = np.arange(L)[None, :]
        want = (kv < sink) | ((p - kv <= left) & (kv - p <= right))
        assert np.array_equal(grid, want), (case, L)
        for r0 in range(0, Sq, 256):
            for c0 in range(0, L, 128):
                blk = want[r0:r0 + 256, c0:c0 + 128]
                kind = out[at]
                at += 1
                assert kind == (0 if not blk.any() else 1 if blk.all() else 2), (case, L, r0, c0)
    assert at == len(out)


def test_mirror_clamps_lengths_and_blocks():
    assert [km.kv_len(s, 40, 1152) for s in (900, -5, 10 ** 6, 0)] == [940, 40, 1152, 40]
    table = [[-3, 2, 99]]
    assert [km.block_of(0, t, nblocks=20, block_rows=128, table=table) for t in (0, 128, 300)] == [0, 2, 19]
    assert km.block_of(1, 5, nblocks=4, block_rows=512, batch_idx=[0, 7]) == 3
    assert km.block_of(2, 5, nblocks=2, block_rows=512) == 1
    items, lens = km.plan([300], Sq=10, new_len=0, nblocks=4, block_rows=128, table=[[3, 1, 0]], sink=0, left=100,
                          right=0)
    assert lens == [300]
    # positions 290 .. 299 see keys 190 .. 299: chunks 1 (ELEM) and 2 (valid 44), never chunk 0's page
    ((b, r0, nr, chunks),) = items
    assert (b, r0, nr) == (0, 0, 10)
    assert chunks == [(1 * 128, 128, True, 1), (0 * 128 + 0, 44, True, 2)]


def _bytes(lib, B, Sq, cap, sink=0, left=BIG, right=0):
    n = C.c_size_t()
    assert lib.svgb_attn_plan_kvcache_bytes(B, Sq, cap, sink, left, right, C.byref(n)) == 0
    return n.value


def test_workspace_bound(lib):
    """16 + align16(4 (B + 2)) + 32 I + 8 I slots, slots = min(ceil(cap / 128), ceil(sink / 128) + (255 + left + right)
    / 128 + 2): host sizes only, and a window shrinks it."""
    def want(B, Sq, cap, sink, left, right):
        items = B * -(-Sq // 256)
        slots = min(-(-cap // 128), -(-sink // 128) + (255 + left + right) // 128 + 2)
        return 16 + -(-4 * (B + 2) // 16) * 16 + 32 * items + 8 * items * slots

    for args in [(1, 4680, 32760, 0, BIG, 0), (1, 4680, 32760, 1560, 14040, 0), (64, 1, 131072, 0, BIG, 0),
                 (3, 300, 1000, 70, 300, 0), (2, 1, 128, 0, 0, 0)]:
        assert _bytes(lib, *args) == want(*args), args
    assert _bytes(lib, 1, 4680, 32760, 1560, 14040, 0) < _bytes(lib, 1, 4680, 32760)


def _plan_call(lib, *, seqlens=PTR, batch_idx=None, table=None, B=2, Sq=100, Snew=0, nblocks=4, rows=512,
               max_pages=0, sink=0, left=10, right=0, ws=1 << 20):
    from svgb200._lib import Plan

    plan = Plan()
    rc = lib.svgb_attn_plan_kvcache(seqlens, batch_idx, table, B, Sq, Snew, nblocks, rows, max_pages, sink, left, right,
                                    PTR, ws, C.byref(plan), None)
    return rc, plan


def test_planner_refusals(lib):
    for kw, needle in [(dict(table=PTR, rows=200, max_pages=4), b"multiple of 128"),
                       (dict(table=PTR, rows=256, max_pages=0), b"max_pages"),
                       (dict(table=PTR, rows=256, max_pages=4, batch_idx=PTR), b"cache_batch_idx"),
                       (dict(sink=-1), b"sink (-1)"), (dict(left=-1), b"left (-1)"), (dict(right=-2), b"right (-2)"),
                       (dict(seqlens=None), b"null pointer"), (dict(ws=64), b"workspace too small"),
                       (dict(nblocks=0), b"bad cache geometry"), (dict(Snew=-1), b"Snew=-1"),
                       (dict(nblocks=1, rows=(1 << 29) + 128), b"exceeds 2^29")]:
        rc, _ = _plan_call(lib, **kw)
        assert rc < 0, kw
        assert needle in lib.svgb_last_error(), (kw, lib.svgb_last_error())


def _append(lib, *, dtype=0, D=128, Snew=4, table=None, rows=512, max_pages=0, batch_idx=None, ptrs=(PTR,) * 4,
            st=(8, 8, 8)):
    s = (C.c_longlong * 3)(*st)
    return lib.svgb_kvcache_append(*ptrs, PTR, batch_idx, table, dtype, 2, Snew, 2, D, 4, rows, max_pages, s, s, s, s,
                                   None)


def test_append_refusals(lib):
    for kw, needle in [(dict(dtype=2), b"bf16 or fp16"), (dict(D=96), b"head_dim 96"), (dict(Snew=0), b"no new rows"),
                       (dict(ptrs=(PTR, None, PTR, PTR)), b"null pointer"),
                       (dict(table=PTR, rows=200, max_pages=2), b"multiple of 128"),
                       (dict(st=(8, 8, 4)), b"multiple of 8")]:
        assert _append(lib, **kw) < 0, kw
        assert needle in lib.svgb_last_error(), (kw, lib.svgb_last_error())


def _kv_plan(B=2, Sq=100, rows=4 * 512):
    from svgb200._lib import Plan

    p = Plan()
    p.kind, p.S, p.BH = 7, B * Sq, rows
    p.mask_mode, (p.m0, p.m1, p.m2) = 10, (0, 10, 0)
    p.max_items, (p.items_off, p.chunks_off, p.bytes) = 2, (48, 112, 4096)
    return p


def test_forward_and_backward_refuse_the_kvcache_plan_by_name(lib):
    """e4m3 inputs, row vectors and every backward entry refuse a KV-cache plan and name it; _gqa takes it."""
    plan = _kv_plan(Sq=100, rows=200)
    assert lib.svgb_attn_fwd(PTR, PTR, PTR, PTR, PTR, PTR, PTR, None, None, None, None, 2, 2, 200, 128, 128, 200 * 128,
                             128, 200 * 128, 0.1, C.byref(plan), PTR, None) < 0
    assert b"KV-cache plans (svgb_attn_plan_kvcache) take bf16 or fp16" in lib.svgb_last_error()
    for rows in [(PTR, None, None), (None, PTR, None), (None, None, PTR)]:
        assert lib.svgb_attn_fwd(PTR, PTR, PTR, None, None, None, PTR, None, *rows, 0, 2, 200, 128, 128, 200 * 128,
                                 128, 200 * 128, 0.1, C.byref(plan), PTR, None) < 0
        assert b"KV-cache plans" in lib.svgb_last_error()
    assert lib.svgb_attn_bwd(PTR, PTR, PTR, PTR, PTR, PTR, PTR, PTR, PTR, 0, 2, 200, 128, 128, 200 * 128, 0.1,
                             C.byref(plan), PTR, C.byref(plan), PTR, PTR, 1 << 20, None) < 0
    assert b"KV-cache plan (svgb_attn_plan_kvcache) has no backward" in lib.svgb_last_error()
    assert lib.svgb_attn_bwd_kv(PTR, PTR, PTR, PTR, PTR, PTR, PTR, PTR, PTR, 0, 2, 200, 300, 128, 128, 200 * 128, 128,
                                300 * 128, 0.1, C.byref(plan), PTR, C.byref(plan), PTR, PTR, 1 << 20, None) < 0
    assert b"has no backward" in lib.svgb_last_error()
    assert lib.svgb_attn_bwd_gqa(PTR, PTR, PTR, PTR, PTR, PTR, PTR, PTR, PTR, 0, 4, 2, 200, 300, 128, 128, 200 * 128,
                                 128, 300 * 128, 0.1, C.byref(plan), PTR, C.byref(plan), PTR, PTR, 1 << 20, None) < 0
    assert b"has no backward" in lib.svgb_last_error()
    s = (C.c_longlong * 3)(8, 8, 8)
    assert lib.svgb_attn_bwd_strided(PTR, PTR, PTR, PTR, PTR, PTR, PTR, PTR, PTR, 0, 1, 2, 2, 200, 300, 128,
                                     *([s] * 8), 0.1, C.byref(plan), PTR, C.byref(plan), PTR, PTR, 1 << 20, None) < 0
    assert b"has no backward" in lib.svgb_last_error()
    # svgb_attn_fwd_gqa checks the plan against the call's lengths, and takes it when they match
    assert lib.svgb_attn_fwd_gqa(PTR, PTR, PTR, PTR, None, 0, 4, 2, 200, 999, 128, 128, 200 * 128, 128, 999 * 128,
                                 128, 200 * 128, 0.1, C.byref(plan), PTR, None) < 0
    assert b"Skv=200" in lib.svgb_last_error()


# --------------------------------------------------------------------------------------------
# Python: the drop-in's mapping and refusals
# --------------------------------------------------------------------------------------------
class _T:
    """A stand-in for a tensor: shape only."""

    def __init__(self, *shape, requires_grad=False):
        self.shape = shape
        self.requires_grad = requires_grad
        self.device = "cuda"

    def numel(self):
        return int(np.prod(self.shape))


@pytest.fixture
def dropin(monkeypatch):
    from svgb200 import core, patch

    calls = []
    monkeypatch.setattr(core, "_seqlens", lambda s, B, dev: ("lens", s, B))
    monkeypatch.setattr(core, "kvcache_append", lambda *a, **kw: calls.append(("append", a, kw)))
    monkeypatch.setattr(core, "plan_kvcache", lambda *a, **kw: calls.append(("plan", a, kw)) or "plan")
    monkeypatch.setattr(core, "attn_fwd", lambda *a, **kw: calls.append(("fwd", a, kw)) or "out")
    return patch, calls


def test_dropin_contiguous_mapping(dropin):
    patch, calls = dropin
    q, kc, vc, k, v = _T(2, 5, 8, 64), _T(3, 1000, 2, 64), _T(3, 1000, 2, 64), _T(2, 5, 2, 64), _T(2, 5, 2, 64)
    bi = _T(2)
    assert patch.flash_attn_with_kvcache(q, kc, vc, k, v, cache_seqlens=7, cache_batch_idx=bi, causal=True,
                                         window_size=(100, 0), softmax_scale=0.5, num_splits=3,
                                         return_softmax_lse=True) == "out"
    ap, pp, fp = calls
    assert ap[0] == "append" and ap[1] == (kc, vc, k, v, ("lens", 7, 2))
    assert ap[2] == dict(block_table=None, cache_batch_idx=bi)
    assert pp[0] == "plan" and pp[1] == (("lens", 7, 2),)
    assert pp[2] == dict(q_len=5, num_blocks=3, new_len=5, cache_len=1000, block_table=None, page_size=None,
                         cache_batch_idx=bi, causal=True, window_size=(100, 0))
    assert fp[0] == "fwd" and fp[1] == (q, kc, vc, "plan") and fp[2] == dict(return_lse=True, sm_scale=0.5)


def test_dropin_paged_mapping_and_defaults(dropin):
    patch, calls = dropin
    q, kc, vc, table = _T(2, 1, 8, 128), _T(40, 256, 2, 128), _T(40, 256, 2, 128), _T(2, 9)
    patch.flash_attn_with_kvcache(q, kc, vc, cache_seqlens=_T(2), block_table=table)
    pp, fp = calls  # no append without k, v
    assert pp[2]["page_size"] == 256 and pp[2]["cache_len"] is None and pp[2]["block_table"] is table
    assert pp[2]["new_len"] == 0 and pp[2]["num_blocks"] == 40
    assert fp[2] == dict(return_lse=False, sm_scale=None)
    calls.clear()
    patch.flash_attn_with_kvcache(q, _T(2, 512, 2, 128), _T(2, 512, 2, 128))  # contiguous: the whole cache
    assert calls[0][1] == (("lens", 512, 2),)


@pytest.mark.parametrize("kw,needle", [
    (dict(rotary_cos=_T(4, 32), rotary_sin=_T(4, 32)), "rotary_cos"), (dict(rotary_sin=_T(4, 32)), "rotary_sin"),
    (dict(cache_leftpad=_T(2)), "cache_leftpad"), (dict(softcap=30.0), "softcap=30.0"),
    (dict(alibi_slopes=_T(8)), "alibi_slopes"), (dict(k=_T(2, 5, 2, 64)), "k and v"),
    (dict(block_table=_T(2, 3)), "needs cache_seqlens"),
])
def test_dropin_refusals(dropin, kw, needle):
    from svgb200._lib import SvgbError

    patch, calls = dropin
    with pytest.raises(SvgbError, match=needle):
        patch.flash_attn_with_kvcache(_T(2, 5, 8, 64), _T(2, 512, 2, 64), _T(2, 512, 2, 64), **kw)
    assert calls == []


def test_dropin_refuses_grad_first(dropin, monkeypatch):
    from svgb200 import core
    from svgb200._lib import SvgbError

    patch, calls = dropin
    monkeypatch.setattr(core.torch, "is_grad_enabled", lambda: True)
    with pytest.raises(SvgbError, match="no backward"):
        patch.flash_attn_with_kvcache(_T(2, 5, 8, 64, requires_grad=True), _T(2, 512, 2, 64), _T(2, 512, 2, 64))
    assert calls == []


def test_plan_kvcache_window_mapping(monkeypatch):
    """FlashAttention's conventions: -1 is unbounded (capacity + Sq), causal sets right = 0 and conflicts with a
    positive right window."""
    from svgb200 import core
    from svgb200._lib import SvgbError

    seen = []
    monkeypatch.setattr(core, "_seqlens", lambda s, B, dev: _Ptr())
    monkeypatch.setattr(core, "_cache_layout", lambda *a: (None, None, 0))
    monkeypatch.setattr(core, "check", lambda rc, what: None)
    monkeypatch.setattr(core.torch, "empty", lambda *a, **kw: _Ptr())

    class _Lib:
        def svgb_attn_plan_kvcache_bytes(self, *a):
            seen.append(("bytes", a[:6]))
            return 0

        def svgb_attn_plan_kvcache(self, *a):
            seen.append(("plan", a[3:12]))
            return 0

    monkeypatch.setattr(core, "lib", lambda: _Lib())
    monkeypatch.setattr(core.torch.cuda, "current_stream", lambda d: type("S", (), {"cuda_stream": 0})())
    bi = _T(3)
    core.plan_kvcache(5, q_len=40, num_blocks=4, cache_len=1000, cache_batch_idx=bi, causal=True, sink=9)
    assert seen[0] == ("bytes", (3, 40, 1000, 9, 1040, 0))
    assert seen[1] == ("plan", (3, 40, 0, 4, 1000, 0, 9, 1040, 0))
    seen.clear()
    core.plan_kvcache(5, q_len=40, num_blocks=4, cache_len=1000, cache_batch_idx=bi, window_size=(100, -1), new_len=3)
    assert seen[1] == ("plan", (3, 40, 3, 4, 1000, 0, 0, 100, 1040))
    with pytest.raises(SvgbError, match="causal=True"):
        core.plan_kvcache(5, q_len=40, num_blocks=4, cache_len=1000, cache_batch_idx=bi, causal=True,
                          window_size=(-1, 4))


class _Ptr:
    def data_ptr(self):
        return 0

    def numel(self):
        return 0
