"""Low-level torch-facing wrappers over the C ABI: pointer/stride plumbing, workspace caching,
argument checks.  Everything here runs the CUDA library; there is no eager fallback.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Optional

import torch

from ._lib import Plan, SvgbError, check, lib

MASK_NONE, MASK_HY, MASK_WAN, MASK_COG = 0, 1, 2, 3
# SVG1 profiling masks (include/svgb200.h SVGB_MASK_PROF_*): the element masks of sample_mse, also accepted by plan_band
MASK_PROF_HY_S, MASK_PROF_HY_T, MASK_PROF_WAN_S, MASK_PROF_WAN_T, MASK_PROF_COG_S, MASK_PROF_COG_T = 4, 5, 6, 7, 8, 9
# local band with attention sinks (SVGB_MASK_LOCAL): m0 = sink, m1 = left, m2 = right; plan_local builds it
MASK_LOCAL = 10
# block-causal mask (SVGB_MASK_BLOCK_CAUSAL): m0 = sink, m1 = block | (block - first_block) << 16, m2 = window;
# plan_block_causal, plan_local_varlen(block=) and plan_kvcache(block=) build it
MASK_BLOCK_CAUSAL = 12
# svgb_plan.kind (include/svgb200.h SVGB_PLAN_*)
PLAN_VARBLOCK, PLAN_BAND, PLAN_GATHER, PLAN_BAND_T, PLAN_SEG, PLAN_SEG_T, PLAN_KVCACHE = 1, 2, 3, 4, 5, 6, 7
PLAN_KVCACHE_SPLIT = 8
# SVGB_PLAN_SEG_BOUNDS_OFF: a segment plan's {nseg, cu_q, cu_k} in its workspace, a KV-cache plan's {B, Sq, L_b}
SEG_BOUNDS_OFF = 16
_E4M3 = 2  # SVGB_E4M3 (the 16-bit dtype ids come from _dt)

# launches issued through this module since import (bench.py reports it as gpu_launches)
launch_count = 0


def _bump(n=1):
    global launch_count
    launch_count += n


def _dt(t: torch.Tensor) -> int:
    if t.dtype == torch.bfloat16:
        return 0
    if t.dtype == torch.float16:
        return 1
    raise SvgbError(f"unsupported dtype {t.dtype}: svgb200 kernels take bfloat16 or float16")


def _stream(t: torch.Tensor) -> int:
    return torch.cuda.current_stream(t.device).cuda_stream


def _need_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise SvgbError("svgb200 operators need CUDA tensors (no CPU fallback)")


def _p(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


_ws_cache: dict = {}


def workspace(key, nbytes: int, device) -> torch.Tensor:
    """Cached uint8 scratch buffer (stream-ordered reuse on the current stream)."""
    k = (key, str(device))
    buf = _ws_cache.get(k)
    if buf is None or buf.numel() < nbytes:
        buf = torch.empty(max(int(nbytes), 256), dtype=torch.uint8, device=device)
        _ws_cache[k] = buf
    return buf


def device_check():
    a, b, c = C.c_int(), C.c_int(), C.c_int()
    check(lib().svgb_device_check(C.byref(a), C.byref(b), C.byref(c)), "svgb_device_check")
    return a.value, b.value, c.value


# ----------------------------------------------------------------------------------------------
# plans
# ----------------------------------------------------------------------------------------------
@dataclass
class AttnPlan:
    """Device-resident work list + its host descriptor.  `source` keeps what a variable-block plan was built from
    (map, row sizes, column sizes, and their torch version counters at build time) so that key_major() can plan the
    transpose, and a segment plan's segment count; `_key_major` caches that plan."""
    desc: Plan
    ws: torch.Tensor
    source: Optional[tuple] = None
    _key_major: Optional["AttnPlan"] = None

    @property
    def S(self):
        return self.desc.S

    @property
    def S_kv(self):
        """Key/value length: a rectangular variable-block plan records it in m0, a segment plan (which serves every
        head) in BH, and so does a KV-cache plan (the cache's rows) (include/svgb200.h, svgb_plan)."""
        d = self.desc
        if d.kind in (PLAN_SEG, PLAN_SEG_T, PLAN_KVCACHE, PLAN_KVCACHE_SPLIT):
            return d.BH
        return d.m0 if d.kind == PLAN_VARBLOCK and d.m0 > 0 else d.S

    def key_major(self) -> "AttnPlan":
        """The plan the backward's dK / dV kernel walks (one work list per key range), built on first use: the band
        mask's transposed plan, or the variable-block planner on the transposed map with row and column sizes swapped.
        Gather plans and the profiling masks have no backward."""
        if self._key_major is None:
            d = self.desc
            if d.kind == PLAN_BAND:
                if _is_profiling(d.mask_mode):
                    raise SvgbError(f"attention backward: the profiling mask mode {d.mask_mode} has no backward "
                                    "(executed masks NONE / HY / WAN / COG / LOCAL only)")
                self._key_major = plan_band_t(d.mask_mode, d.m0, d.m1, d.m2, d.BH, d.S, self.ws.device)
            elif d.kind == PLAN_SEG:
                # from the plan's own copy of the bounds {nseg, cu_q, cu_k}, which is what the forward ran; source holds
                # nseg for the host
                (nseg,) = self.source
                cu = self.ws.data_ptr() + SEG_BOUNDS_OFF + 4
                if d.mask_mode == MASK_BLOCK_CAUSAL:  # (sink, W, C, F) from m0..m2 = sink, C | (C - F) << 16, W
                    name, params = "svgb_attn_plan_block_varlen_t", (d.m0, d.m2, d.m1 & 0xffff,
                                                                     (d.m1 & 0xffff) - (d.m1 >> 16))
                else:
                    name, params = "svgb_attn_plan_local_varlen_t", (d.m0, d.m1, d.m2)
                self._key_major = _plan_local_varlen(name, cu, cu + 4 * (nseg + 1), nseg, d.S, d.BH, *params,
                                                     self.ws.device)
            elif d.kind == PLAN_VARBLOCK and self.source is not None:
                *ts, versions = self.source
                if tuple(t._version for t in ts) != versions:
                    # the key-major plan must describe the mask this plan was built from (the one the forward ran)
                    raise SvgbError("attention backward: the block map or block sizes of this plan were modified in "
                                    "place after the plan was built; rebuild the plan")
                m, r, c = ts
                kt = plan_varblock(m.transpose(1, 2), c, r, self.S_kv, S_kv=d.S)
                if d.items_stride == 0:  # one map shared by every head (svgb200.h, svgb_plan): so is its transpose
                    kt.desc.items_stride = 0
                self._key_major = kt
            elif d.kind == PLAN_GATHER:
                raise SvgbError("attention backward: gather plans (row-gather path, q_rows / kv_rows) have no backward")
            elif d.kind == PLAN_KVCACHE:
                raise SvgbError("attention backward: a KV-cache plan (plan_kvcache) has no backward; it runs forward "
                                "only, as flash_attn_with_kvcache does")
            elif d.kind == PLAN_KVCACHE_SPLIT:
                raise SvgbError("attention backward: a split KV-cache plan (plan_kvcache(num_splits=)) has no "
                                "backward; it runs forward only")
            else:
                raise SvgbError(f"attention backward: plan kind {d.kind} has no key-major form")
        return self._key_major


def plan_varblock(block_map: torch.Tensor, row_sz: torch.Tensor, col_sz: torch.Tensor, S: int,
                  gather: bool = False, *, S_kv: Optional[int] = None) -> AttnPlan:
    """block_map [BH,QC,KC] bool/uint8, row_sz [BH,QC], col_sz [BH,KC] (any int dtype) on GPU.
    gather=True lowers the map for the row-gather kernel path (exactly-full chunks, optional fused
    permutation through attn_fwd(..., q_rows=, kv_rows=)).
    S_kv: key/value length when it differs from the query length S (row sizes sum to S, column sizes to S_kv): the
    rectangular plan of svgb_attn_plan_varblock_kv, which attn_fwd / attn_bwd / attention run on k, v of S_kv rows.
    S_kv == S (or None) is the square planner's call.  As for the square planner, the sizes are device tensors and are
    not checked against S / S_kv: sizes that overrun them make the kernels read and store rows past the tensors.

    Every plan owns its device work list (torch's caching allocator makes the per-call allocation free of
    cudaMalloc / syncs), so plans of one shape can be held and executed in any order or on different streams."""
    _need_cuda(block_map, row_sz, col_sz)
    BH, QC, KC = block_map.shape
    m = block_map.contiguous()
    m = m.view(torch.uint8) if m.dtype == torch.bool else m.to(torch.uint8)
    r = row_sz.reshape(BH, QC).to(torch.int32).contiguous()
    c = col_sz.reshape(BH, KC).to(torch.int32).contiguous()
    rect = S_kv is not None and S_kv != S
    if rect and gather:
        raise SvgbError(f"gather plans need S_kv == S (got S={S}, S_kv={S_kv}): the rectangular plan is TMA only")
    # the rectangular planner pair takes S_kv after S; the square and gather planners share one workspace query
    name, lens = ("svgb_attn_plan_varblock_kv", (S, S_kv)) if rect else ("svgb_attn_plan_varblock", (S,))
    nbytes = C.c_size_t()
    check(getattr(lib(), name + "_bytes")(BH, *lens, QC, KC, C.byref(nbytes)), name + "_bytes")
    ws = torch.empty(nbytes.value, dtype=torch.uint8, device=m.device)
    desc = Plan()
    name += "_gather" if gather else ""
    check(getattr(lib(), name)(m.data_ptr(), r.data_ptr(), c.data_ptr(), BH, *lens, QC, KC, ws.data_ptr(), ws.numel(),
                               C.byref(desc), _stream(m)), name)
    _bump()
    return AttnPlan(desc, ws, None if gather else (m, r, c, (m._version, r._version, c._version)))


def _plan_band(bytes_fn, plan_fn, name, mask_mode, m0, m1, m2, BH, S, device) -> AttnPlan:
    nbytes = C.c_size_t()
    check(bytes_fn(S, C.byref(nbytes)), f"{name}_bytes")
    ws = torch.empty(nbytes.value, dtype=torch.uint8, device=device)  # owned by the plan (long-lived)
    desc = Plan()
    check(plan_fn(mask_mode, m0, m1, m2, BH, S, ws.data_ptr(), ws.numel(), C.byref(desc),
                  torch.cuda.current_stream(device).cuda_stream), f"svgb_attn_{name}")
    _bump()
    return AttnPlan(desc, ws)


def plan_band(mask_mode: int, m0: int, m1: int, m2: int, BH: int, S: int, device) -> AttnPlan:
    return _plan_band(lib().svgb_attn_plan_band_bytes, lib().svgb_attn_plan_band, "plan_band", mask_mode, m0, m1, m2,
                      BH, S, device)


def plan_band_t(mask_mode: int, m0: int, m1: int, m2: int, BH: int, S: int, device) -> AttnPlan:
    """Key-major form of plan_band's mask (include/svgb200.h svgb_attn_plan_band_t), for attn_bwd."""
    return _plan_band(lib().svgb_attn_plan_band_t_bytes, lib().svgb_attn_plan_band_t, "plan_band_t", mask_mode, m0,
                      m1, m2, BH, S, device)


def plan_local(BH: int, S: int, device, *, causal: bool = False, window_size=(-1, -1), sink: int = 0) -> AttnPlan:
    """Causal or sliding-window attention with attention sinks, in FlashAttention's conventions: query q sees key kv
    when kv < sink, or when kv lies at most window_size[0] positions behind q and at most window_size[1] ahead of it
    (-1: unbounded); causal=True sets the right window to 0 and conflicts with a positive window_size[1].  A band plan
    of MASK_LOCAL(sink, left, right), so every entry that runs band plans runs it, forward and backward."""
    left, right = (int(w) for w in window_size)
    if causal:
        if right > 0:
            raise SvgbError(f"plan_local: causal=True looks no key ahead, but window_size[1] = {right}")
        right = 0
    left, right = (S if w == -1 else w for w in (left, right))
    return plan_band(MASK_LOCAL, int(sink), left, right, BH, S, device)


def _block_m1(who, block, first_block, window, sink):
    """(m1, W) of MASK_BLOCK_CAUSAL from block C, first_block F (None: C) and window W (-1: unbounded, returned as -1),
    refused by name before any launch when C, F, W or sink is out of range or C does not fit its 16 bits."""
    C_ = int(block)
    F = C_ if first_block is None else int(first_block)
    W, sink = int(window), int(sink)
    if not 1 <= C_ < 1 << 16:
        raise SvgbError(f"{who}: block={C_} must lie in [1, 65536) (it is packed in 16 bits)")
    if not 1 <= F <= C_:
        raise SvgbError(f"{who}: first_block={F} must lie in [1, block={C_}]")
    if W != -1 and W < C_:
        raise SvgbError(f"{who}: window={W} must be -1 (unbounded) or >= block={C_}, so that every query keeps its own "
                        "block")
    if sink < 0:
        raise SvgbError(f"{who}: sink={sink} must be >= 0")
    return C_ | (C_ - F) << 16, W


def plan_block_causal(BH: int, S: int, device, *, block: int, first_block: Optional[int] = None, window: int = -1,
                      sink: int = 0) -> AttnPlan:
    """Block-causal attention of autoregressive video (chunk-wise causal, as CausVid and Self-Forcing train): positions
    0 .. S-1 form blocks of `block` = C positions, the first one `first_block` = F long (1 <= F <= C, default C), so block
    ends lie at F, F + C, F + 2C, ...  Query p sees key kv when kv < sink, or when kv lies before the end e(p) of p's block
    and at most `window` = W keys back from it: e(p) - W <= kv < e(p) (W >= C, -1: unbounded).  Every query sees its whole
    block and all earlier ones.  A band plan of MASK_BLOCK_CAUSAL, so every entry that runs band plans runs it, forward
    and backward (attention(), attn_fwd, attn_bwd, key_major()); block=1 is plan_local(causal=True, window_size=(W - 1,
    0), sink=sink)."""
    m1, W = _block_m1("plan_block_causal", block, first_block, window, sink)
    if W == -1:
        W = min(int(S) + int(block), 2**31 - 1)  # a block end lies at most S + C - 1 past key 0
    return plan_band(MASK_BLOCK_CAUSAL, int(sink), m1, W, BH, S, device)


def _plan_local_varlen(name, cu_q, cu_k, nseg, Sq, Skv, *args) -> AttnPlan:
    """args: the planner's mask parameters, (sink, left, right) or for the block entries (sink, W, C, F), then the
    device."""
    *params, device = args
    nbytes = C.c_size_t()
    check(lib().svgb_attn_plan_local_varlen_bytes(nseg, Sq, Skv, C.byref(nbytes)), "svgb_attn_plan_local_varlen_bytes")
    ws = torch.empty(nbytes.value, dtype=torch.uint8, device=device)  # owned by the plan, with its copy of the bounds
    desc = Plan()
    check(getattr(lib(), name)(cu_q, cu_k, nseg, Sq, Skv, *params, ws.data_ptr(), ws.numel(), C.byref(desc),
                               torch.cuda.current_stream(device).cuda_stream), name)
    _bump(2)
    return AttnPlan(desc, ws, (nseg,))


def plan_local_varlen(cu_seqlens_q: torch.Tensor, cu_seqlens_k: Optional[torch.Tensor] = None, *, total_q: int,
                      total_k: Optional[int] = None, causal: bool = False, window_size=(-1, -1),
                      sink: int = 0, block: int = 0, first_block: Optional[int] = None) -> AttnPlan:
    """Causal or sliding-window attention with attention sinks inside packed variable-length segments, in
    FlashAttention's conventions (flash_attn_varlen_func): cu_seqlens_q / cu_seqlens_k are device int [nseg + 1]
    (cu_seqlens_k None: the same segments), query segment i attends key segment i only, and its queries are aligned to
    the END of the key segment (bottom-right), so query qi of segment i sits at key position qi + Lk_i - Lq_i.  Query
    qi sees key kj when kj < sink, or when kj lies at most window_size[0] positions behind that position and at most
    window_size[1] ahead (-1: unbounded); causal=True sets the right window to 0 and conflicts with a positive
    window_size[1].  total_q / total_k (default total_q) are the packed lengths, q.shape[0] and k.shape[0] of a
    [total, H, D] call: they are passed rather than read from cu_seqlens so that planning never waits on the device.
    One plan for every head (any H, batch, GQA group or view); attention() runs it forward and backward, in 'shd' and in
    'bhsd' (every batch element segmented alike).  Rows without an allowed key get o = 0 and lse = -inf.
    block > 0: the block-causal rule of plan_block_causal inside every segment, its blocks anchored at the segment's key
    0 (blocks of `block` keys, the first ending at `first_block`, default block): query position p of segment i sees its
    key kj when kj < sink or e(p) - W <= kj < e(p), with W = window_size[0] counted back from the block end (-1:
    unbounded) and window_size[1] = -1; causal=True is refused (the rule is causal).  Segments whose queries start
    mid-block (Lq_i < Lk_i) round them inside the key segment's grid, as plan_kvcache(block=) does.  One clip per
    segment of a packed batch is chunk-wise causal video training; block=0 is the token rule above."""
    if block:
        if causal:
            raise SvgbError("plan_local_varlen: causal=True is redundant with block= (the block rule is causal); pass "
                            "window_size=(W, -1)")
        W, right = (int(w) for w in window_size)
        if right != -1:
            raise SvgbError(f"plan_local_varlen: with block=, window_size[1] = {right} must be -1 (no key past the "
                            "block end)")
        m1, W = _block_m1("plan_local_varlen", block, first_block, W, sink)
    try:
        _need_cuda(cu_seqlens_q, cu_seqlens_k)
    except SvgbError as e:
        if not block:
            raise
        # the block form plans on the device only: name the mask that was asked for, not just the missing device
        raise SvgbError(f"plan_local_varlen: block-causal masks inside packed segments are not supported on CPU "
                        f"tensors: {e}") from None
    cu_q = cu_seqlens_q.to(torch.int32).contiguous()
    cu_k = cu_q if cu_seqlens_k is None else cu_seqlens_k.to(torch.int32).contiguous()
    if cu_q.dim() != 1 or cu_k.shape != cu_q.shape or cu_q.numel() < 2:
        raise SvgbError(f"plan_local_varlen: cu_seqlens_q {tuple(cu_q.shape)} and cu_seqlens_k {tuple(cu_k.shape)} must "
                        "be 1-D with the same nseg + 1 >= 2 entries")
    Sq = int(total_q)
    Skv = Sq if total_k is None else int(total_k)
    if block:
        C_ = m1 & 0xffff
        if W == -1:  # no block end lies further than the longest segment + C past its key 0
            W = min(max(Sq, Skv) + C_, 2**31 - 1)
        return _plan_local_varlen("svgb_attn_plan_block_varlen", cu_q.data_ptr(), cu_k.data_ptr(), cu_q.numel() - 1,
                                  Sq, Skv, int(sink), W, C_, C_ - (m1 >> 16), cu_q.device)
    left, right = (int(w) for w in window_size)
    if causal:
        if right > 0:
            raise SvgbError(f"plan_local_varlen: causal=True looks no key ahead, but window_size[1] = {right}")
        right = 0
    # -1: no segment is longer than its total, and no query position lies further than that from a key
    left, right = (max(Sq, Skv) if w == -1 else w for w in (left, right))
    return _plan_local_varlen("svgb_attn_plan_local_varlen", cu_q.data_ptr(), cu_k.data_ptr(), cu_q.numel() - 1, Sq,
                              Skv, int(sink), left, right, cu_q.device)


def _seqlens(cache_seqlens, B, device) -> torch.Tensor:
    """cache_seqlens as a device int32 [B]: an int is broadcast on the device, a tensor converted there."""
    if isinstance(cache_seqlens, torch.Tensor):
        _need_cuda(cache_seqlens)
        t = cache_seqlens.to(torch.int32).reshape(-1).contiguous()
        if t.numel() != B:
            raise SvgbError(f"cache_seqlens has {t.numel()} entries for {B} streams")
        return t
    return torch.full((B,), int(cache_seqlens), dtype=torch.int32, device=device)


def _cache_layout(B, block_table, cache_batch_idx):
    """(block_table, cache_batch_idx, max_pages) in the form the KV-cache entries take: device int32, contiguous."""
    if block_table is not None and cache_batch_idx is not None:
        raise SvgbError("cache_batch_idx is for contiguous caches; a paged cache (block_table) takes no cache_batch_idx")
    bt = bi = None
    max_pages = 0
    if block_table is not None:
        _need_cuda(block_table)
        if block_table.dim() != 2 or block_table.shape[0] != B:
            raise SvgbError(f"block_table {tuple(block_table.shape)} must be [B={B}, max_pages]")
        bt = block_table.to(torch.int32).contiguous()
        max_pages = bt.shape[1]
    if cache_batch_idx is not None:
        _need_cuda(cache_batch_idx)
        bi = cache_batch_idx.to(torch.int32).reshape(-1).contiguous()
        if bi.numel() != B:
            raise SvgbError(f"cache_batch_idx has {bi.numel()} entries for {B} streams")
    return bt, bi, max_pages


def kvcache_append(k_cache: torch.Tensor, v_cache: torch.Tensor, k: torch.Tensor, v: torch.Tensor, cache_seqlens, *,
                   block_table: Optional[torch.Tensor] = None, cache_batch_idx: Optional[torch.Tensor] = None,
                   k_scale: Optional[torch.Tensor] = None, v_scale: Optional[torch.Tensor] = None,
                   cu_seqlens: Optional[torch.Tensor] = None):
    """Write the new rows k, v [B, Snew, Hkv, D] into the cache in place, at keys cache_seqlens[b] .. + Snew - 1 of each
    stream b, in one launch.  The cache is contiguous, k_cache / v_cache [B_cache, S_cache, Hkv, D] with stream b in
    row cache_batch_idx[b] (default b), or paged, [num_pages, page_size, Hkv, D] with block_table int [B, max_pages]
    (page_size a multiple of 128).  cache_seqlens: int or device int tensor [B], read on the device only.  Rows whose key
    or block falls outside the cache are not written (include/svgb200.h, svgb_kvcache_append).
    FP8 cache: caches of dtype torch.float8_e4m3fn take 16-bit k, v and k_scale, v_scale, float32 device tensors whose
    shape picks the format.  [Hkv]: one scale per head fixed for the cache's lifetime; each element is stored as
    RN-satfinite(x * (1 / scale[h])), values past 448 * scale saturating (svgb_kvcache_append_e4m3).  [num_blocks, Hkv,
    block_rows] (contiguous, block_rows a multiple of 4, D = 128): one power-of-two scale per cache row, which the append
    computes from the row's absmax and writes there, so nothing saturates (svgb_kvcache_append_e4m3_rows).  16-bit
    caches take no scales.
    cu_seqlens (device int [B + 1], FlashAttention 3's cu_seqlens_k_new): variable-length appends, k, v packed as
    [total_new, Hkv, D] with stream b's rows at [cu_seqlens[b], cu_seqlens[b+1]), written at keys cache_seqlens[b] ..
    under the same rules, in every cache format and one launch (svgb_kvcache_append_varlen)."""
    who = "kvcache_append"
    packed = cu_seqlens is not None
    _need_cuda(k_cache, v_cache, k, v)
    if k_cache.dim() != 4 or k.dim() != (3 if packed else 4) or k_cache.shape != v_cache.shape or k.shape != v.shape:
        raise SvgbError(f"{who}: {'with cu_seqlens, ' if packed else ''}k_cache, v_cache {tuple(k_cache.shape)} must "
                        f"be [blocks, rows, Hkv, D] and k, v {tuple(k.shape)} "
                        f"{'[total_new, Hkv, D]' if packed else '[B, Snew, Hkv, D]'}, each pair of one shape")
    if k.shape[-2:] != k_cache.shape[2:]:
        raise SvgbError(f"{who}: k {tuple(k.shape)} and k_cache {tuple(k_cache.shape)} differ in heads or D")
    if packed:
        cu = _cu_seqlens(who, "cu_seqlens", cu_seqlens, None, k.device)
        B = cu.numel() - 1
    else:
        B = k.shape[0]
    scales, per_row = _cache_format(who, k_cache, v_cache, k_scale, v_scale)
    if k.dtype != v.dtype or (scales is None and k.dtype != k_cache.dtype):
        raise SvgbError(f"{who}: the new rows k, v must share one dtype, and with a 16-bit cache the cache's")
    dt = _dt(k)
    N, Hkv, D = k.shape[-3:]  # new rows per stream, or packed rows
    if N == 0:
        return
    for c in (k_cache, v_cache):
        if not _addressable(c.transpose(1, 2), "bhsd"):
            raise SvgbError(f"{who}: the cache is written in place, so it must be 16-byte aligned with a last "
                            "stride of 1 and other strides that are nonzero multiples of 8 elements")
    layout = "shd" if packed else "bhsd"
    k, v = (_addressed(t if packed else t.transpose(1, 2), layout) for t in (k, v))
    bt, bi, max_pages = _cache_layout(B, block_table, cache_batch_idx)
    lens = _seqlens(cache_seqlens, B, k.device)
    fill = 8 if scales is None else 16  # e4m3 cache strides are multiples of 16 bytes
    sc = tuple(t.data_ptr() for t in scales or ())
    if packed:  # one entry for every format: the scales (or none) and which format they are
        name, bounds, sc = "svgb_kvcache_append_varlen", (cu.data_ptr(),), (sc or (None, None)) + (int(per_row),)
    else:
        name, bounds = "svgb_kvcache_append" + ("" if scales is None else "_e4m3_rows" if per_row else "_e4m3"), ()
    check(getattr(lib(), name)(k_cache.data_ptr(), v_cache.data_ptr(), k.data_ptr(), v.data_ptr(), *bounds,
                               lens.data_ptr(), _p(bi), _p(bt), dt, B, N, Hkv, D, k_cache.shape[0], k_cache.shape[1],
                               max_pages, _st(k_cache.transpose(1, 2), "bhsd", fill),
                               _st(v_cache.transpose(1, 2), "bhsd", fill), _st(k, layout), _st(v, layout), *sc,
                               _stream(k)), name)
    _bump()


def _cache_format(who, k_cache, v_cache, k_scale, v_scale):
    """(scales, per_row) of a KV cache [num_blocks, block_rows, Hkv, D]: (None, False) for a 16-bit cache, which takes
    no scales; for a float8_e4m3fn cache its (k_scale, v_scale), per cache row when either is 3-D (_row_scales, per_row
    True), else per key/value head (_fp8_scales)."""
    if v_cache.dtype != k_cache.dtype:
        raise SvgbError(f"{who}: k_cache ({k_cache.dtype}) and v_cache ({v_cache.dtype}) must share one dtype")
    if k_cache.dtype != torch.float8_e4m3fn:
        if k_scale is not None or v_scale is not None:
            raise SvgbError(f"{who}: k_scale / v_scale are for float8_e4m3fn caches; a {k_cache.dtype} cache takes none")
        return None, False
    rows = _row_scales(who, k_scale, v_scale, k_cache)
    return rows or _fp8_scales(who, k_scale, v_scale, k_cache.shape[2]), rows is not None


def _fp8_scales(who, k_scale, v_scale, Hkv):
    """The per-KV-head dequantisation scales of an e4m3 cache: both float32 device tensors [Hkv]."""
    if k_scale is None or v_scale is None:
        raise SvgbError(f"{who}: a float8_e4m3fn cache needs k_scale and v_scale (float32 [Hkv], one scale per key/value "
                        "head)")
    for name, t in (("k_scale", k_scale), ("v_scale", v_scale)):
        if not isinstance(t, torch.Tensor) or t.dtype != torch.float32 or tuple(t.shape) != (Hkv,):
            shown = tuple(t.shape) if isinstance(t, torch.Tensor) else type(t).__name__
            raise SvgbError(f"{who}: {name} must be a float32 tensor [Hkv={Hkv}] per head, or [num_blocks, Hkv, "
                            f"block_rows] per row (got {shown}{', ' + str(t.dtype) if isinstance(t, torch.Tensor) else ''})")
    _need_cuda(k_scale, v_scale)
    return k_scale.contiguous(), v_scale.contiguous()


def _row_scales(who, k_scale, v_scale, cache):
    """The per-row scales of an e4m3 cache [num_blocks, block_rows, Hkv, D]: (k_scale, v_scale) when either is 3-D, both
    then float32 device tensors [num_blocks, Hkv, block_rows], contiguous (written in place), with D = 128 and block_rows
    a multiple of 4; None for the per-head format ([Hkv], checked by _fp8_scales)."""
    if not any(isinstance(t, torch.Tensor) and t.dim() == 3 for t in (k_scale, v_scale)):
        return None
    nb, rows, Hkv, D = cache.shape
    want = (nb, Hkv, rows)
    for name, t in (("k_scale", k_scale), ("v_scale", v_scale)):
        if not isinstance(t, torch.Tensor) or t.dim() != 3:
            raise SvgbError(f"{who}: k_scale and v_scale mix formats: per-row scales [num_blocks, Hkv, block_rows] go "
                            f"with per-row scales, not {tuple(t.shape) if isinstance(t, torch.Tensor) else t!r}")
        if t.dtype != torch.float32 or tuple(t.shape) != want or not t.is_contiguous():
            raise SvgbError(f"{who}: per-row {name} must be a contiguous float32 tensor [num_blocks, Hkv, block_rows]="
                            f"{list(want)} (got {tuple(t.shape)}, {t.dtype})")
    if D != 128 or rows % 4:
        raise SvgbError(f"{who}: per-row scales need head_dim 128 (got {D}) and block_rows a multiple of 4 (got {rows})")
    _need_cuda(k_scale, v_scale)
    return k_scale, v_scale


def plan_kvcache(cache_seqlens, *, q_len: Optional[int] = None, num_blocks: int, new_len: int = 0,
                 cache_len: Optional[int] = None, block_table: Optional[torch.Tensor] = None,
                 page_size: Optional[int] = None, cache_batch_idx: Optional[torch.Tensor] = None, causal: bool = False,
                 window_size=(-1, -1), sink: int = 0, num_splits: int = 1, num_heads: Optional[int] = None,
                 block: int = 0, first_block: Optional[int] = None, cu_seqlens_q: Optional[torch.Tensor] = None,
                 total_q: Optional[int] = None, max_seqlen_q: Optional[int] = None,
                 cu_seqlens_new: Optional[torch.Tensor] = None) -> AttnPlan:
    """Attention of B streams of q_len queries into a KV cache, in FlashAttention's conventions
    (flash_attn_with_kvcache): stream b holds L_b = cache_seqlens[b] + new_len keys (new_len rows appended before this
    attention, e.g. by kvcache_append) and its query i sits at logical position L_b - q_len + i.  Query p sees key kv
    when kv < sink, or when kv lies at most window_size[0] positions behind p and at most window_size[1] ahead (-1:
    unbounded); causal=True sets the right window to 0 and conflicts with a positive window_size[1].
    The cache is k_cache.shape[0] = num_blocks blocks: contiguous, cache_len = S_cache rows each (stream b in block
    cache_batch_idx[b], default b), or paged, page_size rows each (a multiple of 128) with block_table int [B, max_pages].
    cache_seqlens: int or device int tensor [B]; nothing is read on the host.  attn_fwd runs the plan on q [B, q_len, Hq,
    D] and the cache, any Hq = G * Hkv; it has no backward (attention() under grad and key_major() raise).
    num_splits: 1 is the single pass, one CTA per 256-query item and head.  n > 1 splits every item's keys into n pieces
    (svgb_attn_plan_kvcache_split), which attn_fwd runs as n times the CTAs writing fp32 partials and a merge, so that
    decode and short chunks fill the GPU.  0 picks n on the host from the SM count, the CTAs B ceil(q_len / 256)
    num_heads (num_heads = q's heads, required then) and the chunk slots per item (kvcache_num_splits).
    block > 0: the block-causal rule of plan_block_causal on logical positions (blocks of `block` keys, the first ends at
    `first_block`, default block): query p sees kv < sink and e(p) - W <= kv < e(p), with W = window_size[0] counted
    back from the block end (-1: unbounded) and window_size[1] = -1; causal=True is refused (the rule is causal).  When
    the q_len queries form one block, they all attend [L_b - W, L_b) plus the sinks.  A rolling cache that renumbers its
    positions down by d keys keeps its blocks with first_block = ((F - d - 1) mod block) + 1 (INTEGRATION.md).
    Variable-length queries (FlashAttention 3's cu_seqlens_q, in place of q_len): cu_seqlens_q device int [B + 1], stream
    b's Lq_b = cu_seqlens_q[b+1] - cu_seqlens_q[b] queries are packed rows [cu_seqlens_q[b], cu_seqlens_q[b+1]) of q
    [total_q, Hq, D], and its query i sits at L_b - Lq_b + i; total_q (q.shape[0]) is required and max_seqlen_q, the
    longest Lq_b when known, tightens the plan's item bound (a stream longer than it gives an unspecified result).
    cu_seqlens_new, device int [B + 1], gives the rows appended before this attention per stream (kvcache_append(...,
    cu_seqlens=)) in place of new_len.  Every mask rule, num_splits and block= work as above, with one (block,
    first_block) for the batch; Lq_b = 0 is legal.  attn_fwd then takes q [total_q, Hq, D] and returns o [total_q, Hq,
    D] and lse [Hq, total_q].  Nothing is read on the host (svgb_attn_plan_kvcache_varlen)."""
    who = "plan_kvcache"
    if (q_len is None) == (cu_seqlens_q is None):
        raise SvgbError(f"{who}: pass q_len (B streams of q_len queries) or cu_seqlens_q (variable-length queries), "
                        "exactly one of them")
    if cu_seqlens_new is not None and cu_seqlens_q is None:
        raise SvgbError(f"{who}: cu_seqlens_new (variable-length appends) goes with cu_seqlens_q; uniform plans take "
                        "new_len")
    # geometry: rows per cache block and a stream's capacity, the streams B, the device, and the longest query run Qmax
    # of a stream
    if block_table is not None:
        if page_size is None:
            raise SvgbError(f"{who}: a paged cache (block_table) needs page_size")
        rows = int(page_size)
        cap = block_table.shape[1] * rows
    else:
        if cache_len is None:
            raise SvgbError(f"{who}: a contiguous cache needs cache_len (its rows per stream, k_cache.shape[1])")
        rows = cap = int(cache_len)
    cu_q = cu_new = None
    if cu_seqlens_q is not None:
        if total_q is None:
            raise SvgbError(f"{who}: cu_seqlens_q needs total_q (q.shape[0], the packed query rows), which is passed "
                            "rather than read from the device")
        if cu_seqlens_new is not None and int(new_len):
            raise SvgbError(f"{who}: cu_seqlens_new and new_len={new_len} both give the appended rows; pass one")
        cu_q = _cu_seqlens(who, "cu_seqlens_q", cu_seqlens_q, None, None)
        B, device = cu_q.numel() - 1, cu_q.device
        Sq = int(total_q)  # the plan runs as one block of total_q packed rows
        if Sq < 1:
            raise SvgbError(f"{who}: total_q={Sq} must be >= 1")
        Qmax = Sq if max_seqlen_q is None else int(max_seqlen_q)
        if not 1 <= Qmax <= Sq:
            raise SvgbError(f"{who}: max_seqlen_q={Qmax} must lie in [1, total_q={Sq}]")
        if cu_seqlens_new is not None:
            cu_new = _cu_seqlens(who, "cu_seqlens_new", cu_seqlens_new, B, device)
    else:
        Sq = Qmax = int(q_len)
        if block_table is not None:
            B = block_table.shape[0]
        elif isinstance(cache_seqlens, torch.Tensor):
            B = cache_seqlens.numel()
        elif cache_batch_idx is not None:
            B = cache_batch_idx.numel()
        else:
            raise SvgbError(f"{who}: with an int cache_seqlens pass a tensor or cache_batch_idx for B")
        device = (cache_seqlens if isinstance(cache_seqlens, torch.Tensor) else
                  block_table if block_table is not None else cache_batch_idx).device
    # mask: a local band (left, right), or block-causal (W, C, F) whose chunk slots are bounded as the band
    # (left = W - 1, right = C - 1, svgb_attn_plan_kvcache_block); -1 is unbounded, no query position lying further than
    # cap + Qmax from a key, nor a query's block end further than cap + Qmax + C from key 0
    sink = int(sink)
    if block:
        if causal:
            raise SvgbError(f"{who}: causal=True is redundant with block= (the block rule is causal); pass "
                            "window_size=(W, -1)")
        W, right = (int(w) for w in window_size)
        if right != -1:
            raise SvgbError(f"{who}: with block=, window_size[1] = {right} must be -1 (no key past the block end)")
        m1, W = _block_m1(who, block, first_block, W, sink)
        C_, F = m1 & 0xffff, (m1 & 0xffff) - (m1 >> 16)
        if W == -1:
            W = min(cap + Qmax + C_, 2**31 - 1)
        left, right = W - 1, C_ - 1
    else:
        left, right = (int(w) for w in window_size)
        if causal:
            if right > 0:
                raise SvgbError(f"{who}: causal=True looks no key ahead, but window_size[1] = {right}")
            right = 0
        left, right = (min(cap + Qmax, 2**31 - 1) if w == -1 else w for w in (left, right))
    # the items of the single pass: B ceil(Sq / 256), or for packed queries the bound I of
    # svgb_attn_plan_kvcache_varlen_bytes
    items = B * -(-Sq // 256) if cu_q is None else min(B * -(-Qmax // 256), (Sq + 255 * B) // 256)
    n = _num_splits(num_splits, num_heads, items, cap, sink, left, right)
    bt, bi, max_pages = _cache_layout(B, block_table, cache_batch_idx)
    lens = _seqlens(cache_seqlens, B, device)
    if cu_q is not None and lens.device != device:
        raise SvgbError(f"{who}: cache_seqlens is on {lens.device}, cu_seqlens_q on {device}")
    # the planner pair: the _bytes query takes (sizes, cap, sink, mask), the planner (bounds, sizes, [Snew,] cache
    # geometry, sink, mask), the mask ending in n on every entry but the single local one
    if cu_q is not None:
        name, bounds, sizes, new = "svgb_attn_plan_kvcache_varlen", (cu_q, lens, cu_new), (B, Sq, Qmax), ()
        mask = (0, 0, W, C_, F, n) if block else (left, right, 0, 0, 0, n)
    else:
        bounds, sizes, new = (lens,), (B, Sq), (int(new_len),)
        if block:
            name, mask = "svgb_attn_plan_kvcache_block", (W, C_, F, n)
        elif n == 1:
            name, mask = "svgb_attn_plan_kvcache", (left, right)
        else:
            name, mask = "svgb_attn_plan_kvcache_split", (left, right, n)
    nbytes = C.c_size_t()
    check(getattr(lib(), name + "_bytes")(*sizes, cap, sink, *mask, C.byref(nbytes)), name + "_bytes")
    ws = torch.empty(nbytes.value, dtype=torch.uint8, device=device)  # owned by the plan, with its copy of the lengths
    desc = Plan()
    check(getattr(lib(), name)(*(_p(t) for t in bounds), _p(bi), _p(bt), *sizes, *new, int(num_blocks), rows,
                               max_pages, sink, *mask, ws.data_ptr(), ws.numel(), C.byref(desc),
                               torch.cuda.current_stream(device).cuda_stream), name)
    _bump()
    # attn_fwd runs a variable-length plan as one block of total_q packed rows
    return AttnPlan(desc, ws, (B, Sq) if cu_q is None else (1, Sq))


def _cu_seqlens(who, name, cu, B, device) -> torch.Tensor:
    """A cu_seqlens argument as device int32 [B + 1] (B None: any B >= 1), refused by name before any launch."""
    if not isinstance(cu, torch.Tensor):
        raise SvgbError(f"{who}: {name} must be a device int tensor [B + 1] (got {type(cu).__name__})")
    if not cu.is_cuda:
        raise SvgbError(f"{who}: {name} is on the CPU; variable-length KV-cache plans and appends read their bounds on "
                        "the device only (no host read), so pass a CUDA tensor")
    if cu.dim() != 1 or cu.numel() < 2 or (B is not None and cu.numel() != B + 1) or cu.is_floating_point():
        want = "B + 1 >= 2" if B is None else f"B + 1 = {B + 1}"
        raise SvgbError(f"{who}: {name} must be a 1-D int tensor of {want} entries (got {tuple(cu.shape)}, {cu.dtype})")
    if device is not None and cu.device != device:
        raise SvgbError(f"{who}: {name} is on {cu.device}, the other tensors on {device}")
    return cu.to(torch.int32).contiguous()


def _num_splits(num_splits, num_heads, items, cap, sink, left, right):
    """The split count n of a plan whose single pass has `items` 256-query items per head (num_splits=0: automatic)."""
    n = int(num_splits)
    if n < 0:
        raise SvgbError(f"plan_kvcache: num_splits={n} must be >= 0 (0: automatic, 1: no split)")
    if n == 0:
        if num_heads is None:
            raise SvgbError("plan_kvcache: num_splits=0 picks the split count from the grid, so it needs num_heads (q's "
                            "query heads)")
        n = kvcache_num_splits(items * int(num_heads), _kvcache_slots(cap, sink, left, right), _sm_count())
    return n


# The automatic split count of plan_kvcache(num_splits=0), from tools/kvcache_perf.py on the H100 (DESIGN.md): split only
# while the single pass leaves SMs idle, into the fewest splits whose grid fills its last wave to _SPLIT_WAVE_FILL (or,
# when no count does, the most that fit in one wave), with at least _SPLIT_MIN_SLOTS chunk slots per split and at most
# _SPLIT_MAX splits (the merge reads every split).
_SPLIT_WAVE_FILL, _SPLIT_MIN_SLOTS, _SPLIT_MAX = 0.85, 4, 32


def kvcache_num_splits(ctas: int, slots: int, num_sms: int) -> int:
    """Split count for a KV-cache attention of `ctas` single-pass CTAs (B ceil(Sq / 256) Hq) whose items have `slots`
    chunk slots, on `num_sms` SMs (the kernel fits one CTA per SM): 1 once the single pass fills the machine."""
    if ctas >= num_sms:
        return 1
    top = min(_SPLIT_MAX, slots // _SPLIT_MIN_SLOTS)
    for n in range(2, top + 1):
        waves = -(-n * ctas // num_sms)
        if n * ctas >= _SPLIT_WAVE_FILL * waves * num_sms:
            return n
    return max(1, min(top, num_sms // ctas))


def _kvcache_slots(cap, sink, left, right):
    """Chunk slots per item of a KV-cache plan (include/svgb200.h, svgb_attn_plan_kvcache_bytes)."""
    return min(-(-cap // 128), -(-sink // 128) + (255 + left + right) // 128 + 2)


_sms: Optional[int] = None


def _sm_count() -> int:
    global _sms
    if _sms is None:
        _sms = device_check()[2]
    return _sms


def _is_profiling(mask_mode: int) -> bool:
    """The SVG1 profiling masks (modes 4-9): band plans the forward runs and the backward does not."""
    return MASK_PROF_HY_S <= mask_mode <= MASK_PROF_COG_T


# ----------------------------------------------------------------------------------------------
# attention
# ----------------------------------------------------------------------------------------------
def _geometry(q, layout):
    if layout == "bhsd":
        B, H, S, D = q.shape
        return B * H, S, D, D, S * D
    if layout == "shd":
        S, H, D = q.shape
        return H, S, D, H * D, D
    raise SvgbError(f"unknown layout {layout}")


def _kv_geometry(q, k, layout):
    """(BH, Sq, Skv, D, q strides, k/v strides), BH counting q's heads.  k's sequence length may differ from q's, and
    its head count (dim 1 in both layouts) may be q's divided by a whole G = _kv_group(q, k) (grouped-query attention:
    query head h attends with key/value head h // G); every other dimension must match."""
    BH, Sq, D, qrs, qhs = _geometry(q, layout)
    if q.dim() != k.dim():
        raise SvgbError(f"q {tuple(q.shape)} and k {tuple(k.shape)} differ in rank")
    BHk, Skv, Dk, kvrs, kvhs = _geometry(k, layout)
    seq = 2 if layout == "bhsd" else 0
    if ([n for i, n in enumerate(q.shape) if i not in (seq, 1)] != [n for i, n in enumerate(k.shape) if i not in (seq, 1)]
            or k.shape[1] == 0 or q.shape[1] % k.shape[1]):
        raise SvgbError(f"q {tuple(q.shape)} and k, v {tuple(k.shape)} may differ in the sequence length only, and "
                        "in a key/value head count that divides q's (grouped-query attention)")
    return BH, Sq, Skv, D, (qrs, qhs), (kvrs, kvhs)


def _kv_group(q, k):
    """Query heads per key/value head, once _kv_geometry has accepted q and k."""
    return q.shape[1] // k.shape[1]


def _strides(t, layout, fill=8):
    """(batch, head, row) element strides of an attention operand, as the strided entries take them; 'shd' is one batch
    element.  A dimension of extent 1 is never stepped, so a stride there that the ABI would refuse is replaced by fill:
    8 elements for the 16-bit entries, 16 (bytes) for the e4m3 ones."""
    if layout == "bhsd":
        n, st = t.shape[:3], t.stride()[:3]
    else:
        n, st = (1, t.shape[1], t.shape[0]), (t.shape[1] * t.stride(1), t.stride(1), t.stride(0))
    return tuple(fill if e == 1 and not (x and x % fill == 0) else x for e, x in zip(n, st))


def _addressable(t, layout):
    """True when the strided entries (svgb_attn_fwd_strided / svgb_attn_bwd_strided) read or write t in place: the
    last stride is 1, the base 16-byte aligned and the (batch, head, row) strides nonzero multiples of 8 elements."""
    return t.stride(-1) == 1 and t.data_ptr() % 16 == 0 and all(x and x % 8 == 0 for x in _strides(t, layout))


def _addressed(t, layout):
    """t itself when the strided entries can read it, otherwise a contiguous copy (a zero stride such as the expanded
    gradient of o.sum(), a misaligned view, a last stride other than 1).  A clone rather than .contiguous(), which
    would return a misaligned contiguous tensor itself."""
    return t if _addressable(t, layout) else t.clone(memory_format=torch.contiguous_format)


def _st(t, layout, fill=8):
    return (C.c_longlong * 3)(*_strides(t, layout, fill))


def _attn(q, k, v, o, plan, layout, dtype, scales, rows, return_lse, sm_scale):
    """One attention launch.  Operands that are not all contiguous take svgb_attn_fwd_strided, each at its own strides
    (_addressable): 16-bit, no scales, no row vectors, no gather plan.  Otherwise fewer key/value heads than query
    heads (G > 1) take svgb_attn_fwd_gqa: 16-bit, no scales, no row vectors, no gather plan.  Otherwise equal sequence
    lengths take svgb_attn_fwd: 16-bit or e4m3 (dtype) with its per-head scales, and the row vectors rows = (q_rows,
    kv_rows, o_rows); other lengths svgb_attn_fwd_kv: q and o over Sq rows, k and v over Skv rows, each pair with its
    own strides; 16-bit, no scales, no row vectors."""
    BH, Sq, Skv, D, qs, kvs = _kv_geometry(q, k, layout)
    G = _kv_group(q, k)
    if G > 1:
        _gqa_check(dtype, plan, rows)
    lse = torch.empty(BH, Sq, dtype=torch.float32, device=q.device) if return_lse else None
    scale = float(D) ** -0.5 if sm_scale is None else float(sm_scale)
    if not all(t.is_contiguous() for t in (q, k, v, o)):
        B = q.shape[0] if layout == "bhsd" else 1
        check(lib().svgb_attn_fwd_strided(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), _p(lse), dtype, B,
                                          q.shape[1], k.shape[1], Sq, Skv, D, *(_st(t, layout) for t in (q, k, v, o)),
                                          scale, C.byref(plan.desc), plan.ws.data_ptr(), _stream(q)),
              "svgb_attn_fwd_strided")
    elif G > 1:
        check(lib().svgb_attn_fwd_gqa(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), _p(lse), dtype, BH,
                                      BH // G, Sq, Skv, D, *qs, *kvs, *qs, scale, C.byref(plan.desc),
                                      plan.ws.data_ptr(), _stream(q)), "svgb_attn_fwd_gqa")
    elif Sq == Skv:
        rows = [None if r is None else r.reshape(BH, Sq).to(torch.int32).contiguous() for r in rows]
        check(lib().svgb_attn_fwd(q.data_ptr(), k.data_ptr(), v.data_ptr(), *map(_p, scales), o.data_ptr(), _p(lse),
                                  *map(_p, rows), dtype, BH, Sq, D, *qs, *qs, scale, C.byref(plan.desc),
                                  plan.ws.data_ptr(), _stream(q)), "svgb_attn_fwd")
    else:
        check(lib().svgb_attn_fwd_kv(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), _p(lse), dtype, BH, Sq,
                                     Skv, D, *qs, *kvs, *qs, scale, C.byref(plan.desc), plan.ws.data_ptr(), _stream(q)),
              "svgb_attn_fwd_kv")
    _bump()
    return (o, lse) if return_lse else o


def _gqa_check(dtype, plan, rows=()):
    """What grouped-query attention does not take, refused before any device work."""
    if dtype == _E4M3:
        raise SvgbError("grouped-query attention (fewer k, v heads than q heads) has no FP8 path: the per-head scales "
                        "are indexed by query head")
    if any(r is not None for r in rows):
        raise SvgbError("grouped-query attention (fewer k, v heads than q heads) takes no row vectors "
                        "(o_rows / q_rows / kv_rows)")
    if plan.desc.kind == PLAN_GATHER:
        raise SvgbError("grouped-query attention (fewer k, v heads than q heads) takes no gather plan: its kv_rows are "
                        "indexed by query head")


def attn_fwd(q, k, v, plan: AttnPlan, *, layout: str = "bhsd", o_rows: Optional[torch.Tensor] = None,
             q_rows: Optional[torch.Tensor] = None, kv_rows: Optional[torch.Tensor] = None,
             return_lse: bool = False, sm_scale: Optional[float] = None, out: Optional[torch.Tensor] = None,
             k_scale: Optional[torch.Tensor] = None, v_scale: Optional[torch.Tensor] = None):
    """layout 'bhsd': q,k,v [B,H,S,D];  'shd': [S,H,D] (ops API).  q, k, v may be views ([B, S, H, D] passed as
    x.transpose(1, 2), one of a packed projection's unbind(2), every other head, a batch slice): they are read in place
    when their last stride is 1, their base 16-byte aligned and their other strides nonzero multiples of 8 elements,
    and copied with .contiguous() otherwise.  o is torch.empty_like(q), so it keeps a view's memory order; out= may be
    a view too, and only its elements are written.
    o_rows scatters the output rows; q_rows / kv_rows gather the input rows and need a gather plan
    (plan_varblock(..., gather=True)); all three are int [BH,S] (include/svgb200.h, svgb_attn_fwd).  Row vectors and
    gather plans take contiguous q, k, v and out only.
    k, v may have another sequence length S_kv than q (same batch, heads, D and dtype): the plan is then a rectangular
    variable-block plan (plan_varblock(..., S_kv=)), o has q's shape, and row vectors are not taken.
    k, v may have fewer heads than q, Hq = G * Hkv (grouped-query attention, FlashInfer's mapping: query head h attends
    with key/value head h // G): a variable-block plan is then built over the B * Hkv key/value heads and shared by
    each group, band plans are shared by every head already; no row vectors, FP8 or gather plans.
    k_scale, v_scale: the scales of float8_e4m3fn caches under a KV-cache plan, per key/value head [Hkv] or per cache row
    [num_blocks, Hkv, block_rows] (see _attn_kvcache)."""
    _need_cuda(q, k, v)
    if plan.desc.kind in (PLAN_KVCACHE, PLAN_KVCACHE_SPLIT):
        if any(r is not None for r in (q_rows, kv_rows, o_rows)):
            raise SvgbError("a KV-cache plan (plan_kvcache) takes no row vectors (o_rows / q_rows / kv_rows)")
        return _attn_kvcache(q, k, v, plan, return_lse, sm_scale, out, k_scale, v_scale)
    if k_scale is not None or v_scale is not None:
        raise SvgbError("k_scale / v_scale are for float8_e4m3fn caches under a KV-cache plan (plan_kvcache); other "
                        "FP8 attention takes attn_fwd_fp8")
    rows = (q_rows, kv_rows, o_rows)
    if any(r is not None for r in rows) or plan.desc.kind == PLAN_GATHER:
        # the row vectors and the row-gather kernel index one flat [BH, S, D] stride pair
        if not (q.is_contiguous() and k.is_contiguous() and v.is_contiguous()):
            raise SvgbError("q, k, v must be contiguous")
        if out is not None and not out.is_contiguous():
            raise SvgbError("out must be contiguous with row vectors or a gather plan")
    else:
        q, k, v = (_addressed(t, layout) for t in (q, k, v))
    if not (q.dtype == k.dtype == v.dtype) or k.shape != v.shape:
        raise SvgbError("q, k, v must share dtype, and k, v their shape")
    if out is not None and (out.shape != q.shape or out.dtype != q.dtype):
        raise SvgbError(f"out {tuple(out.shape)} {out.dtype} must have q's shape and dtype")
    o = torch.empty_like(q) if out is None or not _addressable(out, layout) else out
    if q.shape[1] == k.shape[1] and q.shape != k.shape and any(r is not None for r in rows):
        raise SvgbError("row vectors (o_rows / q_rows / kv_rows) need k, v of q's sequence length")
    res = _attn(q, k, v, o, plan, layout, _dt(q), (None, None, None), rows, return_lse, sm_scale)
    if out is None or o is out:
        return res
    out.copy_(o)  # an out= the kernels cannot address
    return (out, res[1]) if return_lse else out


def _attn_kvcache(q, k_cache, v_cache, plan, return_lse, sm_scale, out, k_scale=None, v_scale=None):
    """attn_fwd under a KV-cache plan: q [B, Sq, Hq, D] (variable-length plans: [total_q, Hq, D]) as R = B * Sq
    (total_q) packed rows, the cache [blocks, rows, Hkv, D] as blocks * rows rows (both views); returns o of q's shape
    (out itself when given) and lse [B, Hq, Sq] ([Hq, total_q]), flash_attn_with_kvcache's shapes.  A split plan runs as
    two launches, the attention into fp32 partials in a cached workspace and their merge into o.
    float8_e4m3fn caches (FP8 KV cache) take bf16 q, D = 128 and k_scale, v_scale, and o is bf16.  With per-head scales
    [Hkv] q is quantised per query head over the call's R rows (quantize_e4m3 on a transposed [Hq, R, D] copy), with
    per-row scales [num_blocks, Hkv, block_rows] each q row on its own (quantize_e4m3_rows, read in place)."""
    if q.dim() not in (3, 4) or k_cache.dim() != 4 or k_cache.shape != v_cache.shape:
        raise SvgbError(f"a KV-cache plan takes q [B, Sq, Hq, D] or [total_q, Hq, D] (got {tuple(q.shape)}) and "
                        f"k_cache, v_cache [blocks, rows, Hkv, D] of one shape (got {tuple(k_cache.shape)}, "
                        f"{tuple(v_cache.shape)})")
    nb, rows, Hkv, Dc = k_cache.shape
    if nb * rows != plan.S_kv:
        raise SvgbError(f"the KV-cache plan was built for {plan.S_kv} cache rows, the cache {tuple(k_cache.shape)} has "
                        f"{nb * rows}")
    fp8 = k_cache.dtype == torch.float8_e4m3fn
    Hq, D = q.shape[-2:]
    if fp8:
        if q.dtype != torch.bfloat16:
            raise SvgbError(f"an FP8 KV cache takes bf16 q (got {q.dtype}); it is quantised here, and the output is "
                            "bf16")
        if D != 128 or Dc != 128:
            raise SvgbError(f"an FP8 KV cache needs head_dim 128 (got q {D}, cache {Dc}): 64-byte e4m3 rows have no "
                            "128-byte swizzle")
    elif q.dtype != k_cache.dtype:
        raise SvgbError("q and the caches must share one dtype")
    if D != Dc or not Hkv or Hq % Hkv:
        raise SvgbError(f"q {tuple(q.shape)} and the cache {tuple(k_cache.shape)} differ in D, or q's {Hq} heads are "
                        f"not a multiple of the cache's {Hkv} key/value heads")
    o_dtype = torch.bfloat16 if fp8 else q.dtype
    if out is not None and (out.shape != q.shape or out.dtype != o_dtype):
        raise SvgbError(f"out {tuple(out.shape)} {out.dtype} must have q's shape and dtype{' bf16' if fp8 else ''}")
    scales, per_row = _cache_format("attn_fwd on a KV cache", k_cache, v_cache, k_scale, v_scale)
    if needs_grad(q, k_cache, v_cache):
        raise SvgbError("attention into a KV cache has no backward: the KV-cache plan (plan_kvcache) runs forward only")
    B, Sq = plan.source
    varlen = plan.desc.varlen_items > 0
    if varlen and (q.dim() != 3 or q.shape[0] != Sq):
        raise SvgbError(f"a variable-length KV-cache plan for total_q={Sq} query rows takes q [total_q, Hq, D] (got "
                        f"{tuple(q.shape)})")
    if not varlen and (q.dim() != 4 or q.shape[:2] != (B, Sq)):
        raise SvgbError(f"a KV-cache plan for B={B} streams of Sq={Sq} queries takes q [B, Sq, Hq, D] (got "
                        f"{tuple(q.shape)})")
    R = B * Sq
    # the q operand and its (batch, head, row) strides; the cache as [nb * rows, Hkv, D] views, e4m3 read in place
    if scales is None:
        dt, fill = _dt(q), 8
        qa = _addressed(q.reshape(R, Hq, D), "shd")
        q_st = _st(qa, "shd")
        kf, vf = (_addressed(c.flatten(0, 1), "shd") for c in (k_cache, v_cache))
    else:
        dt, fill = _E4M3, 16
        if per_row:
            qa, q_scale = quantize_e4m3_rows(q.reshape(R, Hq, D))
            q_st = _st(qa, "shd", 16)
        else:  # [Hq, R, D]: one batch element of the scale kernel's [heads, rows, D]
            qa, q_scale = quantize_e4m3(q.reshape(R, Hq, D).transpose(0, 1).contiguous())
            q_st = _st(qa[None], "bhsd", 16)
        scales = (q_scale, *scales)
        kf, vf = (c.flatten(0, 1).view(torch.uint8) for c in (k_cache, v_cache))
    lse = torch.empty(Hq, R, dtype=torch.float32, device=q.device) if return_lse else None
    scale = float(D) ** -0.5 if sm_scale is None else float(sm_scale)
    split = plan.desc.kind == PLAN_KVCACHE_SPLIT
    if split:  # the merge writes a contiguous out= in place
        o = (out.view(R, Hq, D) if out is not None and out.is_contiguous() else
             torch.empty(R, Hq, D, dtype=o_dtype, device=q.device))
        n = plan.desc.max_items // (plan.desc.varlen_items or B * -(-Sq // 256))
        nbytes = C.c_size_t()
        check(lib().svgb_attn_fwd_kvcache_split_bytes(n, R, Hq, D, C.byref(nbytes)),
              "svgb_attn_fwd_kvcache_split_bytes")
        buf = workspace("kvcache_split", nbytes.value, q.device)
        name = "svgb_attn_fwd_kvcache_split"
        args = (*map(_p, scales or (None,) * 3), o.data_ptr(), _p(lse), dt, int(per_row), B, Hq, Hkv, Sq, nb, rows, D)
        ws = (buf.data_ptr(), buf.numel())
    else:
        o = torch.empty_like(qa) if scales is None else torch.empty(R, Hq, D, dtype=o_dtype, device=q.device)
        ws = ()
        if scales is None:  # q, o as one batch element, each at its own strides
            name, args = "svgb_attn_fwd_strided", (o.data_ptr(), _p(lse), dt, 1, Hq, Hkv, R, nb * rows, D)
        elif per_row:
            name, args = "svgb_attn_fwd_kvcache_e4m3_rows", (*map(_p, scales), o.data_ptr(), _p(lse), Hq, Hkv, R, nb,
                                                              rows, D)
        else:
            name, args = "svgb_attn_fwd_strided_e4m3", (*map(_p, scales), o.data_ptr(), _p(lse), 1, Hq, Hkv, R,
                                                         nb * rows, D)
    check(getattr(lib(), name)(qa.data_ptr(), kf.data_ptr(), vf.data_ptr(), *args, q_st, _st(kf, "shd", fill),
                               _st(vf, "shd", fill), _st(o, "shd"), scale, C.byref(plan.desc), plan.ws.data_ptr(), *ws,
                               _stream(q)), name)
    _bump(2 if split else 1)
    if out is None:
        o = o.view(q.shape)
    else:
        if o.data_ptr() != out.data_ptr():
            out.copy_(o.view(out.shape))  # an out= the kernels did not write
        o = out
    if not return_lse:
        return o
    return o, lse if varlen else lse.view(Hq, B, Sq).transpose(0, 1)


def attn_bwd(q, k, v, o, do, lse, plan: AttnPlan, *, layout: str = "bhsd", sm_scale: Optional[float] = None,
             out: Optional[tuple] = None):
    """Gradients (dq, dk, dv) of o = attn_fwd(q, k, v, plan, layout=layout, sm_scale=sm_scale) for the output gradient
    do; lse is the forward's return_lse output.  Variable-block and band plans (mask NONE / HY / WAN / COG / LOCAL); the plan's
    key-major companion is built on the first call (AttnPlan.key_major).  Deterministic: two calls give the same bits.
    k, v may have another sequence length than q under a rectangular variable-block plan, and fewer heads (grouped-query
    attention, as attn_fwd); dk, dv then have k's shape, a group's dk and dv summing over its query heads.
    Every tensor may be a view, as in attn_fwd: q, k, v, o, do are read in place where the strided entry can address
    them and copied with .contiguous() otherwise (do with a zero stride, for instance).
    out: optional (dq, dk, dv) tensors of q's, k's and v's dtype and shape, written and returned instead of new ones;
    each may be a view, whose every element is written and nothing outside it.  Without out, dq, dk, dv are
    torch.empty_like(q / k / v) and keep the inputs' memory order."""
    _need_cuda(q, k, v, o, do, lse)
    if out is not None and len(out) != 3:
        raise SvgbError("out must be a (dq, dk, dv) tuple")
    q, k, v, o, do = (_addressed(t, layout) for t in (q, k, v, o, do))
    ts = (q, k, v, o, do) + (tuple(out) if out is not None else ())
    like = (q, k, k, q, q) + ((q, k, k) if out is not None else ())
    if not all(t.dtype == q.dtype and t.shape == r.shape for t, r in zip(ts, like)):
        raise SvgbError("q, k, v, o, do (and out) must share dtype; o, do, dq have q's shape, v, dk, dv k's")
    BH, Sq, Skv, D, qs, kvs = _kv_geometry(q, k, layout)
    G = _kv_group(q, k)
    if G > 1:
        _gqa_check(_dt(q), plan)
    plan_t = plan.key_major()
    lse = lse.to(torch.float32).contiguous()
    grads = (torch.empty_like(t) for t in (q, k, v)) if out is None else out
    dq, dk, dv = (g if _addressable(g, layout) else torch.empty_like(r) for g, r in zip(grads, (q, k, v)))
    _need_cuda(dq, dk, dv)
    scale = float(D) ** -0.5 if sm_scale is None else float(sm_scale)
    if not all(t.is_contiguous() for t in (q, k, v, o, do, dq, dk, dv)):
        B = q.shape[0] if layout == "bhsd" else 1
        lens = (B, q.shape[1], k.shape[1], Sq, Skv)
        nbytes = C.c_size_t()
        check(lib().svgb_attn_bwd_strided_bytes(*lens, C.byref(nbytes)), "svgb_attn_bwd_strided_bytes")
        ws = workspace(("attn_bwd", BH, Sq), nbytes.value, q.device)
        check(lib().svgb_attn_bwd_strided(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), do.data_ptr(),
                                          lse.data_ptr(), dq.data_ptr(), dk.data_ptr(), dv.data_ptr(), _dt(q), *lens, D,
                                          *(_st(t, layout) for t in (q, k, v, o, do, dq, dk, dv)), scale,
                                          C.byref(plan.desc), plan.ws.data_ptr(), C.byref(plan_t.desc),
                                          plan_t.ws.data_ptr(), ws.data_ptr(), ws.numel(), _stream(q)),
              "svgb_attn_bwd_strided")
        _bump(3)
        return _written(out, (dq, dk, dv))
    # equal lengths and heads take svgb_attn_bwd, whose q and k share one length and one pair of strides
    if G > 1:
        name, lens, strides = "svgb_attn_bwd_gqa", (BH, BH // G, Sq, Skv), qs + kvs
    elif Sq == Skv:
        name, lens, strides = "svgb_attn_bwd", (BH, Sq), qs
    else:
        name, lens, strides = "svgb_attn_bwd_kv", (BH, Sq, Skv), qs + kvs
    nbytes = C.c_size_t()
    check(getattr(lib(), name + "_bytes")(*lens, C.byref(nbytes)), name + "_bytes")
    ws = workspace(("attn_bwd", BH, Sq), nbytes.value, q.device)
    check(getattr(lib(), name)(q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), do.data_ptr(), lse.data_ptr(),
                               dq.data_ptr(), dk.data_ptr(), dv.data_ptr(), _dt(q), *lens, D, *strides, scale,
                               C.byref(plan.desc), plan.ws.data_ptr(), C.byref(plan_t.desc), plan_t.ws.data_ptr(),
                               ws.data_ptr(), ws.numel(), _stream(q)), name)
    _bump(3)
    return _written(out, (dq, dk, dv))


def _written(out, gs):
    """The gradients, copied into those of the out= tensors the kernels could not address."""
    if out is None:
        return gs
    for o, g in zip(out, gs):
        if o is not g:
            o.copy_(g)
    return tuple(out)


class _Attention(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q, k, v, plan, layout, sm_scale):
        o, lse = attn_fwd(q, k, v, plan, layout=layout, return_lse=True, sm_scale=sm_scale)
        ctx.save_for_backward(q, k, v, o, lse)
        ctx.plan, ctx.layout, ctx.sm_scale = plan, layout, sm_scale
        return o

    @staticmethod
    def backward(ctx, do):
        q, k, v, o, lse = ctx.saved_tensors
        dq, dk, dv = attn_bwd(q, k, v, o, do, lse, ctx.plan, layout=ctx.layout, sm_scale=ctx.sm_scale)
        return dq, dk, dv, None, None, None


def attention(q, k, v, plan: AttnPlan, *, layout: str = "bhsd", sm_scale: Optional[float] = None):
    """attn_fwd, differentiable when an input requires grad (needs_grad): the forward then keeps its LSE and the
    backward runs attn_bwd, and plans without a backward (gather plans, the profiling masks) are rejected before the
    forward runs.  Otherwise it is exactly attn_fwd(q, k, v, plan, layout=layout, sm_scale=sm_scale): one launch, no
    LSE, and the plan is not read here."""
    if not needs_grad(q, k, v):
        return attn_fwd(q, k, v, plan, layout=layout, sm_scale=sm_scale)
    if plan.desc.kind in (PLAN_GATHER, PLAN_KVCACHE, PLAN_KVCACHE_SPLIT) or (plan.desc.kind == PLAN_BAND and
                                                                              _is_profiling(plan.desc.mask_mode)):
        plan.key_major()  # raises, naming what has no backward
    return _Attention.apply(q, k, v, plan, layout, sm_scale)


def needs_grad(*ts) -> bool:
    """True when autograd would record an op on these tensors: attention() then records _Attention, and the layout
    ops _HeadPlacement / _Permute and the pre-attention chain _RowNorm / _QkRope / _QkvPrep their own functions."""
    return torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in ts)


class _HeadPlacement(torch.autograd.Function):
    """head_placement under autograd.  The outputs are the caller's tensors written in place (ctx.mark_dirty, so the
    caller's own objects carry the history; no copy).  Every row of every output is written, so their old contents get
    no gradient.  A placement only moves rows, so its backward is the same kernel in the opposite direction (inverse
    flipped, same text_first), one launch for all incoming gradients.  best_mask_idx is an integer selection and gets
    no gradient (the head choice of sample_mse is a constant, as the BlockMask is to flex_attention)."""

    @staticmethod
    def forward(ctx, args, n, *ts):
        outs = ts[n:]
        _place(ts[:n], outs, *args)
        ctx.mark_dirty(*outs)
        ctx.set_materialize_grads(False)
        ctx.args, ctx.n = args, n
        return outs

    @staticmethod
    def backward(ctx, *gs):
        idx, BH, S, D, context, F, P, text_first, inverse = ctx.args
        want = [i for i in range(ctx.n) if ctx.needs_input_grad[2 + i] and gs[i] is not None]
        grads = [None] * ctx.n
        if want:
            src = [gs[i].contiguous() for i in want]
            dst = [torch.empty_like(g) for g in src]
            head_placement(src, dst, idx, context, F, P, text_first=text_first, inverse=not inverse)
            for i, g in zip(want, dst):
                grads[i] = g
        return (None, None, *grads, *([None] * ctx.n))


class _Permute(torch.autograd.Function):
    """permute_gather / permute_scatter under autograd: the backward of each is the other under the same permutation.
    The permutation (sorted indices from the labels) is an integer selection and gets no gradient."""

    @staticmethod
    def forward(ctx, x, perm, scatter):
        ctx.save_for_backward(perm)
        ctx.scatter = scatter
        return _permute(x, perm, scatter)

    @staticmethod
    def backward(ctx, g):
        perm, = ctx.saved_tensors
        return (permute_gather if ctx.scatter else permute_scatter)(g, perm), None, None


def quantize_e4m3_rows(x: torch.Tensor):
    """Per-row quantisation of a 16-bit [rows, H, 128] tensor, read in place at its row and head strides (a view is
    copied only when they are not multiples of 8 elements): returns (x8 uint8 [rows, H, 128], scale fp32 [H, rows]) with
    x ~= x8.view(float8_e4m3fn) * scale[h, r], scale a power of two from the row's own absmax (include/svgb200.h,
    svgb_kvcache_append_e4m3_rows).  One launch."""
    _need_cuda(x)
    if x.dim() != 3 or x.shape[2] != 128 or x.dtype not in (torch.bfloat16, torch.float16):
        raise SvgbError(f"quantize_e4m3_rows takes a bf16 or fp16 [rows, H, 128] tensor (got {tuple(x.shape)}, {x.dtype})")
    if not _addressable(x, "shd"):
        x = x.clone(memory_format=torch.contiguous_format)
    R, H, D = x.shape
    x8 = torch.empty(R, H, D, dtype=torch.uint8, device=x.device)
    scale = torch.empty(H, R, dtype=torch.float32, device=x.device)
    _, hs, rs = _strides(x, "shd")
    check(lib().svgb_quantize_e4m3_rows(x.data_ptr(), _dt(x), x8.data_ptr(), scale.data_ptr(), R, H, D, rs, hs,
                                        _stream(x)), "svgb_quantize_e4m3_rows")
    _bump()
    return x8, scale


def quantize_e4m3(x: torch.Tensor):
    """Per-head absmax quantisation of a 16-bit [..., S, D] tensor to fp8 e4m3 bytes.
    Returns (x8 uint8 same shape, scale fp32 [BH]) with x ~= x8.view(float8_e4m3fn) * scale[h]."""
    _need_cuda(x)
    S, D = x.shape[-2], x.shape[-1]
    xc = x.contiguous()
    BH = xc.numel() // (S * D)
    x8 = torch.empty(xc.shape, dtype=torch.uint8, device=x.device)
    scale = torch.empty(BH, dtype=torch.float32, device=x.device)
    check(lib().svgb_quantize_e4m3(xc.data_ptr(), _dt(x), x8.data_ptr(), scale.data_ptr(), BH, S, D, _stream(x)),
          "svgb_quantize_e4m3")
    _bump(3)
    return x8, scale


def attn_fwd_fp8(q8, k8, v8, q_scale, k_scale, v_scale, plan: AttnPlan, *, o_rows: Optional[torch.Tensor] = None,
                 q_rows: Optional[torch.Tensor] = None, kv_rows: Optional[torch.Tensor] = None,
                 return_lse: bool = False, sm_scale: Optional[float] = None):
    """FP8 (e4m3) block-sparse attention: q8,k8,v8 uint8 [B,H,S,128] + per-head scales -> bf16 [B,H,S,128].
    With a gather plan (plan_varblock(..., gather=True)), q_rows / kv_rows read the rows through index vectors, as in
    attn_fwd."""
    _need_cuda(q8, k8, v8, q_scale, k_scale, v_scale)
    if q8.dim() == k8.dim() and q8.dim() > 1 and q8.shape[1] != k8.shape[1]:
        _gqa_check(_E4M3, plan)
    if not (q8.dtype == k8.dtype == v8.dtype == torch.uint8) or not (q8.shape == k8.shape == v8.shape):
        raise SvgbError("q8, k8, v8 must be uint8 tensors of one shape")
    B, H, S, D = q8.shape
    o = torch.empty(B, H, S, D, dtype=torch.bfloat16, device=q8.device)
    # temporaries are bound to locals that outlive the launch call (a dropped .contiguous() copy could be recycled
    # by the allocator for the next one and alias two operands)
    q8c, k8c, v8c = q8.contiguous(), k8.contiguous(), v8.contiguous()
    scales = tuple(t.to(torch.float32).contiguous() for t in (q_scale, k_scale, v_scale))
    return _attn(q8c, k8c, v8c, o, plan, "bhsd", _E4M3, scales, (q_rows, kv_rows, o_rows), return_lse, sm_scale)


def density(block_map, row_sz, col_sz):
    _need_cuda(block_map, row_sz, col_sz)
    BH, QC, KC = block_map.shape
    m = block_map.contiguous()
    m = m.view(torch.uint8) if m.dtype == torch.bool else m.to(torch.uint8)
    r = row_sz.reshape(BH, QC).to(torch.int32).contiguous()
    c = col_sz.reshape(BH, KC).to(torch.int32).contiguous()
    out = torch.empty(BH, dtype=torch.float32, device=m.device)
    check(lib().svgb_density(m.data_ptr(), r.data_ptr(), c.data_ptr(), BH, QC, KC, out.data_ptr(), _stream(m)),
          "svgb_density")
    _bump()
    return out


# ----------------------------------------------------------------------------------------------
# layout transforms
# ----------------------------------------------------------------------------------------------
def argsort_labels(labels: torch.Tensor, K: int):
    """labels int [BH,S] in [0,K) -> (perm int32 [BH,S] stable ascending, counts int32 [BH,K])."""
    _need_cuda(labels)
    BH, S = labels.shape
    lab = labels.to(torch.int32).contiguous()
    nbytes = C.c_size_t()
    check(lib().svgb_argsort_labels_bytes(BH, S, K, C.byref(nbytes)), "argsort_labels_bytes")
    ws = workspace(("sort", BH, S, K), nbytes.value, lab.device)
    perm = torch.empty(BH, S, dtype=torch.int32, device=lab.device)
    counts = torch.empty(BH, K, dtype=torch.int32, device=lab.device)
    check(lib().svgb_argsort_labels(lab.data_ptr(), BH, S, K, perm.data_ptr(), counts.data_ptr(),
                                    ws.data_ptr(), ws.numel(), _stream(lab)), "svgb_argsort_labels")
    _bump(3)
    return perm, counts


def _rows_op(fn, name, x, perm):
    _need_cuda(x, perm)
    if x.element_size() != 2:
        raise SvgbError("permute kernels move 16-bit elements")
    shape = x.shape
    D = shape[-1]
    S = shape[-2]
    xf = x.contiguous().view(-1, S, D)
    BH = xf.shape[0]
    p = perm.reshape(BH, S).to(torch.int32).contiguous()
    out = torch.empty_like(xf)
    check(fn(xf.data_ptr(), p.data_ptr(), out.data_ptr(), BH, S, D, _stream(x)), name)
    _bump()
    return out.view(shape)


def _permute(x, perm, scatter):
    if scatter:
        return _rows_op(lib().svgb_permute_scatter, "svgb_permute_scatter", x, perm)
    return _rows_op(lib().svgb_permute_gather, "svgb_permute_gather", x, perm)


def permute_gather(x, perm):
    """out[bh, s] = x[bh, perm[bh, s]].  Differentiable in x when it requires grad (_Permute)."""
    if needs_grad(x):
        return _Permute.apply(x, perm, False)
    return _permute(x, perm, False)


def permute_scatter(x, perm):
    """out[bh, perm[bh, s]] = x[bh, s].  Differentiable in x when it requires grad (_Permute)."""
    if needs_grad(x):
        return _Permute.apply(x, perm, True)
    return _permute(x, perm, True)


def _place(ins, outs, idx, BH, S, D, ctx, F, P, text_first, inverse):
    n = len(ins)
    a_in = (C.c_void_p * n)(*[t.data_ptr() for t in ins])
    a_out = (C.c_void_p * n)(*[t.data_ptr() for t in outs])
    check(lib().svgb_head_placement(a_in, a_out, n, idx.data_ptr(), BH, S, D, ctx, F, P,
                                    1 if text_first else 0, 1 if inverse else 0, _stream(ins[0])),
          "svgb_head_placement")
    _bump()


def head_placement(ins, outs, best_mask_idx, ctx, F, P, *, text_first=False, inverse=False):
    """ins / outs: lists (1..3) of [cfg,H,S,D] contiguous 16-bit tensors; writes outs in place.  When an input
    requires grad the outs (the same objects) carry the history (_HeadPlacement)."""
    _need_cuda(*ins, *outs, best_mask_idx)
    cfg, H, S, D = ins[0].shape
    for t in list(ins) + list(outs):
        if not t.is_contiguous() or t.shape != ins[0].shape or t.element_size() != 2:
            raise SvgbError("placement tensors must be contiguous 16-bit [cfg,H,S,D] of one shape")
    idx = best_mask_idx.reshape(cfg * H).to(torch.int32).contiguous()
    args = (idx, cfg * H, S, D, ctx, F, P, text_first, inverse)
    if needs_grad(*ins, *outs):
        _HeadPlacement.apply(args, len(ins), *ins, *outs)
    else:
        _place(ins, outs, *args)
    return outs


# ----------------------------------------------------------------------------------------------
# flash k-means
# ----------------------------------------------------------------------------------------------
def _km_ws(BH, N, K, D, device):
    nbytes = C.c_size_t()
    check(lib().svgb_kmeans_bytes(BH, N, K, D, C.byref(nbytes)), "svgb_kmeans_bytes")
    return workspace(("km", BH, N, K, D), nbytes.value, device)


def row_sqnorm(x, round_result=True):
    """x [BH,N,D] 16-bit -> fp32 [BH,N]"""
    _need_cuda(x)
    BH, N, D = x.shape
    xc = x.contiguous()
    out = torch.empty(BH, N, dtype=torch.float32, device=x.device)
    check(lib().svgb_row_sqnorm(xc.data_ptr(), out.data_ptr(), BH, N, D, _dt(x), 1 if round_result else 0,
                                _stream(x)), "svgb_row_sqnorm")
    _bump()
    return out


def kmeans_assign(x, c, x_sq):
    _need_cuda(x, c, x_sq)
    BH, N, D = x.shape
    K = c.shape[1]
    xc, cc, sqc = x.contiguous(), c.contiguous(), x_sq.to(torch.float32).contiguous()
    ws = _km_ws(BH, N, K, D, x.device)
    labels = torch.empty(BH, N, dtype=torch.int32, device=x.device)
    check(lib().svgb_kmeans_assign(xc.data_ptr(), cc.data_ptr(), sqc.data_ptr(), labels.data_ptr(),
                                   BH, N, K, D, _dt(x), ws.data_ptr(), ws.numel(), _stream(x)),
          "svgb_kmeans_assign")
    _bump(2)
    return labels


def kmeans_update(x, labels, c_old):
    _need_cuda(x, labels, c_old)
    BH, N, D = x.shape
    K = c_old.shape[1]
    ws = _km_ws(BH, N, K, D, x.device)
    xc, lc, cc = x.contiguous(), labels.to(torch.int32).contiguous(), c_old.contiguous()
    c_new = torch.empty_like(cc)
    counts = torch.empty(BH, K, dtype=torch.int32, device=x.device)
    shift = torch.zeros(1, dtype=torch.float32, device=x.device)
    check(lib().svgb_kmeans_update(xc.data_ptr(), lc.data_ptr(),
                                   cc.data_ptr(), c_new.data_ptr(), counts.data_ptr(),
                                   shift.data_ptr(), BH, N, K, D, _dt(x), ws.data_ptr(), ws.numel(), _stream(x)),
          "svgb_kmeans_update")
    _bump(5)
    return c_new, counts, shift


def kmeans_run(x, init_centroids, max_iters, tol=1e-4, want_perm=False):
    """Whole Lloyd loop on the device (no host sync).  Returns labels int32 [BH,N], centroids [BH,K,D],
    counts int32 [BH,K], n_iter int32[1] (device) and, with want_perm, the stable argsort of the labels int32 [BH,N]
    (the member lists of the last centroid update).  x may be a view whose heads are further apart than N*D (the video
    part of a [H, S, D] tensor): it is clustered in place, without a packing copy."""
    _need_cuda(x, init_centroids)
    BH, N, D = x.shape
    K = init_centroids.shape[1]
    ws = _km_ws(BH, N, K, D, x.device)
    labels = torch.empty(BH, N, dtype=torch.int32, device=x.device)
    cents = torch.empty(BH, K, D, dtype=x.dtype, device=x.device)
    counts = torch.empty(BH, K, dtype=torch.int32, device=x.device)
    n_iter = torch.zeros(1, dtype=torch.int32, device=x.device)
    perm = torch.empty(BH, N, dtype=torch.int32, device=x.device) if want_perm else None
    strided_ok = x.stride(2) == 1 and x.stride(1) == D and (BH == 1 or (x.stride(0) >= N * D and x.stride(0) % 8 == 0))
    xc = x if strided_ok else x.contiguous()
    head_stride = xc.stride(0) if BH > 1 else N * D
    ic = init_centroids.contiguous()
    check(lib().svgb_kmeans_run_sorted(xc.data_ptr(), head_stride, ic.data_ptr(), BH, N, K, D,
                                       _dt(x), int(max_iters), float(tol), labels.data_ptr(), cents.data_ptr(),
                                       counts.data_ptr(), n_iter.data_ptr(), perm.data_ptr() if want_perm else None,
                                       ws.data_ptr(), ws.numel(), _stream(x)),
          "svgb_kmeans_run_sorted")
    _bump(2 + 7 * int(max_iters))
    if want_perm:
        return labels, cents, counts, n_iter, perm
    return labels, cents, counts, n_iter


def dynamic_map(qc, kc, k_sizes, top_p, preserve):
    """qc [BH,QC,D], kc [BH,KC,D] 16-bit, k_sizes int [BH,KC] -> bool [BH,QC,KC]"""
    _need_cuda(qc, kc, k_sizes)
    BH, QC, D = qc.shape
    KC = kc.shape[1]
    out = torch.empty(BH, QC, KC, dtype=torch.uint8, device=qc.device)
    qcc, kcc, ksc = qc.contiguous(), kc.contiguous(), k_sizes.to(torch.int32).contiguous()
    check(lib().svgb_dynamic_map(qcc.data_ptr(), kcc.data_ptr(),
                                 ksc.data_ptr(), BH, QC, KC, D, _dt(qc),
                                 float(top_p), int(preserve), out.data_ptr(), _stream(qc)), "svgb_dynamic_map")
    _bump()
    return out.view(torch.bool)


def sample_mse(q, k, v, rows, layout, ctx, F, P):
    """q,k,v [BH,S,D]; rows int [n] (<=128) -> fp32 [2, BH] (0 = spatial mask, 1 = temporal mask)"""
    _need_cuda(q, k, v, rows)
    BH, S, D = q.shape
    n = rows.numel()
    nbytes = C.c_size_t()
    check(lib().svgb_sample_mse_bytes(BH, S, D, n, C.byref(nbytes)), "svgb_sample_mse_bytes")
    ws = workspace(("smse", BH, S, D), nbytes.value, q.device)
    out = torch.empty(2, BH, dtype=torch.float32, device=q.device)
    r = rows.to(torch.int32).contiguous()
    qc_, kc_, vc_ = q.contiguous(), k.contiguous(), v.contiguous()
    check(lib().svgb_sample_mse(qc_.data_ptr(), kc_.data_ptr(), vc_.data_ptr(),
                                r.data_ptr(), n, BH, S, D, _dt(q), int(layout), ctx, F, P, out.data_ptr(),
                                ws.data_ptr(), ws.numel(), _stream(q)), "svgb_sample_mse")
    _bump(7)
    return out


def selftest_tile(q, k, v, p_scale=0.0625):
    """q,k,v: [128, D] -> (S fp32 [128,128], O fp32 [128,D])"""
    _need_cuda(q, k, v)
    D = q.shape[-1]
    s = torch.empty(128, 128, dtype=torch.float32, device=q.device)
    o = torch.empty(128, D, dtype=torch.float32, device=q.device)
    check(lib().svgb_selftest_tile(q.data_ptr(), k.data_ptr(), v.data_ptr(), s.data_ptr(), o.data_ptr(),
                                   D, _dt(q), p_scale, _stream(q)), "svgb_selftest_tile")
    _bump()
    return s, o


# ---- pre-attention chain (include/svgb200.h: svgb_rms_norm / svgb_layer_norm / svgb_qk_rope / svgb_qkv_prep)
ROPE_TXT_FIRST, ROPE_TXT_LAST, ROPE_COMPLEX_TXT_FIRST = 0, 1, 2
NORM_NONE, NORM_RMS_HEAD, NORM_LAYER, NORM_RMS_HIDDEN = 0, 1, 2, 3


def _dt3(t: torch.Tensor) -> int:
    if t.dtype == torch.float32:
        return 3
    return _dt(t)


def _contig(*ts):
    for t in ts:
        if t is not None and not t.is_contiguous():
            raise SvgbError("tensor must be contiguous")


def _no_backward(what, *ts):
    """Ops and attention paths without a backward raise under grad rather than return a result detached from the
    graph."""
    if needs_grad(*ts):
        raise SvgbError(f"{what} has no backward: call it on tensors that do not require grad "
                        "(or under torch.no_grad())")


def _tables_no_grad(cos, sin):
    if needs_grad(cos, sin):
        raise SvgbError("the RoPE tables cos / sin get no gradient: pass tables that do not require grad (.detach())")


def _row_norm(x, gamma, beta, eps):
    n = x.shape[-1]
    if beta is None:
        check(lib().svgb_rms_norm(x.data_ptr(), gamma.data_ptr(), x.numel() // n, n, float(eps), _dt(x), _stream(x)),
              "svgb_rms_norm")
    else:
        check(lib().svgb_layer_norm(x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), x.numel() // n, n, _dt(x),
                                    _stream(x)), "svgb_layer_norm")
    _bump()


def _row_norm_bwd(x, dy, gamma, eps, layer):
    _need_cuda(x, dy, gamma)
    _contig(x, dy, gamma)
    if dy.shape != x.shape or dy.dtype != x.dtype:
        raise SvgbError("dy must have the shape and dtype of x")
    n = x.shape[-1]
    m = x.numel() // n
    nbytes = C.c_size_t()
    check(lib().svgb_row_norm_bwd_bytes(m, n, C.byref(nbytes)), "svgb_row_norm_bwd_bytes")
    ws = workspace("row_norm_bwd", nbytes.value, x.device)
    dx = torch.empty_like(x)
    dg = torch.empty(n, dtype=torch.float32, device=x.device)
    if layer:
        db = torch.empty(n, dtype=torch.float32, device=x.device)
        check(lib().svgb_layer_norm_bwd(x.data_ptr(), dy.data_ptr(), gamma.data_ptr(), dx.data_ptr(), dg.data_ptr(),
                                        db.data_ptr(), m, n, _dt(x), ws.data_ptr(), ws.numel(), _stream(x)),
              "svgb_layer_norm_bwd")
    else:
        db = None
        check(lib().svgb_rms_norm_bwd(x.data_ptr(), dy.data_ptr(), gamma.data_ptr(), dx.data_ptr(), dg.data_ptr(), m, n,
                                      float(eps), _dt(x), ws.data_ptr(), ws.numel(), _stream(x)), "svgb_rms_norm_bwd")
    _bump(2)
    return dx, dg.to(gamma.dtype), None if db is None else db.to(gamma.dtype)


def rms_norm_bwd(x, dy, gamma, eps: float = 1e-5):
    """Gradients (dx, dgamma) of rms_norm_ at its input x (the values before the in-place norm) for the output gradient
    dy.  dgamma is summed in fp32 in a fixed order and rounded once to gamma's dtype."""
    dx, dg, _ = _row_norm_bwd(x, dy, gamma, eps, False)
    return dx, dg


def layer_norm_bwd(x, dy, gamma):
    """Gradients (dx, dgamma, dbeta) of layer_norm_ at its input x for the output gradient dy."""
    return _row_norm_bwd(x, dy, gamma, 0.0, True)


class _RowNorm(torch.autograd.Function):
    """rms_norm_ / layer_norm_ under autograd.  The norm still runs in place: the caller's tensor (often a .view(-1, D)
    of a non-leaf) is marked dirty and carries the history.  A copy of x taken before the kernel is the one extra
    buffer.  eps gets no gradient."""

    @staticmethod
    def forward(ctx, x, gamma, beta, eps):
        ctx.save_for_backward(x.clone(), gamma)
        ctx.eps, ctx.layer = eps, beta is not None
        _row_norm(x, gamma, beta, eps)
        ctx.mark_dirty(x)
        return x

    @staticmethod
    def backward(ctx, dy):
        x, gamma = ctx.saved_tensors
        dx, dg, db = _row_norm_bwd(x, dy.contiguous(), gamma, ctx.eps, ctx.layer)
        return dx, dg if ctx.needs_input_grad[1] else None, db if ctx.needs_input_grad[2] else None, None


def rms_norm_(x: torch.Tensor, gamma: torch.Tensor, eps: float = 1e-5) -> torch.Tensor:
    """In place on x [m, n] (any leading shape; last dim n in {32,64,128,256}).  Differentiable in x and gamma when
    either requires grad (_RowNorm)."""
    _need_cuda(x, gamma)
    _contig(x, gamma)
    if gamma.dim() != 1 or gamma.shape[0] != x.shape[-1] or gamma.dtype != x.dtype:
        raise SvgbError("gamma must be [n] with the dtype of x")
    if needs_grad(x, gamma):
        return _RowNorm.apply(x, gamma, None, float(eps))
    _row_norm(x, gamma, None, eps)
    return x


def layer_norm_(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor) -> torch.Tensor:
    """In place on x [m, n], eps 1e-5.  Differentiable in x, gamma and beta (_RowNorm)."""
    _need_cuda(x, gamma, beta)
    _contig(x, gamma, beta)
    n = x.shape[-1]
    if gamma.shape != (n,) or beta.shape != (n,) or gamma.dtype != x.dtype or beta.dtype != x.dtype:
        raise SvgbError("gamma / beta must be [n] with the dtype of x")
    if needs_grad(x, gamma, beta):
        return _RowNorm.apply(x, gamma, beta, 0.0)
    _row_norm(x, gamma, beta, 0.0)
    return x


def _rope_check(q, k, cos, sin, len_text, mode):
    _need_cuda(q, k, cos, sin)
    _contig(q, k, cos, sin)
    if q.dim() != 4 or k.dim() != 4 or cos.dim() != 2 or sin.dim() != 2:
        raise SvgbError("q, k must be 4-D and cos, sin 2-D")
    if cos.dtype != torch.float32 or sin.dtype != torch.float32:
        raise SvgbError("cos / sin caches must be float32")
    B, Hq, S, D = q.shape
    if k.shape[0] != B or k.shape[2] != S or k.shape[3] != D or k.dtype != q.dtype:
        raise SvgbError("q and k must agree in batch, sequence, head_dim and dtype")
    valid = S - int(len_text)
    width = D // 2 if mode == ROPE_COMPLEX_TXT_FIRST else D
    if tuple(cos.shape) != (valid, width) or tuple(sin.shape) != (valid, width):
        raise SvgbError(f"cos / sin must be [{valid}, {width}], got {tuple(cos.shape)} / {tuple(sin.shape)}")


def _rope(q, k, cos, sin, len_text, mode):
    B, Hq, S, D = q.shape
    check(lib().svgb_qk_rope(q.data_ptr(), k.data_ptr(), cos.data_ptr(), sin.data_ptr(), B, Hq, k.shape[1], S, D,
                             int(len_text), int(mode), _dt(q), _stream(q)), "svgb_qk_rope")
    _bump()


def qk_rope_bwd(dq, dk, cos, sin, len_text: int, mode: int):
    """Gradients (dq_in, dk_in) of qk_rope_ for the output gradients dq [B,Hq,S,D], dk [B,Hk,S,D]: the transpose of
    each rotation on the rotated rows (exact for tables whose pairs differ), the text rows passed through."""
    _rope_check(dq, dk, cos, sin, len_text, mode)
    gq, gk = torch.empty_like(dq), torch.empty_like(dk)
    B, Hq, S, D = dq.shape
    check(lib().svgb_qk_rope_bwd(dq.data_ptr(), dk.data_ptr(), gq.data_ptr(), gk.data_ptr(), cos.data_ptr(),
                                 sin.data_ptr(), B, Hq, dk.shape[1], S, D, int(len_text), int(mode), _dt(dq),
                                 _stream(dq)), "svgb_qk_rope_bwd")
    _bump()
    return gq, gk


class _QkRope(torch.autograd.Function):
    """qk_rope_ under autograd: in place, q and k marked dirty; the backward is qk_rope_bwd (out of place)."""

    @staticmethod
    def forward(ctx, q, k, cos, sin, len_text, mode):
        _rope(q, k, cos, sin, len_text, mode)
        ctx.save_for_backward(cos, sin)
        ctx.len_text, ctx.mode = len_text, mode
        ctx.mark_dirty(q, k)
        return q, k

    @staticmethod
    def backward(ctx, gq, gk):
        cos, sin = ctx.saved_tensors
        dq, dk = qk_rope_bwd(gq.contiguous(), gk.contiguous(), cos, sin, ctx.len_text, ctx.mode)
        return (dq if ctx.needs_input_grad[0] else None, dk if ctx.needs_input_grad[1] else None,
                None, None, None, None)


def qk_rope_(q: torch.Tensor, k: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor, len_text: int, mode: int):
    """In place on q [B,Hq,S,D], k [B,Hk,S,D]; cos/sin float32 [S-len_text, D] (or [.., D/2] for the complex mode).
    Differentiable in q and k (_QkRope); tables that require grad raise."""
    _tables_no_grad(cos, sin)
    _rope_check(q, k, cos, sin, len_text, mode)
    if needs_grad(q, k):
        return _QkRope.apply(q, k, cos, sin, int(len_text), int(mode))
    _rope(q, k, cos, sin, len_text, mode)
    return q, k


def _check_tables_and_weights(D, HD, dtype, norm, rope, cos, sin, rope_n, weights):
    """The checks qkv_prep and qkv_prep_bwd share.  RoPE tables: float32, contiguous, [rope_n, D] (complex mode:
    [rope_n, D/2]), rope_n defaulting to the tables' rows.  weights: (name, tensor or None) pairs of norm weights, each
    contiguous [D] (NORM_RMS_HIDDEN: [H*D]) of dtype.  Returns rope_n (0 without RoPE)."""
    if rope:
        if cos is None or sin is None or cos.dtype != torch.float32 or sin.dtype != torch.float32:
            raise SvgbError("rope needs float32 cos / sin tables")
        _contig(cos, sin)
        if rope_n is None:
            rope_n = cos.shape[0]
        width = D // 2 if rope == 2 else D
        if tuple(cos.shape) != (rope_n, width) or tuple(sin.shape) != (rope_n, width):
            raise SvgbError(f"cos / sin must be [{rope_n}, {width}]")
    else:
        rope_n = 0
    want = HD if norm == NORM_RMS_HIDDEN else D
    for name, g in weights:
        if g is not None and (g.dtype != dtype or g.numel() != want or not g.is_contiguous()):
            raise SvgbError(f"{name} must be contiguous [{want}] of the input dtype")
    return rope_n


def qkv_prep_bwd(dq, dk, dv, heads: int, S_in: int, *, q_in=None, k_in=None, out_row0: int = 0,
                 norm: int = NORM_NONE, gamma_q=None, gamma_k=None, eps: float = 1e-6, rope: int = 0, cos=None,
                 sin=None, rope_lo: int = 0, rope_n: Optional[int] = None):
    """Gradients of one qkv_prep call for the output gradients dq, dk, dv [B, H, S_out, D] (only rows
    [out_row0, out_row0 + S_in) are read).  q_in, k_in: the forward's inputs (any strides qkv_prep takes), needed when
    norm != NORM_NONE.  Returns (dq_in, dk_in, dv_in) contiguous [B, S_in, H*D] and (dgamma_q, dgamma_k, dbeta_q,
    dbeta_k) in gamma's dtype (None where the norm has none)."""
    _need_cuda(dq, dk, dv, q_in, k_in, gamma_q, gamma_k, cos, sin)
    B, H, S_out, D = dq.shape
    for t in (dq, dk, dv):
        if t.shape != dq.shape or t.dtype != dq.dtype or not t.is_contiguous():
            raise SvgbError("dq, dk, dv must be contiguous [B, H, S_out, D] of one dtype")
    if H != heads or out_row0 < 0 or out_row0 + S_in > S_out:
        raise SvgbError("the gradients must be [B, heads, S_out, D] with out_row0 + S_in <= S_out")
    ts, bs = 0, 0
    if norm != NORM_NONE:
        if q_in is None or k_in is None or gamma_q is None or gamma_k is None:
            raise SvgbError("a norm backward needs q_in, k_in, gamma_q and gamma_k")
        for t in (q_in, k_in):
            if tuple(t.shape) != (B, S_in, H * D) or t.dtype != dq.dtype or t.stride(2) != 1 or t.stride() != q_in.stride():
                raise SvgbError("q_in, k_in must be [B, S_in, H*D] of the gradients' dtype with one set of strides")
        ts, bs = q_in.stride(1), q_in.stride(0)
    weights = (("gamma_q / gamma_k", gamma_q), ("gamma_q / gamma_k", gamma_k)) if norm != NORM_NONE else ()
    rope_n = _check_tables_and_weights(D, H * D, dq.dtype, norm, rope, cos, sin, rope_n, weights)
    nbytes = C.c_size_t()
    check(lib().svgb_qkv_prep_bwd_bytes(B, S_in, H, D, int(norm), C.byref(nbytes)), "svgb_qkv_prep_bwd_bytes")
    ws = workspace("qkv_prep_bwd", nbytes.value, dq.device)
    dx = tuple(torch.empty(B, S_in, H * D, dtype=dq.dtype, device=dq.device) for _ in range(3))
    gw = H * D if norm == NORM_RMS_HIDDEN else D
    f32 = lambda: torch.empty(gw, dtype=torch.float32, device=dq.device)  # noqa: E731
    dg = (f32(), f32()) if norm != NORM_NONE else (None, None)
    db = (f32(), f32()) if norm == NORM_LAYER else (None, None)
    check(lib().svgb_qkv_prep_bwd(dq.data_ptr(), dk.data_ptr(), dv.data_ptr(), S_out * D, H * S_out * D, _p(q_in),
                                  _p(k_in), ts, bs, dx[0].data_ptr(), dx[1].data_ptr(), dx[2].data_ptr(), B, S_in, H, D,
                                  int(out_row0), int(norm), _p(gamma_q), _p(gamma_k), float(eps), int(rope), _p(cos),
                                  _p(sin), int(rope_lo), int(rope_n), _p(dg[0]), _p(dg[1]), _p(db[0]), _p(db[1]),
                                  _dt(dq), ws.data_ptr(), ws.numel(), _stream(dq)), "svgb_qkv_prep_bwd")
    _bump({NORM_NONE: 1, NORM_RMS_HIDDEN: 3}.get(norm, 2))
    cast = [None if g is None else g.to(dq.dtype) for g in (*dg, *db)]
    return (*dx, *cast)


def _prep_streams(heads, S_out, calls, ts):
    """One new (q, k, v) [B, heads, S_out, D] filled by one _qkv_prep per call: ts holds each call's q_in, k_in, v_in,
    gamma_q, gamma_k, beta_q, beta_k, and calls its other keyword arguments."""
    B, _, HD = ts[0].shape
    out = tuple(torch.empty(B, heads, S_out, HD // heads, dtype=ts[0].dtype, device=ts[0].device) for _ in range(3))
    for i, kw in enumerate(calls):
        q_in, k_in, v_in, gq, gk, bq, bk = ts[7 * i:7 * i + 7]
        _qkv_prep(q_in, k_in, v_in, heads, out=out, gamma_q=gq, gamma_k=gk, beta_q=bq, beta_k=bk, **kw)
    return out


class _QkvPrep(torch.autograd.Function):
    """One or more qkv_prep calls into one shared output (a single block: one call; the double block: its video and
    prompt streams) under autograd.  Inputs per call: q_in, k_in, v_in, gamma_q, gamma_k, beta_q, beta_k; `calls` holds
    each call's other arguments (row range, norm, eps, RoPE tables and range), which get no gradient.  The backward
    makes one qkv_prep_bwd per call, each reading its own rows of the incoming gradient, with no copies."""

    @staticmethod
    def forward(ctx, heads, S_out, calls, *ts):
        out = _prep_streams(heads, S_out, calls, ts)
        saved = []
        for i, call in enumerate(calls):
            q_in, k_in, _, gq, gk = ts[7 * i:7 * i + 5]
            keep = call["norm"] != NORM_NONE  # the norm backward reads x; a transpose or a rotation does not
            saved += [q_in if keep else None, k_in if keep else None, gq, gk]
        ctx.save_for_backward(*saved)
        ctx.heads, ctx.calls, ctx.rows = heads, calls, [t.shape[1] for t in ts[::7]]
        return out

    @staticmethod
    def backward(ctx, dq, dk, dv):
        dq, dk, dv = (g.contiguous() for g in (dq, dk, dv))
        saved = ctx.saved_tensors
        grads = []
        for i, call in enumerate(ctx.calls):
            q_in, k_in, gq, gk = saved[4 * i:4 * i + 4]
            dqi, dki, dvi, dgq, dgk, dbq, dbk = qkv_prep_bwd(dq, dk, dv, ctx.heads, ctx.rows[i], q_in=q_in, k_in=k_in,
                                                             gamma_q=gq, gamma_k=gk, **call)
            grads += [dqi, dki, dvi, dgq, dgk, dbq, dbk]
        return (None, None, None, *grads)


def qkv_prep_streams(streams, heads: int, S_out: int):
    """Several qkv_prep calls into one new (q, k, v) [B, H, S_out, D]: streams is a list of ((q_in, k_in, v_in),
    kwargs) with qkv_prep's keyword arguments (out_row0 places each).  Under grad one _QkvPrep records them all;
    otherwise they are the plain calls."""
    ts, calls = [], []
    for ins, kw in streams:
        kw = dict(kw)
        ts += [*ins, *(kw.pop(n, None) for n in ("gamma_q", "gamma_k", "beta_q", "beta_k"))]
        calls.append(kw)
    if needs_grad(*ts, *(kw.get(n) for kw in calls for n in ("cos", "sin"))):
        for kw in calls:
            _tables_no_grad(kw.get("cos"), kw.get("sin"))
            kw.setdefault("norm", NORM_NONE)
        return _QkvPrep.apply(heads, S_out, calls, *ts)
    return _prep_streams(heads, S_out, calls, ts)


def qkv_prep(q_in, k_in, v_in, heads: int, *, out=None, out_row0: int = 0, out_rows: Optional[int] = None,
             norm: int = NORM_NONE, gamma_q=None, gamma_k=None, beta_q=None, beta_k=None, eps: float = 1e-6,
             rope: int = 0, cos=None, sin=None, rope_lo: int = 0, rope_n: Optional[int] = None):
    """[B, S_in, H*D] x3 -> (q, k, v) [B, H, S_out, D] rows [out_row0, out_row0+S_in) in one pass (transpose + QK norm
    + RoPE).  q_in/k_in/v_in may be views of one packed projection (last dim contiguous).  Differentiable in the
    inputs and the norm weights when one requires grad (_QkvPrep); then out= is refused (a partly written buffer has
    no clean in-place history) and so are RoPE tables that require grad."""
    if needs_grad(q_in, k_in, v_in, gamma_q, gamma_k, beta_q, beta_k, cos, sin):
        _tables_no_grad(cos, sin)
        if out is not None:
            raise SvgbError("qkv_prep(out=...) has no backward: under grad let it allocate its outputs")
        _need_cuda(q_in, k_in, v_in, gamma_q, gamma_k, beta_q, beta_k, cos, sin)
        kw = dict(out_row0=out_row0, norm=norm, gamma_q=gamma_q, gamma_k=gamma_k, beta_q=beta_q, beta_k=beta_k,
                  eps=eps, rope=rope, cos=cos, sin=sin, rope_lo=rope_lo, rope_n=rope_n)
        S_out = out_rows if out_rows is not None else q_in.shape[1]
        return qkv_prep_streams([((q_in, k_in, v_in), kw)], heads, S_out)
    return _qkv_prep(q_in, k_in, v_in, heads, out=out, out_row0=out_row0, out_rows=out_rows, norm=norm,
                     gamma_q=gamma_q, gamma_k=gamma_k, beta_q=beta_q, beta_k=beta_k, eps=eps, rope=rope, cos=cos,
                     sin=sin, rope_lo=rope_lo, rope_n=rope_n)


def _qkv_prep(q_in, k_in, v_in, heads: int, *, out=None, out_row0: int = 0, out_rows: Optional[int] = None,
              norm: int = NORM_NONE, gamma_q=None, gamma_k=None, beta_q=None, beta_k=None, eps: float = 1e-6,
              rope: int = 0, cos=None, sin=None, rope_lo: int = 0, rope_n: Optional[int] = None):
    _need_cuda(q_in, k_in, v_in, gamma_q, gamma_k, beta_q, beta_k, cos, sin)
    B, S_in, HD = q_in.shape
    D = HD // heads
    for t in (q_in, k_in, v_in):
        if t.shape != q_in.shape or t.dtype != q_in.dtype or t.stride(2) != 1 or t.stride() != q_in.stride():
            raise SvgbError("q_in, k_in, v_in must share shape, dtype and strides (last dim contiguous)")
    S_out = out_rows if out_rows is not None else (out[0].shape[2] if out is not None else S_in)
    if out is None:
        out = tuple(torch.empty(B, heads, S_out, D, dtype=q_in.dtype, device=q_in.device) for _ in range(3))
    for t in out:
        if tuple(t.shape) != (B, heads, S_out, D) or not t.is_contiguous() or t.dtype != q_in.dtype:
            raise SvgbError("outputs must be contiguous [B, H, S_out, D] of the input dtype")
    if out_row0 + S_in > S_out:
        raise SvgbError("out_row0 + S_in exceeds the output rows")
    weights = (("gamma_q", gamma_q), ("gamma_k", gamma_k), ("beta_q", beta_q), ("beta_k", beta_k))
    rope_n = _check_tables_and_weights(D, HD, q_in.dtype, norm, rope, cos, sin, rope_n, weights)
    check(lib().svgb_qkv_prep(q_in.data_ptr(), k_in.data_ptr(), v_in.data_ptr(), q_in.stride(1), q_in.stride(0),
                              out[0].data_ptr(), out[1].data_ptr(), out[2].data_ptr(), S_out * D, heads * S_out * D,
                              B, S_in, heads, D, int(out_row0), int(norm), _p(gamma_q), _p(gamma_k), _p(beta_q),
                              _p(beta_k), float(eps), int(rope), _p(cos), _p(sin), int(rope_lo), int(rope_n),
                              _dt(q_in), _stream(q_in)), "svgb_qkv_prep")
    _bump()
    return out


# ---- Wan transformer-block glue (svgb_layernorm_modulate / svgb_rmsnorm_hidden / svgb_modulate_shift / svgb_gate_residual)
# No backward: under grad these raise at entry (_no_backward) instead of returning a detached result.
_TORCH_DT = {torch.bfloat16: 0, torch.float16: 1, torch.float32: 3}


def _mod_vec(v, N):
    """scale / shift / gate: float32 [N], [nb, N] or [nb, 1, N] -> (tensor [nb, N], nb)."""
    if v.dtype != torch.float32:
        raise SvgbError("modulation vectors must be float32")
    v = v.reshape(-1, N)
    _contig(v)
    return v, v.shape[0]


def _out_dt(out_dtype) -> int:
    if out_dtype not in _TORCH_DT:
        raise SvgbError(f"unsupported out_dtype {out_dtype}: bfloat16, float16 or float32")
    return _TORCH_DT[out_dtype]


def _norm_weights(N, weight, bias=None):
    """The glue's norm weight and bias: [N] each, and one dtype (the kernel reads both with one w_dtype)."""
    for name, t in (("weight", weight), ("bias", bias)):
        if t is not None and t.numel() != N:
            raise SvgbError(f"{name} must hold the hidden size {N} elements, got {t.numel()}")
    if weight is not None and bias is not None and bias.dtype != weight.dtype:
        raise SvgbError(f"bias dtype {bias.dtype} differs from weight dtype {weight.dtype}")


def _rows_per_batch(rows, nb):
    if nb == 1:
        return 0
    if rows % nb:
        raise SvgbError("rows not divisible by the number of modulation vectors")
    return rows // nb


def layernorm_modulate(x, weight=None, bias=None, eps=1e-6, scale=None, shift=None, out_dtype=None):
    _no_backward("layernorm_modulate", x, weight, bias, scale, shift)
    N = x.shape[-1]
    rows = x.numel() // N
    out_dtype = out_dtype or torch.float32
    y_dt = _out_dt(out_dtype)
    _norm_weights(N, weight, bias)
    rpb = 0
    if scale is not None:
        scale, nb = _mod_vec(scale, N)
        shift, nb2 = _mod_vec(shift, N)
        if nb != nb2:
            raise SvgbError("scale and shift must have the same batch")
        rpb = _rows_per_batch(rows, nb)
    _need_cuda(x, weight, bias, scale, shift)
    _contig(x, weight, bias)
    y = torch.empty(x.shape, dtype=out_dtype, device=x.device)
    check(lib().svgb_layernorm_modulate(x.data_ptr(), _dt3(x), _p(weight), _p(bias),
                                        _dt3(weight) if weight is not None else 0, float(eps), _p(scale), _p(shift),
                                        rpb, y.data_ptr(), y_dt, rows, N, _stream(x)),
          "svgb_layernorm_modulate")
    _bump()
    return y


def rmsnorm_hidden(x, weight, eps, out_dtype=None):
    _no_backward("rmsnorm_hidden", x, weight)
    N = x.shape[-1]
    out_dtype = out_dtype or x.dtype
    y_dt = _out_dt(out_dtype)
    _norm_weights(N, weight)
    _need_cuda(x, weight)
    _contig(x, weight)
    y = torch.empty(x.shape, dtype=out_dtype, device=x.device)
    check(lib().svgb_rmsnorm_hidden(x.data_ptr(), _dt3(x), weight.data_ptr(), _dt3(weight), float(eps), y.data_ptr(),
                                    y_dt, x.numel() // N, N, _stream(x)), "svgb_rmsnorm_hidden")
    _bump()
    return y


def modulate_shift(x, scale, shift, out_dtype=torch.float32):
    _no_backward("modulate_shift", x, scale, shift)
    N = x.shape[-1]
    rows = x.numel() // N
    y_dt = _out_dt(out_dtype)
    scale, nb = _mod_vec(scale, N)
    shift, nb2 = _mod_vec(shift, N)
    if nb != nb2:
        raise SvgbError("scale and shift must have the same batch")
    rpb = _rows_per_batch(rows, nb)
    _need_cuda(x, scale, shift)
    _contig(x)
    y = torch.empty(x.shape, dtype=out_dtype, device=x.device)
    check(lib().svgb_modulate_shift(x.data_ptr(), _dt3(x), scale.data_ptr(), shift.data_ptr(), rpb, y.data_ptr(), y_dt,
                                    rows, N, _stream(x)), "svgb_modulate_shift")
    _bump()
    return y


def gate_residual(residual, x, gate, out_dtype=torch.float32):
    _no_backward("gate_residual", residual, x, gate)
    if residual.shape != x.shape:
        raise SvgbError("residual and x must have the same shape")
    N = x.shape[-1]
    rows = x.numel() // N
    y_dt = _out_dt(out_dtype)
    gate, nb = _mod_vec(gate, N)
    rpb = _rows_per_batch(rows, nb)
    _need_cuda(residual, x, gate)
    _contig(residual, x)
    y = torch.empty(x.shape, dtype=out_dtype, device=x.device)
    check(lib().svgb_gate_residual(residual.data_ptr(), _dt3(residual), x.data_ptr(), _dt3(x), gate.data_ptr(),
                                   rpb, y.data_ptr(), y_dt, rows, N, _stream(x)),
          "svgb_gate_residual")
    _bump()
    return y
