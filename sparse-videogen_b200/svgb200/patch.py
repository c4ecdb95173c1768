"""Install the svgb200 operators into an importable copy of the reference (svg-project/Sparse-VideoGen).

The reference's attention processors resolve their operators as module globals
(svg/models/hyvideo/attention.py:12-28); replacing those names is the same mechanism the reference uses
for its own monkey patches (custom_models.py:259-263).  No reference file is edited.

    import svg.models.hyvideo.attention as A
    import svgb200.patch as P
    P.install(A)            # hyvideo / wan / cosmos / cog attention modules
    P.install_kmeans_utils()  # svg.kmeans_utils names used elsewhere
"""
from __future__ import annotations

from . import kmeans_utils as _ku
from . import permute as _pm
from . import placement as _pl

_NAMES = {
    "apply_inverse_permutation_triton": _pm.apply_inverse_permutation_triton,
    "permute_tensor_by_labels_triton": _pm.permute_tensor_by_labels_triton,
    "batch_kmeans_Euclid": _ku.batch_kmeans_Euclid,
    "density_calculation": _ku.density_calculation,
    "dynamic_block_sparse_fwd_flashinfer": _ku.dynamic_block_sparse_fwd_flashinfer,
    "dynamic_block_sparse_fwd_triton": _ku.dynamic_block_sparse_fwd_triton,
    "identify_dynamic_map": _ku.identify_dynamic_map,
    "hunyuan_sparse_head_placement": _pl.hunyuan_sparse_head_placement,
    "hunyuan_hidden_states_placement": _pl.hunyuan_hidden_states_placement,
    "wan_sparse_head_placement": _pl.wan_sparse_head_placement,
    "wan_hidden_states_placement": _pl.wan_hidden_states_placement,
    "cosmos_sparse_head_placement": _pl.cosmos_sparse_head_placement,
    "cosmos_hidden_states_placement": _pl.cosmos_hidden_states_placement,
    "sparse_head_placement": _pl.sparse_head_placement,
    "hidden_states_placement": _pl.hidden_states_placement,
}


def _flex_attention(name, attend, query, key, value, block_mask, kw):
    from .models.common import BandMask

    if not isinstance(block_mask, BandMask):
        raise TypeError(f"svgb200.patch.{name} needs the BandMask returned by the patched prepare_flexattention "
                        f"(got {type(block_mask).__name__}); rebuild block_mask after patch.install()")
    if kw:
        raise TypeError(f"unsupported flex_attention arguments: {sorted(kw)}")
    return attend(query, key, value, block_mask)


def flex_attention(query, key, value, block_mask=None, **kw):
    """Stand-in for torch.nn.attention.flex_attention.flex_attention as the reference processors call it
    (`flex_attention(q, k, v, block_mask=cls.block_mask)`, hyvideo/attention.py:401-403): block_mask must be the
    BandMask built by the patched prepare_flexattention."""
    from .models.common import sparse_flex_attention

    return _flex_attention("flex_attention", sparse_flex_attention, query, key, value, block_mask, kw)


def flex_attention_fp8(query, key, value, block_mask=None, **kw):
    """flex_attention with the band attention on e4m3 Q, K, V (models.common.sparse_flex_attention_fp8)."""
    from .models.common import sparse_flex_attention_fp8

    return _flex_attention("flex_attention_fp8", sparse_flex_attention_fp8, query, key, value, block_mask, kw)


def _varlen_segments(cu_seqlens_q, cu_seqlens_kv):
    """(query segments, key segments) of a varlen call: segment i of the queries attends segment i of the keys.  When
    the two give the same lengths both are the non-empty query segments (the same object); otherwise only the pairs
    where both sides are empty are dropped (queries whose key segment is empty have no keys and get 0)."""
    seg_q = (cu_seqlens_q[1:] - cu_seqlens_q[:-1]).tolist()
    seg_kv = seg_q if cu_seqlens_kv is cu_seqlens_q else (cu_seqlens_kv[1:] - cu_seqlens_kv[:-1]).tolist()
    if seg_kv == seg_q:
        seg = [n for n in seg_q if n > 0]
        return seg, seg
    if len(seg_kv) != len(seg_q):
        from .core import SvgbError

        raise SvgbError(f"cu_seqlens_q and cu_seqlens_kv must hold the same number of segments "
                        f"({len(seg_q)} vs {len(seg_kv)})")
    pairs = [(a, b) for a, b in zip(seg_q, seg_kv) if a > 0 or b > 0]
    return [a for a, _ in pairs], [b for _, b in pairs]


def flashinfer_varlen_func(q, k, v, cu_seqlens_q, cu_seqlens_kv, max_seqlen_q, max_seqlen_kv):
    """hyvideo/attention.py:807-875: dense attention inside each cu_seqlens segment, q,k,v [B,H,S,D].  Query segment i
    attends key segment i (cu_seqlens_kv; k, v may be longer or shorter than q)."""
    from .models.common import dense_attention

    seg, seg_kv = _varlen_segments(cu_seqlens_q, cu_seqlens_kv)
    return dense_attention(q, k, v, seg, None if seg_kv is seg and k.shape[2] == q.shape[2] else seg_kv)


def flash_attn_varlen_func(q, k, v, cu_seqlens_q, cu_seqlens_kv, max_seqlen_q, max_seqlen_kv, dropout_p=0.0,
                           softmax_scale=None, causal=False, window_size=(-1, -1), softcap=0.0, alibi_slopes=None,
                           deterministic=False, return_attn_probs=False, block_table=None):
    """flash_attn.flash_attn_interface.flash_attn_varlen_func (FlashAttention 2's signature) as hyvideo/attention.py:
    452-470 calls it: q,k,v [L, B*H, D] (sequence first), segments given by cu_seqlens: query segment i attends key
    segment i (k, v may have another length than q).  causal= and window_size= mask inside each segment as
    FlashAttention does (queries aligned to the end of their key segment; core.plan_local_varlen), softmax_scale=
    replaces head_dim ** -0.5, and deterministic= is accepted (these kernels always are).  dropout_p, softcap,
    alibi_slopes, return_attn_probs and block_table other than their defaults raise SvgbError rather than being
    ignored.  Without a mask the call is the dense per-segment attention of models.common.segment_attention."""
    from .core import SvgbError

    for name, value, ok in (("dropout_p", dropout_p, dropout_p == 0.0), ("softcap", softcap, softcap == 0.0),
                            ("alibi_slopes", alibi_slopes, alibi_slopes is None),
                            ("return_attn_probs", return_attn_probs, not return_attn_probs),
                            ("block_table", block_table, block_table is None)):
        if not ok:
            shown = value if isinstance(value, (int, float, bool)) else type(value).__name__
            raise SvgbError(f"flash_attn_varlen_func: {name}={shown} is not supported (no kernel for it)")
    if causal or tuple(window_size) != (-1, -1):
        from . import core

        plan = core.plan_local_varlen(cu_seqlens_q, cu_seqlens_kv, total_q=q.shape[0], total_k=k.shape[0],
                                      causal=causal, window_size=window_size)
        return core.attention(q, k, v, plan, layout="shd", sm_scale=softmax_scale)
    from .models.common import segment_attention

    seg, seg_kv = _varlen_segments(cu_seqlens_q, cu_seqlens_kv)
    return segment_attention("flash_attn_varlen_func", q, k, v, seg, seg_kv,
                             layout="shd", sm_scale=softmax_scale)


def _is_fp8(t) -> bool:
    import torch

    return getattr(t, "dtype", None) in (torch.float8_e4m3fn, torch.float8_e5m2)


def flash_attn_with_kvcache(q, k_cache, v_cache, k=None, v=None, rotary_cos=None, rotary_sin=None, cache_seqlens=None,
                            cache_batch_idx=None, cache_leftpad=None, block_table=None, softmax_scale=None, causal=False,
                            window_size=(-1, -1), softcap=0.0, rotary_interleaved=True, alibi_slopes=None,
                            num_splits=0, return_softmax_lse=False, *, q_descale=None, k_descale=None, v_descale=None,
                            cu_seqlens_q=None, cu_seqlens_k_new=None, max_seqlen_q=None):
    """flash_attn.flash_attn_with_kvcache (FlashAttention 2's signature and return convention), forward only.
    q [B, Sq, Hq, D]; k_cache, v_cache [B_cache, S_cache, Hkv, D] (stream b in row cache_batch_idx[b], default b) or
    paged [num_pages, page_size, Hkv, D] with block_table int32 [B, max_pages] (page_size a multiple of 128).  k, v
    [B, Snew, Hkv, D], when given, are written into the cache in place at cache_seqlens[b] (core.kvcache_append), and
    the queries then attend the cache_seqlens[b] + Snew keys of their stream, aligned to its end (core.plan_kvcache),
    under causal= / window_size=.  cache_seqlens: int or device int tensor [B] (None: the whole S_cache of a contiguous
    cache); nothing is read on the host.  Returns out [B, Sq, Hq, D], and lse [B, Hq, Sq] with return_softmax_lse.
    num_splits is a scheduling hint and is ignored; rotary_cos / rotary_sin, cache_leftpad, softcap and alibi_slopes
    other than their defaults raise SvgbError rather than being ignored (video models apply their own RoPE before
    caching).
    FP8 KV cache: k_cache, v_cache of dtype torch.float8_e4m3fn with k_descale, v_descale, keyword-only and named as in
    FlashAttention 3, float32 [Hkv]: one dequantisation scale per key/value head for the whole cache (FlashAttention 3
    takes [B, Hkv], one per stream, which is refused by shape).  q stays bf16 and is quantised per query head inside the
    call; k, v stay 16-bit and are quantised by the append; out is bf16, D = 128.  An fp8 q, fp8 k / v and q_descale
    are refused.  Without k_descale / v_descale the call makes exactly the 16-bit launches.
    Variable-length streams (keyword-only, named as in FlashAttention 3): cu_seqlens_q device int [B + 1] packs stream
    b's queries at rows [cu_seqlens_q[b], cu_seqlens_q[b+1]) of q [total_q, Hq, D]; cu_seqlens_k_new, device int
    [B + 1], packs its new rows k, v [total_k_new, Hkv, D] likewise (required with k, v then), and max_seqlen_q, the
    longest stream's queries, tightens the plan.  Returns out [total_q, Hq, D] and lse [Hq, total_q].  Still one
    append, one plan and one forward (core.plan_kvcache(cu_seqlens_q=))."""
    import torch

    from . import core
    from .core import SvgbError

    for name, value, ok in (("rotary_cos", rotary_cos, rotary_cos is None), ("rotary_sin", rotary_sin, rotary_sin is None),
                            ("cache_leftpad", cache_leftpad, cache_leftpad is None),
                            ("softcap", softcap, softcap == 0.0), ("alibi_slopes", alibi_slopes, alibi_slopes is None)):
        if not ok:
            shown = value if isinstance(value, (int, float, bool)) else type(value).__name__
            raise SvgbError(f"flash_attn_with_kvcache: {name}={shown} is not supported (no kernel for it)")
    if core.needs_grad(q, k_cache, v_cache, k, v):
        raise SvgbError("flash_attn_with_kvcache has no backward: the KV-cache plan (plan_kvcache) runs forward only")
    if (k is None) != (v is None):
        raise SvgbError("flash_attn_with_kvcache: k and v are given together or not at all")
    if q_descale is not None:
        raise SvgbError("flash_attn_with_kvcache: q_descale is not supported: q is bf16 and quantised per query head "
                        "inside the call")
    for name, t in (("q", q), ("k", k), ("v", v)):
        if _is_fp8(t):
            raise SvgbError(f"flash_attn_with_kvcache: {name} is {t.dtype}; q and the new k, v rows are 16-bit (an FP8 "
                            "cache quantises them itself)")
    for name, t in (("k_descale", k_descale), ("v_descale", v_descale)):
        if t is not None and (not isinstance(t, torch.Tensor) or t.dim() != 1):
            shown = tuple(t.shape) if isinstance(t, torch.Tensor) else type(t).__name__
            raise SvgbError(f"flash_attn_with_kvcache: {name} must be [Hkv], one scale per key/value head for the whole "
                            f"cache (got {shown}; FlashAttention 3's per-stream [B, Hkv] is not supported)")
    given = k_descale is not None or v_descale is not None
    if _is_fp8(k_cache) != given or (given and (k_descale is None or v_descale is None)):
        raise SvgbError("flash_attn_with_kvcache: k_descale and v_descale (float32 [Hkv]) go together with a "
                        "float8_e4m3fn cache, and only with one")
    scales = dict(k_scale=k_descale, v_scale=v_descale) if given else {}
    if cu_seqlens_q is not None or cu_seqlens_k_new is not None or max_seqlen_q is not None:
        return _with_kvcache_varlen(q, k_cache, v_cache, k, v, cache_seqlens, cache_batch_idx, block_table,
                                    softmax_scale, causal, window_size, return_softmax_lse, scales, cu_seqlens_q,
                                    cu_seqlens_k_new, max_seqlen_q)
    B, Sq = q.shape[:2]
    if cache_seqlens is None:
        if block_table is not None:
            raise SvgbError("flash_attn_with_kvcache: a paged cache (block_table) needs cache_seqlens")
        cache_seqlens = k_cache.shape[1]
    lens = core._seqlens(cache_seqlens, B, q.device)
    if k is not None:
        core.kvcache_append(k_cache, v_cache, k, v, lens, block_table=block_table, cache_batch_idx=cache_batch_idx,
                            **scales)
    paged = block_table is not None
    plan = core.plan_kvcache(lens, q_len=Sq, num_blocks=k_cache.shape[0], new_len=0 if k is None else k.shape[1],
                             cache_len=None if paged else k_cache.shape[1], block_table=block_table,
                             page_size=k_cache.shape[1] if paged else None, cache_batch_idx=cache_batch_idx,
                             causal=causal, window_size=window_size)
    return core.attn_fwd(q, k_cache, v_cache, plan, return_lse=return_softmax_lse, sm_scale=softmax_scale, **scales)


def _with_kvcache_varlen(q, k_cache, v_cache, k, v, cache_seqlens, cache_batch_idx, block_table, softmax_scale, causal,
                        window_size, return_softmax_lse, scales, cu_seqlens_q, cu_seqlens_k_new, max_seqlen_q):
    """flash_attn_with_kvcache with FlashAttention 3's variable-length keywords: core.kvcache_append(cu_seqlens=),
    core.plan_kvcache(cu_seqlens_q=) and core.attn_fwd on q [total_q, Hq, D]."""
    from . import core
    from .core import SvgbError

    if cu_seqlens_q is None:
        raise SvgbError("flash_attn_with_kvcache: cu_seqlens_k_new and max_seqlen_q go with cu_seqlens_q (variable-length "
                        "queries)")
    if (k is None) != (cu_seqlens_k_new is None):
        raise SvgbError("flash_attn_with_kvcache: with cu_seqlens_q, new rows k, v [total_k_new, Hkv, D] come with "
                        "cu_seqlens_k_new, and cu_seqlens_k_new only with them")
    if q.dim() != 3:
        raise SvgbError(f"flash_attn_with_kvcache: with cu_seqlens_q, q must be [total_q, Hq, D] (got {tuple(q.shape)})")
    cu_q = core._cu_seqlens("flash_attn_with_kvcache", "cu_seqlens_q", cu_seqlens_q, None, q.device)
    B = cu_q.numel() - 1
    if cu_seqlens_k_new is not None:  # refused here, before the append launches
        cu_seqlens_k_new = core._cu_seqlens("flash_attn_with_kvcache", "cu_seqlens_k_new", cu_seqlens_k_new, B, q.device)
    if max_seqlen_q is not None and not 1 <= int(max_seqlen_q) <= q.shape[0]:
        raise SvgbError(f"flash_attn_with_kvcache: max_seqlen_q={max_seqlen_q} must lie in [1, total_q={q.shape[0]}]")
    if cache_seqlens is None:
        if block_table is not None:
            raise SvgbError("flash_attn_with_kvcache: a paged cache (block_table) needs cache_seqlens")
        cache_seqlens = k_cache.shape[1]
    lens = core._seqlens(cache_seqlens, B, q.device)
    if k is not None:
        core.kvcache_append(k_cache, v_cache, k, v, lens, block_table=block_table, cache_batch_idx=cache_batch_idx,
                            cu_seqlens=cu_seqlens_k_new, **scales)
    paged = block_table is not None
    plan = core.plan_kvcache(lens, cu_seqlens_q=cu_q, total_q=q.shape[0], max_seqlen_q=max_seqlen_q,
                             cu_seqlens_new=cu_seqlens_k_new, num_blocks=k_cache.shape[0],
                             cache_len=None if paged else k_cache.shape[1], block_table=block_table,
                             page_size=k_cache.shape[1] if paged else None, cache_batch_idx=cache_batch_idx,
                             causal=causal, window_size=window_size)
    return core.attn_fwd(q, k_cache, v_cache, plan, return_lse=return_softmax_lse, sm_scale=softmax_scale, **scales)


def _model_of(module):
    name = getattr(module, "__name__", "")
    for m in ("hyvideo", "wan", "cosmos", "cog"):
        if f".{m}." in name or name.endswith("." + m):
            return m
    return None


_NAMES_FP8 = {
    "dynamic_block_sparse_fwd_flashinfer": _ku.dynamic_block_sparse_fwd_flashinfer_fp8,
    "dynamic_block_sparse_fwd_triton": _ku.dynamic_block_sparse_fwd_triton_fp8,
}


def install(module, sample_mse: bool = True, fp8: bool = False) -> list:
    """Replace every operator name the module already defines (the reference resolves them as module globals,
    svg/models/hyvideo/attention.py:12-28).  Besides the kernels this covers the module-level attention entry points
    `flex_attention`, `prepare_flexattention`, `flashinfer_varlen_func`, `flash_attn_varlen_func`, and — with
    sample_mse=True — the processors' `sample_mse` method (the reference version needs the materialised
    [10000, S] profiling masks in `attention_masks`; ours evaluates them analytically).  fp8=True installs FP8 (e4m3,
    head_dim 128) versions of the sparse attention calls, `flex_attention` and `dynamic_block_sparse_fwd_flashinfer` /
    `_triton`; profiling, k-means, the maps, the permutations and the dense calls stay 16-bit.  Returns the names
    replaced."""
    done = []
    names = {**_NAMES, **_NAMES_FP8} if fp8 else _NAMES
    for name, fn in names.items():
        if hasattr(module, name):
            setattr(module, name, fn)
            done.append(name)
    for name, fn in (("flex_attention", flex_attention_fp8 if fp8 else flex_attention),
                     ("flashinfer_varlen_func", flashinfer_varlen_func),
                     ("flash_attn_varlen_func", flash_attn_varlen_func)):
        if hasattr(module, name):
            setattr(module, name, fn)
            done.append(name)
    model = _model_of(module)
    if model is not None and hasattr(module, "prepare_flexattention"):
        from .models import cog, hyvideo, wan

        module.prepare_flexattention = {"hyvideo": hyvideo, "wan": wan, "cosmos": wan, "cog": cog}[model].prepare_flexattention
        done.append("prepare_flexattention")
    if sample_mse and model is not None:
        layout = {"hyvideo": 0, "wan": 1, "cosmos": 1, "cog": 2}[model]
        for obj in vars(module).values():
            if isinstance(obj, type) and "sample_mse" in vars(obj):
                obj.sample_mse = _make_sample_mse(layout)
                done.append(f"{obj.__name__}.sample_mse")
    return done


def _make_sample_mse(layout: int):
    def sample_mse(self, query, key, value):
        """<Model>_SVGAttn_Processor.sample_mse (hyvideo/attention.py:375-399) on the svgb200 kernel: same sampled
        rows (CPU generator, :381), same [2, cfg, H] result in query.dtype; the profiling masks are evaluated
        analytically, `attention_masks` is not needed."""
        import torch

        from . import core

        cfg, H, S, D = query.shape
        n = min(self.num_sampled_rows, S)
        high = S if layout == 2 else self.sample_mse_max_row  # cog/attention.py:124 samples the whole sequence
        rows = torch.randint(low=0, high=high, size=(n,))
        mse = core.sample_mse(query.reshape(cfg * H, S, D), key.reshape(cfg * H, S, D), value.reshape(cfg * H, S, D),
                              rows.to(query.device), layout, self.context_length, self.num_frame, self.frame_size)
        mse = mse.view(2, cfg, H).to(query.dtype)
        if layout == 2:  # empty text rows of the Cog temporal mask -> NaN in the reference (cog/utils.py:76-86)
            text_row = (rows < self.context_length).any().to(query.device)
            mse[1] = torch.where(text_row, torch.full_like(mse[1], float("nan")), mse[1])
        return mse

    return sample_mse


def install_kmeans_utils(module=None) -> list:
    if module is None:
        import svg.kmeans_utils as module  # noqa: WPS433 (the reference must be importable)
    names = ["batch_kmeans_Euclid", "density_calculation", "dynamic_block_sparse_fwd_flashinfer",
             "dynamic_block_sparse_fwd_triton", "identify_dynamic_map", "euclid_assign_triton",
             "triton_centroid_update_sorted_euclid"]
    for n in names:
        setattr(module, n, getattr(_ku, n))
    return names


def install_native_kernels() -> None:
    """Make `import _kernels` (svg/models/*/attention.py: `sys.path.append("svg/kernels/build/"); import _kernels`)
    resolve to the svgb200 implementation, so the reference's ENABLE_FAST_KERNEL branch runs these kernels."""
    import sys

    from . import _kernels as k

    sys.modules["_kernels"] = k


def install_triton_glue(module) -> list:
    """Replace the Triton glue names a reference module imported (svg/models/wan/custom_models.py:16-17,
    svg/models/wan/attention.py:16)."""
    from . import triton_glue as g

    done = []
    for name in ("triton_rmsnorm_forward", "triton_layernorm_forward", "triton_modulate_shift_forward",
                 "triton_modulate_gate_residual_forward"):
        if hasattr(module, name):
            setattr(module, name, getattr(g, name))
            done.append(name)
    return done
