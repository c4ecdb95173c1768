"""Shared host logic of the SVG1 / SVG2 attention cores (what attention_core_logic does between the QKV
projection and the output projection in svg/models/<m>/attention.py)."""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Optional

import torch

from .. import core
from ..timer import time_logging_decorator
from ..kmeans_utils import batch_kmeans_Euclid, batch_kmeans_Euclid_sorted


def sparsity_to_width(sparsity, context_length, num_frame, frame_size):
    """svg/models/hyvideo/utils.py:142-151 (identical in wan / cog)."""
    seq_len = context_length + num_frame * frame_size
    total_elements = seq_len ** 2
    sparsity = (sparsity * total_elements - 2 * seq_len * context_length) / total_elements
    width = seq_len * (1 - math.sqrt(1 - sparsity))
    return width / frame_size


@dataclass
class BandMask:
    """What the reference's torch BlockMask is to flex_attention: the compiled executed mask.
    Built once (prepare_flexattention) and shared by every head / layer / step."""
    plan: core.AttnPlan
    mode: int
    m0: int
    m1: int
    m2: int
    seq_len: int


def sparse_flex_attention(query, key, value, block_mask: BandMask):
    """hyvideo/attention.py:401-403: flex_attention(q, k, v, block_mask=...)  [cfg,H,S,D].  Differentiable when an input
    requires grad (core.attention)."""
    return core.attention(query, key, value, block_mask.plan)


def check_fp8_head_dim(D):
    if D != 128:
        raise core.SvgbError(f"fp8 attention needs head_dim 128 (got {D}): the e4m3 kernel is built for 128-byte rows")


def quantize_qkv(query, key, value):
    """Per-head e4m3 quantisation of Q, K, V -> ((q8, s_q), (k8, s_k), (v8, s_v))."""
    return tuple(core.quantize_e4m3(t) for t in (query, key, value))


def fp8_attention(query, key, value, plan: core.AttnPlan, **rows):
    """Attention under `plan` in FP8: Q, K, V [B,H,S,128] quantised to e4m3 per head and run on the e4m3 kernel
    (rows: q_rows / kv_rows / o_rows of core.attn_fwd_fp8).  The kernel writes bf16; the result comes back in
    query.dtype.  FP8 attention has no backward: an input that requires grad raises."""
    core._no_backward("fp8 attention", query, key, value)
    check_fp8_head_dim(query.shape[-1])
    (q8, sq), (k8, sk), (v8, sv) = quantize_qkv(query, key, value)
    return core.attn_fwd_fp8(q8, k8, v8, sq, sk, sv, plan, **rows).to(query.dtype)


def sparse_flex_attention_fp8(query, key, value, block_mask: BandMask):
    """sparse_flex_attention in FP8 (fp8_attention under the band plan)."""
    core._no_backward("fp8 attention", query, key, value)
    check_fp8_head_dim(query.shape[-1])  # before block_mask is read: a head_dim-64 model fails on its cause
    return fp8_attention(query, key, value, block_mask.plan)


def check_segments(what, segs, kv_segs, S, S_kv):
    """Segment lists that pair query segment i with key segment i must be as many and sum to the two lengths: the plan's
    block sizes are not checked on the device, and key blocks past S_kv would have dK / dV rows stored past the end of
    k's gradient.  Only the call with equal lengths and equal lists skips this check, as it did before S_kv existed."""
    if S_kv == S and kv_segs == segs:
        return
    if len(kv_segs) != len(segs) or sum(segs) != S or sum(kv_segs) != S_kv:
        raise core.SvgbError(f"{what}: query segments {segs} must sum to {S} and key segments {kv_segs} to {S_kv}, "
                             "one key segment per query segment")


def segment_attention(what, query, key, value, segs, kv_segs, layout="bhsd", sm_scale=None):
    """core.attention in which query segment i attends key segment i only: the segment lists pass check_segments
    (`what` names the caller in its error), then one rectangular plan of the diagonal block map over them.  layout
    'bhsd' or 'shd', as core.attention takes it.  The map is built over key's heads, so key / value may have fewer
    heads than query (grouped-query attention).  sm_scale: the softmax scale (None: head_dim ** -0.5)."""
    seq = 2 if layout == "bhsd" else 0
    S, S_kv = query.shape[seq], key.shape[seq]
    check_segments(what, segs, kv_segs, S, S_kv)
    BH = key.shape[0] * key.shape[1] if layout == "bhsd" else key.shape[1]
    n, dev = len(segs), query.device
    bm = torch.eye(n, dtype=torch.bool, device=dev).expand(BH, n, n).contiguous()
    sz = torch.tensor(segs, dtype=torch.int32, device=dev).expand(BH, n).contiguous()
    kv_sz = sz if kv_segs == segs else torch.tensor(kv_segs, dtype=torch.int32, device=dev).expand(BH, n).contiguous()
    plan = core.plan_varblock(bm, sz, kv_sz, S, S_kv=S_kv)
    if sm_scale is None:
        return core.attention(query, key, value, plan, layout=layout)
    return core.attention(query, key, value, plan, layout=layout, sm_scale=sm_scale)


def segment_lengths(cu_seqlens):
    """The non-empty segment lengths of one cu_seqlens row, as a host list."""
    return [s for s in (cu_seqlens[1:] - cu_seqlens[:-1]).tolist() if s > 0]


def dense_attention(query, key, value, seg_lens=None, kv_seg_lens=None):
    """Dense fall-back (b11).  seg_lens: optional list of segment lengths that only attend inside
    themselves (HunyuanVideo's padded-prompt varlen split, hyvideo/attention.py:308-316,807-875).
    key / value may be longer or shorter than query (cross-attention, [cfg,H,S_kv,D]); kv_seg_lens then gives their
    segments, query segment i attending key segment i (None: the whole key sequence, or seg_lens when the lengths
    match).  Differentiable when an input requires grad (core.attention)."""
    S, S_kv = query.shape[2], key.shape[2]
    segs = [S] if seg_lens is None else [int(x) for x in seg_lens]
    if kv_seg_lens is None and seg_lens is None:
        kv_segs = [S_kv]
    elif kv_seg_lens is None and S_kv == S:
        kv_segs = segs
    elif kv_seg_lens is None:
        raise core.SvgbError(f"dense_attention: {len(segs)} query segments and a key sequence of another length "
                             f"({S} vs {S_kv}) need kv_seg_lens")
    else:
        kv_segs = [int(x) for x in kv_seg_lens]
    return segment_attention("dense_attention", query, key, value, segs, kv_segs)


class KMeansState:
    """Centroids persist across diffusion steps and warm-start the next call (hyvideo/attention.py:
    566-626 keeps them in class-level dicts keyed by layer; wan keeps them per processor instance)."""

    def __init__(self):
        self.q_centroids = {}
        self.k_centroids = {}

    def cluster(self, key, query, kmat, num_q, num_k, iters_init, iters_step, sorted_members=False):
        """query/kmat: [BH, N, D] (views with a larger head stride are clustered in place).  Returns (qlabels, qcent,
        qsizes, klabels, kcent, ksizes); with sorted_members the labels are int32 and the stable argsorts of both label
        sets are appended (q_perm, k_perm)."""
        run = batch_kmeans_Euclid_sorted if sorted_members else batch_kmeans_Euclid
        if key not in self.q_centroids:
            rq = run(query, num_q, max_iters=iters_init)
            rk = run(kmat, num_k, max_iters=iters_init)
        else:
            rq = run(query, num_q, max_iters=iters_step, init_centroids=self.q_centroids[key])
            rk = run(kmat, num_k, max_iters=iters_step, init_centroids=self.k_centroids[key])
        self.q_centroids[key] = rq[1]
        self.k_centroids[key] = rk[1]
        if sorted_members:
            return rq[0], rq[1], rq[2], rk[0], rk[1], rk[2], rq[4], rk[4]
        return rq[0], rq[1], rq[2], rk[0], rk[1], rk[2]


class SVG1Core:
    """Sparse VideoGen v1 attention core: online profiling -> head placement -> one band mask -> inverse
    placement (svg/models/hyvideo/attention.py:473-524; wan :284-328; cosmos :200-238; cog :164-196).

    Subclasses fix the text layout (`text_first`, `smse_layout`) and build `block_mask`.

    fp8=True runs the band attention on e4m3 Q, K, V (sparse_flex_attention_fp8, head_dim 128 only); sample_mse, the
    placements and the dense branch stay 16-bit, so the head choice is the 16-bit core's.

    Gradients: sparse_core (16-bit) is differentiable in Q, K and V through the placements (core._HeadPlacement) and
    the band attention (core.attention); the head choice of sample_mse is a constant.  The FP8 core,
    sparse_core_head_parallel and sparse_core_from_host have no backward and raise under grad."""

    text_first = False
    smse_layout = 0  # svgb_sample_mse layout id (0 = HY text-last band 1.5*P, 1 = WAN sink band 2*P)

    def __init__(self, context_length, num_frame, frame_size, num_sampled_rows=64, sample_mse_max_row=10000,
                 first_layers_fp=0, first_times_fp=0, layer_idx=0, fp8=False):
        self.context_length, self.num_frame, self.frame_size = context_length, num_frame, frame_size
        self.num_sampled_rows, self.sample_mse_max_row = num_sampled_rows, sample_mse_max_row
        self.first_layers_fp, self.first_times_fp, self.layer_idx = first_layers_fp, first_times_fp, layer_idx
        self.fp8 = fp8
        self.block_mask: Optional[BandMask] = None

    # -- reference method names ---------------------------------------------------------------------
    def sample_mse(self, query, key, value, sampled_rows=None):
        """hyvideo/attention.py:375-399 -> [2, cfg, H] in query.dtype (0 = spatial, 1 = temporal).
        `sampled_rows` defaults to torch.randint on the CPU generator exactly like the reference (:381)."""
        cfg, H, S, D = query.shape
        n = min(self.num_sampled_rows, S)
        if sampled_rows is None:
            sampled_rows = torch.randint(low=0, high=self.sample_mse_max_row, size=(n,))
        rows = sampled_rows.to(query.device, non_blocking=True)
        mse = core.sample_mse(query.view(cfg * H, S, D), key.view(cfg * H, S, D), value.view(cfg * H, S, D), rows,
                              self.smse_layout, self.context_length, self.num_frame, self.frame_size)
        return mse.view(2, cfg, H).to(query.dtype)

    def sparse_flex_attention(self, query, key, value, block_mask):
        if self.fp8:
            return sparse_flex_attention_fp8(query, key, value, block_mask)
        return sparse_flex_attention(query, key, value, block_mask)

    def fast_sparse_head_placement(self, query, key, value, query_out, key_out, value_out, best_mask_idx,
                                   context_length, num_frame, frame_size):
        core.head_placement([query, key, value], [query_out, key_out, value_out], best_mask_idx, context_length,
                            num_frame, frame_size, text_first=self.text_first)
        return query_out, key_out, value_out

    def fast_hidden_states_placement(self, hidden_states, output_hidden_states, best_mask_idx, context_length,
                                     num_frame, frame_size):
        core.head_placement([hidden_states], [output_hidden_states], best_mask_idx, context_length, num_frame,
                            frame_size, text_first=self.text_first, inverse=True)

    # -- the sparse branch ---------------------------------------------------------------------------
    def sparse_core(self, query, key, value, sampled_rows=None, attn_events=None):
        if self.fp8:
            core._no_backward("the SVG1 core with fp8 attention", query, key, value)
        # stage labels = the reference's TIME_BENCH table (hyvideo/attention.py:375,401,405,439)
        with time_logging_decorator("Level 3 - sample mse"):
            sampled_mses = self.sample_mse(query, key, value, sampled_rows)
            best_mask_idx = torch.argmin(sampled_mses, dim=0)  # ties -> 0 (spatial), like the reference (:508)
        with time_logging_decorator("Level 3 - fast sparse head placement"):
            q_out, k_out, v_out = torch.empty_like(query), torch.empty_like(key), torch.empty_like(value)
            self.fast_sparse_head_placement(query, key, value, q_out, k_out, v_out, best_mask_idx,
                                            self.context_length, self.num_frame, self.frame_size)
        if attn_events is not None:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
        with time_logging_decorator("Level 3 - sparse flex attention"):
            hidden = self.sparse_flex_attention(q_out, k_out, v_out, self.block_mask)
        if attn_events is not None:
            b.record()
            attn_events.append((a, b))
        with time_logging_decorator("Level 3 - fast hidden states placement"):
            out = torch.empty_like(query)
            self.fast_hidden_states_placement(hidden, out, best_mask_idx, self.context_length, self.num_frame,
                                              self.frame_size)
        return out

    def sparse_core_head_parallel(self, query, key, value, hp, sampled_rows=None, out=None, attn_events=None,
                                  trace=None):
        """Same as sparse_core on this rank's heads ([1, H_local, S, D]), with the output all-gather of every
        head issued on a side stream as soon as that head's attention + inverse placement finished, so the
        NVLink transfer of head i overlaps the attention of head i+1 (svgb200.parallel.HeadParallel).
        Returns the full [1, H_local * world, S, D] output (heads interleaved: global h = i*world + rank)."""
        # the output is assembled by all-gathers into a plain buffer, outside the autograd graph
        core._no_backward("the head-parallel SVG1 core (sparse_core_head_parallel)", query, key, value)
        cfg, Hl, S, D = query.shape
        assert cfg == 1
        if trace is not None:
            t0 = torch.cuda.Event(enable_timing=True)
            t0.record()
            trace["t0"] = t0
        sampled_mses = self.sample_mse(query, key, value, sampled_rows)
        best_mask_idx = torch.argmin(sampled_mses, dim=0)
        q_out, k_out, v_out = torch.empty_like(query), torch.empty_like(key), torch.empty_like(value)
        self.fast_sparse_head_placement(query, key, value, q_out, k_out, v_out, best_mask_idx, self.context_length,
                                        self.num_frame, self.frame_size)

        def one_head(i):
            if attn_events is not None:
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
            hid = self.sparse_flex_attention(q_out[:, i:i + 1], k_out[:, i:i + 1], v_out[:, i:i + 1], self.block_mask)
            if attn_events is not None:
                b.record()
                attn_events.append((a, b))
            o = torch.empty_like(hid)
            self.fast_hidden_states_placement(hid, o, best_mask_idx[:, i:i + 1].contiguous(), self.context_length,
                                              self.num_frame, self.frame_size)
            return o

        return hp.run_overlapped(one_head, Hl, S, D, query.dtype, query.device, out=out, trace=trace)

    def sparse_core_from_host(self, hq, hk, hv, ho, sampled_rows=None, heads_per_stage=2, hp=None, gathered=None):
        """End-to-end entry for callers whose Q/K/V live in (pinned) host memory: heads are streamed through
        a 3-stage pipeline — H2D copy of group g+1 | compute of group g | D2H copy of group g-1 — on three
        CUDA streams, so the PCIe transfers hide behind the attention.

        Head-parallel (hp = svgb200.parallel.HeadParallel, world > 1): hq/hk/hv/ho hold this rank's heads; each
        group's output is additionally all-gathered into `gathered` [1, H_local*world, S, D] on the device (the
        downstream projection needs every head) on hp's communication stream, overlapping the next group."""
        # heads travel through staging copies, outside the autograd graph
        core._no_backward("the host-pipelined SVG1 core (sparse_core_from_host)", hq, hk, hv)
        cfg, H, S, D = hq.shape
        assert cfg == 1
        dev = self.block_mask.plan.ws.device
        if not hasattr(self, "_pipe"):
            self._pipe = {"h2d": torch.cuda.Stream(dev), "d2h": torch.cuda.Stream(dev), "bufs": {}}
        P_ = self._pipe
        G = heads_per_stage
        key = (G, S, D, hq.dtype)
        if key not in P_["bufs"]:
            P_["bufs"][key] = [[torch.empty(1, G, S, D, dtype=hq.dtype, device=dev) for _ in range(4)] for _ in range(2)]
        bufs = P_["bufs"][key]
        cur = torch.cuda.current_stream(dev)
        if sampled_rows is None:
            sampled_rows = torch.randint(low=0, high=self.sample_mse_max_row, size=(min(self.num_sampled_rows, S),))
        rows_dev = sampled_rows.to(dev, non_blocking=True)
        # slot reuse ACROSS calls: the staging buffers are still being read by the previous call's last head groups
        # (queued on `cur`) and drained by its D2H copies -> this call's first H2D copies must wait for both
        P_["h2d"].wait_stream(cur)
        P_["h2d"].wait_stream(P_["d2h"])
        groups = [(g0, min(H, g0 + G)) for g0 in range(0, H, G)]
        ready, done_compute, done_d2h, gather_done = {}, {}, {}, {}

        def issue_h2d(gi):
            g0, g1 = groups[gi]
            slot = bufs[gi & 1]
            with torch.cuda.stream(P_["h2d"]):
                if gi >= 2:
                    P_["h2d"].wait_event(done_d2h[gi - 2])  # slot reuse: its output must have left first
                    if (gi - 2) in gather_done:
                        P_["h2d"].wait_event(gather_done[gi - 2])
                for dst, src in zip(slot[:3], (hq, hk, hv)):
                    dst[:, : g1 - g0].copy_(src[:, g0:g1], non_blocking=True)
                ev = torch.cuda.Event()
                ev.record(P_["h2d"])
                ready[gi] = ev

        issue_h2d(0)
        for gi, (g0, g1) in enumerate(groups):
            if gi + 1 < len(groups):
                issue_h2d(gi + 1)
            slot = bufs[gi & 1]
            n = g1 - g0
            cur.wait_event(ready[gi])
            o = self.sparse_core(slot[0][:, :n], slot[1][:, :n], slot[2][:, :n], sampled_rows=rows_dev)
            slot[3][:, :n].copy_(o)
            ev = torch.cuda.Event()
            ev.record(cur)
            done_compute[gi] = ev
            if hp is not None and hp.world > 1:
                import torch.distributed as dist

                comm, _ = hp.streams(dev)
                with torch.cuda.stream(comm):
                    comm.wait_event(ev)
                    for i in range(n):
                        dist.all_gather_into_tensor(gathered[0, (g0 + i) * hp.world:(g0 + i + 1) * hp.world],
                                                    slot[3][0, i:i + 1], group=hp.group)
                    evg = torch.cuda.Event()
                    evg.record(comm)
                gather_done[gi] = evg
            with torch.cuda.stream(P_["d2h"]):
                P_["d2h"].wait_event(ev)
                ho[:, g0:g1].copy_(slot[3][:, :n], non_blocking=True)
                ev2 = torch.cuda.Event()
                ev2.record(P_["d2h"])
                done_d2h[gi] = ev2
        cur.wait_stream(P_["d2h"])
        if hp is not None and hp.world > 1:
            cur.wait_stream(hp.streams(dev)[0])
        return ho

    def dense_core(self, query, key, value, cu_max_seqlens=None):
        seg = None if cu_max_seqlens is None else segment_lengths(cu_max_seqlens[0])
        with time_logging_decorator("Level 3 - Dense Flash Attention"):
            return dense_attention(query, key, value, seg)

    def attention_core_logic(self, query, key, value, timestep, layer_idx=None, cu_max_seqlens=None):
        cfg, H, S, D = query.shape
        assert S == self.context_length + self.num_frame * self.frame_size, (
            f"Query Shape: {S} is not equivalent to {self.context_length} + {self.num_frame} * {self.frame_size}")
        full = self.layer_idx < self.first_layers_fp or bool(timestep[0] > self.first_times_fp)
        if full:
            return self.dense_core(query, key, value, cu_max_seqlens)
        return self.sparse_core(query, key, value)


class SAPCore:
    """Sparse VideoGen v2 (semantic-aware permutation) attention core
    (svg/models/hyvideo/attention.py:555-804; wan :375-559; cosmos :290-469).

    k-means on Q and K -> centroid top-p dynamic map -> permute Q,K,V by cluster -> variable-block sparse
    attention -> inverse permutation.  Here the inverse permutation is fused into the attention epilogue
    (o_rows) and the text tokens ride the same gather (no write-back copies).

    fp8=True runs the sparse attention on e4m3 Q, K, V (head_dim 128 only): the un-permuted tensors are quantised per
    head and the row-gather kernel reads them through the cluster permutations, so no permuted copy is made.
    k-means, the dynamic map and the dense branch stay 16-bit, so the maps and permutations are the 16-bit core's."""

    def __init__(self, context_length, num_frame, frame_size, num_q_centroids, num_k_centroids, top_p_kmeans,
                 min_kc_ratio, kmeans_iter_init, kmeans_iter_step, prompt_length=0, zero_step_kmeans_init=False,
                 first_layers_fp=0, first_times_fp=0, layer_idx=0, state: Optional[KMeansState] = None,
                 logging_file: Optional[str] = None, fp8=False):
        self.fp8 = fp8
        self.context_length, self.num_frame, self.frame_size = context_length, num_frame, frame_size
        self.prompt_length = prompt_length
        self.logging_file = logging_file  # density JSONL (hyvideo/attention.py:786-802); None = off
        self.num_q_centroids, self.num_k_centroids = num_q_centroids, num_k_centroids
        self.top_p_kmeans, self.min_kc_ratio = top_p_kmeans, min_kc_ratio
        self.kmeans_iter_init, self.kmeans_iter_step = kmeans_iter_init, kmeans_iter_step
        self.zero_step_kmeans_init = zero_step_kmeans_init
        self.first_layers_fp, self.first_times_fp, self.layer_idx = first_layers_fp, first_times_fp, layer_idx
        self.state = state if state is not None else KMeansState()
        self.last = {}

    def kmeans_clustering(self, query_video, key_video, layer_idx, sorted_members=False):
        BH, N, D = query_video.shape[0] * query_video.shape[1], query_video.shape[2], query_video.shape[3]
        as3 = (lambda t: t[0]) if query_video.shape[0] == 1 else (lambda t: t.reshape(BH, N, D))  # keep views views
        return self.state.cluster(layer_idx, as3(query_video), as3(key_video),
                                  self.num_q_centroids, self.num_k_centroids, self.kmeans_iter_init,
                                  self.kmeans_iter_step, sorted_members=sorted_members)

    def _text_constants(self, H, V, S, dev):
        """Identity order of the text tokens and the (prompt, padding) block sizes; built once per shape (a fresh
        torch.tensor(..., device=) per call is a synchronous pageable copy)."""
        key = (H, V, S, str(dev), self.prompt_length)
        if getattr(self, "_text_key", None) != key:
            ctx = S - V
            self._text_tail = torch.arange(V, S, device=dev, dtype=torch.int32).expand(H, ctx)
            self._text_extra = torch.tensor([self.prompt_length, ctx - self.prompt_length], dtype=torch.int32,
                                            device=dev).expand(H, 2)
            self._text_key = key
        return self._text_tail, self._text_extra

    def log_density(self, timestep, layer_idx, dyn_map, q_sizes, k_sizes):
        """One JSON line per sparse call in the reference's schema (hyvideo/attention.py:786-802), read by
        svg/utils/density.py and densities_get_mean.py: {"timestep", "layer", "avg_density", "density"}."""
        import json

        from ..kmeans_utils import density_calculation

        H = dyn_map.shape[0]
        densities = density_calculation(dyn_map[None], q_sizes.view(1, H, -1), k_sizes.view(1, H, -1))
        t = timestep[0].item() if hasattr(timestep, "__getitem__") else timestep
        entry = {"timestep": t, "layer": layer_idx, "avg_density": densities.mean().item(),
                 "density": densities.tolist()}
        with open(self.logging_file, "a") as f:
            f.write(json.dumps(entry) + "\n")
        return entry

    def sparse_core(self, query, key, value, layer_idx=None, timestep=None):
        from ..kmeans_utils import identify_dynamic_map

        cfg, H, S, D = query.shape
        assert cfg == 1, "Batch size must be 1 for kmeans block sparse attention"
        # the permutations and the fused inverse-permutation store have no backward
        core._no_backward("the SVG2 sparse core (clustered permutation, o_rows)", query, key, value)
        if self.fp8:
            check_fp8_head_dim(D)
        layer_idx = self.layer_idx if layer_idx is None else layer_idx
        ctx, V = self.context_length, self.num_frame * self.frame_size
        dev = query.device
        # the video part is clustered in place (a strided view; the reference packs it with .contiguous()), and the
        # cluster-sorted token order comes back from the last centroid update instead of two more argsort passes
        qv = query[:, :, :V] if ctx else query
        kv = key[:, :, :V] if ctx else key
        with time_logging_decorator("Level 3.5 - kmeans clustering"):
            ql, qc, qs, kl, kc, ks, q_perm, k_perm = self.kmeans_clustering(qv, kv, layer_idx, sorted_members=True)
        QC, KC = self.num_q_centroids, self.num_k_centroids
        dyn = identify_dynamic_map(qc.view(cfg, H, QC, D), kc.view(cfg, H, KC, D), qs.view(cfg, H, QC),
                                   ks.view(cfg, H, KC), self.top_p_kmeans, self.min_kc_ratio).view(H, QC, KC)
        row_sz, col_sz = qs.view(H, QC), ks.view(H, KC)
        if ctx:
            # HunyuanVideo: prompt block <-> everything but the padding, padding <-> itself
            # (dynamic_map_post_processing, hyvideo/attention.py:657-702)
            tail, extra = self._text_constants(H, V, S, dev)
            q_perm = torch.cat([q_perm, tail], dim=1)
            k_perm = torch.cat([k_perm, tail], dim=1)
            dyn = torch.nn.functional.pad(dyn, (0, 2, 0, 2), value=False)
            dyn[:, -2, :-1] = True
            dyn[:, :-1, -2] = True
            dyn[:, -1, -1] = True
            row_sz = torch.cat([row_sz, extra], dim=1)
            col_sz = torch.cat([col_sz, extra], dim=1)
        if self.fp8:
            with time_logging_decorator("Level 3 - fp8 quantization"):
                (q8, sq), (k8, sk), (v8, sv) = quantize_qkv(query, key, value)
            with time_logging_decorator("Level 3 - sparse flashinfer attention"):
                plan = core.plan_varblock(dyn, row_sz, col_sz, S, gather=True)
                out = core.attn_fwd_fp8(q8, k8, v8, sq, sk, sv, plan, q_rows=q_perm, kv_rows=k_perm,
                                        o_rows=q_perm).to(query.dtype)
        else:
            with time_logging_decorator("Level 3 - semantic aware permutation"):
                qp = core.permute_gather(query, q_perm)
                kp = core.permute_gather(key, k_perm)
                vp = core.permute_gather(value, k_perm)
            with time_logging_decorator("Level 3 - sparse flashinfer attention"):
                plan = core.plan_varblock(dyn, row_sz, col_sz, S)
                out = core.attn_fwd(qp, kp, vp, plan, o_rows=q_perm)  # inverse permutation fused into the store
        self.last = {"dynamic_map": dyn, "q_sizes": row_sz, "k_sizes": col_sz, "q_sorted_indices": q_perm,
                     "k_sorted_indices": k_perm}
        if self.logging_file is not None:
            with time_logging_decorator("Level 3 - density calculation and logging"):
                self.log_density(0 if timestep is None else timestep, layer_idx, dyn, row_sz, col_sz)
        return out

    def sparse_core_head_parallel(self, query, key, value, hp, layer_idx=None, timestep=None, out=None):
        """SVG2 core on this rank's heads ([1, H_local, S, D], interleaved ownership: global head = i * world + rank),
        followed by the output all-gather (svgb200.parallel.HeadParallel).  Every SVG2 stage is independent per head
        (k-means, dynamic map, permutation, attention), so no other exchange is needed; the centroid state of this
        object covers the local heads only.  Returns [1, H_local * world, S, D]."""
        o_local = self.sparse_core(query, key, value, layer_idx, timestep)
        return hp.gather_heads(o_local, out=out)

    def attention_core_logic(self, query, key, value, timestep, layer_idx=None, cu_max_seqlens=None):
        cfg, H, S, D = query.shape
        layer_idx = self.layer_idx if layer_idx is None else layer_idx
        assert S == self.context_length + self.num_frame * self.frame_size
        full = self.layer_idx < self.first_layers_fp or bool(timestep[0] > self.first_times_fp)
        if full:
            if self.zero_step_kmeans_init:
                V = self.num_frame * self.frame_size
                self.kmeans_clustering(query[:, :, :V].contiguous(), key[:, :, :V].contiguous(), layer_idx)
            seg = None if cu_max_seqlens is None else segment_lengths(cu_max_seqlens[0])
            return dense_attention(query, key, value, seg)
        return self.sparse_core(query, key, value, layer_idx, timestep)
