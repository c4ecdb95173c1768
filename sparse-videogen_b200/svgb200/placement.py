"""Mirror of svg/models/{hyvideo,wan,cosmos,cog}/placement.py: SVG1 head placement and its inverse.

hunyuan_sparse_head_placement(q,k,v,q_out,k_out,v_out,best_mask_idx,ctx,F,P) writes the outs in place
(placement.py:124-153); *_hidden_states_placement(h, h_out, best_mask_idx, ctx, F, P) is the inverse on O
(placement.py:360-387).  wan / cosmos share the text-last kernel (ctx = 0); cog is text-first.

Differentiable when an input requires grad: the caller's outs carry the history and the backward is the placement in
the opposite direction (core._HeadPlacement); best_mask_idx is a constant.
"""
from __future__ import annotations

from . import core


def _fwd(text_first):
    def f(query, key, value, query_out, key_out, value_out, best_mask_idx, context_length, num_frame, frame_size):
        core.head_placement([query, key, value], [query_out, key_out, value_out], best_mask_idx, context_length,
                            num_frame, frame_size, text_first=text_first, inverse=False)
    return f


def _inv(text_first):
    def f(hidden_states, hidden_states_out, best_mask_idx, context_length, num_frame, frame_size):
        core.head_placement([hidden_states], [hidden_states_out], best_mask_idx, context_length, num_frame,
                            frame_size, text_first=text_first, inverse=True)
        return hidden_states_out
    return f


hunyuan_sparse_head_placement = _fwd(False)
hunyuan_hidden_states_placement = _inv(False)
wan_sparse_head_placement = _fwd(False)
wan_hidden_states_placement = _inv(False)
cosmos_sparse_head_placement = _fwd(False)
cosmos_hidden_states_placement = _inv(False)
cog_sparse_head_placement = _fwd(True)
cog_hidden_states_placement = _inv(True)
# svg/models/cog/placement.py uses unprefixed names (cog/attention.py:12-17)
sparse_head_placement = cog_sparse_head_placement
hidden_states_placement = cog_hidden_states_placement
