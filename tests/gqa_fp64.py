"""fp64 oracle of grouped-query attention for the GQA tests: K and V repeated per group (query head h attends with
key/value head h // G), then the masked softmax per query head.  Autograd through the repeat sums each key/value
head's gradient over the G query heads of its group."""
import torch


def gqa_attention(q, k, v, masks, sm_scale=None):
    """q [Hq, Sq, D]; k, v [Hkv, Skv, D]; masks: bool [Hq, Sq, Skv] (or one [Sq, Skv] for every head) -> o [Hq, Sq, D]
    in q's dtype; rows without an allowed key give 0."""
    G = q.shape[0] // k.shape[0]
    scale = q.shape[-1] ** -0.5 if sm_scale is None else sm_scale
    kr, vr = (t.repeat_interleave(G, 0) for t in (k, v))
    s = (q @ kr.transpose(1, 2) * scale).masked_fill(~masks, float("-inf"))
    return torch.nan_to_num(torch.softmax(s, dim=-1), nan=0.0) @ vr


def gqa_grads(q, k, v, do, masks, sm_scale=None):
    """(o, dq, dk, dv) in fp64 of gqa_attention for the output gradient do; dk, dv have k's shape."""
    x = [t.detach().double().requires_grad_() for t in (q, k, v)]
    o = gqa_attention(*x, masks, sm_scale)
    o.backward(do.double())
    return o.detach(), x[0].grad, x[1].grad, x[2].grad
