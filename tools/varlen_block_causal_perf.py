"""Block-causal attention inside packed variable-length segments (plan_local_varlen(block=)) on the H100, bf16,
D = 128: a packed training batch of Wan-480p clips of 21, 13, 9 and 5 latent frames (1 560 tokens per frame, 74 880
tokens in all), every clip chunk-wise causal on its own with chunks of 3 frames and a first chunk of 1 frame (the I2V
layout), at 12 heads (Wan 1.3B) and 40 heads (14B), forward and forward + backward (torch.autograd.backward) of

    packed   one core.plan_local_varlen(block=4680, first_block=1560) over the packed batch
    flex     compiled flex_attention under a document-block-causal BlockMask of the same mask
    loop     one core.plan_block_causal + core.attention per clip on its slice, outputs concatenated (torch.cat)

under two masks: `block` (unbounded window, no sink) and `block-window-sink` (a 9-frame window counted back from the
block end and a one-frame sink, both per clip).  flex's and the loop's forward outputs are compared with the packed
call's (norm-wise relative difference).

Each figure is the median of R rounds with the rounds' min and max, the three ways alternated within every round;
plans, key-major plans and BlockMasks are built outside the timed region.  The card name and power limit are read in
the same run.

    python tools/varlen_block_causal_perf.py [--rounds R] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "sparse-videogen_b200"), str(ROOT / "tools")]

from local_attn_perf import alternate, card, inputs, step  # noqa: E402

FRAME = 1560
CLIPS = (21, 13, 9, 5)  # latent frames per clip
CHUNK, FIRST, WINDOW, SINK = 3 * FRAME, FRAME, 9 * FRAME, FRAME
HEADS = (12, 40)
MASKS = {"block": dict(window=-1, sink=0), "block-window-sink": dict(window=WINDOW, sink=SINK)}


def _rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm())


def run(dev, rounds):
    from torch.nn.attention.flex_attention import create_block_mask, flex_attention

    from svgb200 import core

    flex = torch.compile(flex_attention)
    cu = [0]
    for f in CLIPS:
        cu.append(cu[-1] + f * FRAME)
    S = cu[-1]
    cu_t = torch.tensor(cu, dtype=torch.int32, device=dev)
    # per position: its clip and the clip's first token; per query: its block end, all in packed coordinates
    lens = torch.tensor([f * FRAME for f in CLIPS], device=dev)
    clip = torch.repeat_interleave(torch.arange(len(CLIPS), device=dev), lens)
    start = torch.tensor(cu[:-1], device=dev)[clip]
    rel = torch.arange(S, device=dev) - start
    ends = start + FIRST + ((rel - FIRST).div(CHUNK, rounding_mode="floor") + 1).clamp(min=0) * CHUNK

    def mod_of(window, sink):
        def mod(b, h, q, kv):
            near = kv < ends[q]
            if window != -1:
                near = near & (kv >= ends[q] - window)
            return (clip[q] == clip[kv]) & ((kv - start[kv] < sink) | near)

        return mod

    out = []
    for H in HEADS:
        x = inputs(1, H, S, dev)
        for name, m in MASKS.items():
            packed = core.plan_local_varlen(cu_t, total_q=S, block=CHUNK, first_block=FIRST,
                                            window_size=(m["window"], -1), sink=m["sink"])
            per_clip = [core.plan_block_causal(H, b - a, dev, block=CHUNK, first_block=FIRST, **m)
                        for a, b in zip(cu, cu[1:])]
            for p in [packed, *per_clip]:
                p.key_major()
            bmask = create_block_mask(mod_of(**m), None, None, S, S, device=dev, _compile=True)

            def loop(q, k, v, plans=per_clip):
                return torch.cat([core.attention(q[:, :, a:b], k[:, :, a:b], v[:, :, a:b], p)
                                  for (a, b), p in zip(zip(cu, cu[1:]), plans)], dim=2)

            fns = {"packed": lambda *t, p=packed: core.attention(*t, p),
                   "flex": lambda *t, bm_=bmask: flex(*t, block_mask=bm_),
                   "loop": loop}
            case = {"case": name, "S": S, "H": H, "clips": list(CLIPS)}
            for bwd in (False, True):
                case["fwd_bwd" if bwd else "fwd"] = alternate(
                    {w: (lambda f=f: step(f, x, bwd)) for w, f in fns.items()}, rounds)
            o = fns["packed"](*x[:3])
            case["rel_diff_flex"] = _rel(fns["flex"](*x[:3]), o)
            case["rel_diff_loop"] = _rel(fns["loop"](*x[:3]), o)
            print(json.dumps(case), flush=True)
            out.append(case)
            del packed, per_clip, bmask
        del x
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("varlen_block_causal_perf.py measures on the GPU; no CUDA device found")
    dev = torch.device("cuda:0")
    res = {"card": card()}
    print(json.dumps(res), flush=True)
    res["packed"] = run(dev, a.rounds)
    if a.out:
        Path(a.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
