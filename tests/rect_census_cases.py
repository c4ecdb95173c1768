"""The rectangular census cases (Sq != Skv) shared by tests/test_attention_rect_census_cpu.py and
tests/test_attention_rect_census_gpu.py: variable-block maps, local and block-causal masks inside packed segments of
unequal totals, the 16-bit KV cache at Sq < L, and one production shape.  TEST INFRASTRUCTURE ONLY.

Every case has one mask predicate over [Sq, Skv], taken from the modules that already state it for these plans
(tests/varlen_local_mask.py, tests/varlen_block_causal_mask.py, the local and block-causal predicates that
tests/kvcache_mask.py and tests/block_causal_mask.py evaluate at p = i + L - Sq, and the element mask of a block map).
`mod(h, mutant=)` also gives the oracle mutants the CPU tests show the censuses see:
  top_left       queries aligned to the first key of their segment (p = qi) instead of its last (p = qi + Lk - Lq)
  drop_last_key  key Skv - 1 never attended
  valid_from_sq  the last key chunk's valid count taken from Sq ((Sq - 1) % 128 + 1) instead of Skv
The totals are chosen so that Sq % 128 != Skv % 128 on every case and the last chunk is 1, 64, 65 and 127 columns wide
on each side somewhere in the list."""
from __future__ import annotations

import dataclasses
from dataclasses import dataclass, field

import torch

import block_causal_mask as bm
import local_mask as lm
import varlen_block_causal_mask as vb
import varlen_local_mask as vm
from oracle import bwd_census as bc
from oracle import softmax as sm

BIG = 10 ** 6
MASK_MUTANTS = ("top_left", "drop_last_key", "valid_from_sq")


def _cu(lens):
    out = [0]
    for n in lens:
        out.append(out[-1] + n)
    return out


@dataclass
class Rect:
    name: str
    kind: str                      # "varblock", "local", "block" (packed segments) or "kvcache"
    Sq: int
    Skv: int
    H: int = 2
    bm: torch.Tensor | None = None     # varblock: [H, QC, KC] map, rows [H, QC], cols [H, KC]
    rows: torch.Tensor | None = None
    cols: torch.Tensor | None = None
    cu_q: list | None = None           # local / block: packed bounds and (sink, left, right) / (sink, C, F, W)
    cu_k: list | None = None
    args: tuple = ()
    kv: dict = field(default_factory=dict)  # kvcache: mask ("causal", "window", "block"), sink, left, C, F, W, page
    softmax: dict = field(default_factory=dict)  # oracle.softmax builder parameters (L, C, frac, offset)
    backward: bool = True

    # ---------------------------------------------------------------- the mask
    def _base(self, cu_q, cu_k):
        if self.kind == "local":
            return vm.mask_fn(cu_q, cu_k, *self.args)
        return vb.mask_fn(cu_q, cu_k, *self.args)

    def _kv_base(self):
        k = self.kv
        if k["mask"] == "block":
            return bm.block_causal_mask_fn(k["C"], k["F"], k["W"], k["sink"])
        return lm.local_mask_fn(k["sink"], BIG if k["mask"] == "causal" else k["left"], 0)

    def _shifted(self, shift):
        """The segment predicate with every query position moved by shift[i] in segment i: the predicate of virtual
        segments whose key segment is longer by max(d, 0) and query segment by max(-d, 0), evaluated at the real
        queries and keys (the predicate reads a key only relative to its segment's key 0)."""
        lq = [b - a for a, b in zip(self.cu_q, self.cu_q[1:])]
        lk = [b - a for a, b in zip(self.cu_k, self.cu_k[1:])]
        vq = _cu([a + max(-d, 0) for a, d in zip(lq, shift)])
        vk = _cu([a + max(d, 0) for a, d in zip(lk, shift)])
        base = self._base(vq, vk)
        cq, ck, tq, tk = (torch.tensor(x) for x in (self.cu_q, self.cu_k, vq, vk))

        def mod(q_idx, kv_idx):
            q_idx, kv_idx = torch.as_tensor(q_idx).long(), torch.as_tensor(kv_idx).long()
            sq = (torch.searchsorted(cq.to(q_idx.device), q_idx.contiguous(), right=True) - 1).clamp(max=len(lq) - 1)
            sk = (torch.searchsorted(ck.to(kv_idx.device), kv_idx.contiguous(), right=True) - 1).clamp(max=len(lk) - 1)
            return base(q_idx - cq.to(q_idx.device)[sq] + tq.to(q_idx.device)[sq],
                        kv_idx - ck.to(kv_idx.device)[sk] + tk.to(kv_idx.device)[sk])

        return mod

    def mod(self, h: int = 0, mutant: str | None = None):
        """allowed(q_idx, kv_idx) of head h over [Sq, Skv] on index tensors; mutant: one of MASK_MUTANTS or None."""
        if mutant == "top_left":
            if self.kind == "kvcache":
                base, off = self._kv_base(), 0
                return lambda q, k: base(torch.as_tensor(q) + off, k)
            lq = [b - a for a, b in zip(self.cu_q, self.cu_q[1:])]
            lk = [b - a for a, b in zip(self.cu_k, self.cu_k[1:])]
            return self._shifted([a - b for a, b in zip(lq, lk)])
        if self.kind == "varblock":
            from oracle.attention import block_mask_to_element_mask

            dense = block_mask_to_element_mask(self.bm[h], self.rows[h], self.cols[h])

            def true(q, k):
                q, k = torch.as_tensor(q).long(), torch.as_tensor(k).long()
                return dense.to(q.device)[q, k]
        elif self.kind == "kvcache":
            base, off = self._kv_base(), self.Skv - self.Sq
            true = lambda q, k: base(torch.as_tensor(q) + off, k)  # noqa: E731
        else:
            true = self._base(self.cu_q, self.cu_k)
        if mutant is None:
            return true
        if mutant == "drop_last_key":
            return lambda q, k: true(q, k) & (torch.as_tensor(k) != self.Skv - 1)
        assert mutant == "valid_from_sq", mutant
        end = (self.Skv - 1) // 128 * 128 + (self.Sq - 1) % 128 + 1
        return lambda q, k: true(q, k) & (torch.as_tensor(k) < end)

    def applies(self, mutant: str) -> bool:
        if mutant == "top_left":
            return self.kind != "varblock"
        if mutant == "valid_from_sq":
            return (self.Sq - 1) % 128 < (self.Skv - 1) % 128
        return True

    def dense(self, h: int = 0, mutant: str | None = None, device="cpu") -> torch.Tensor:
        return self.mod(h, mutant)(torch.arange(self.Sq, device=device).view(-1, 1),
                                   torch.arange(self.Skv, device=device).view(1, -1))

    # ---------------------------------------------------------------- census inputs
    def softmax_case(self, D=128, c=None, vs=None, device="cpu"):
        """The oracle.softmax case of this mask (plan order: queries and keys in packed / logical order)."""
        if self.kind == "varblock":
            return sm.rect_blockmap_case(self.name, self.bm, self.rows, self.cols, D=D, c=c, vs=vs, **self.softmax)
        return sm.mask_case(self.name, self.mod(), self.Sq, self.Skv, D=D, H=self.H, c=c, vs=vs, device=device,
                            **self.softmax)

    def grad_case(self, D=128, seed=7):
        if self.kind == "varblock":
            return bc.grad_rect_case(self.name, self.Sq, self.Skv, D=D, H=self.H, seed=seed, bm=self.bm,
                                     rows=self.rows, cols=self.cols)
        return bc.grad_rect_case(self.name, self.Sq, self.Skv, D=D, H=self.H, seed=seed, mod=self.mod())

    def with_mask(self, case, mutant):
        """A softmax or gradient case equal to `case` (same inputs, row classes and values) except that head 0 runs
        the mutant's mask."""
        return dataclasses.replace(case, mod=self.mod(0, mutant), bm=None)


# --------------------------------------------------------------------------------------------
# variable-block maps
# --------------------------------------------------------------------------------------------
def edge_sizes(total, special, n, gen):
    """n block sizes summing to total: the `special` sizes (the r % 128 and r % 256 edges, 0 for an empty block) and a
    random partition of the rest, shuffled."""
    rest = total - sum(special)
    k = n - len(special)
    assert rest >= k >= 1
    cuts = torch.sort(torch.randperm(rest - 1, generator=gen)[: k - 1] + 1)[0] if k > 1 else torch.zeros(0).long()
    part = torch.diff(torch.cat([torch.tensor([0]), cuts, torch.tensor([rest])]))
    s = torch.cat([torch.tensor(special), part])
    return s[torch.randperm(n, generator=gen)].int()


def varblock(name, Sq, Skv, rspecial, cspecial, QC, KC, seed, H=2, softmax=None):
    """Per-head maps of density 0.6 with edge sizes on both axes, an empty q-block and an empty key block, one
    non-empty q-block that selects nothing (keyless rows), one non-empty key block no q-block selects (dK = dV = 0) and
    one that every q-block selects."""
    g = torch.Generator().manual_seed(seed)
    rows = torch.stack([edge_sizes(Sq, rspecial, QC, g) for _ in range(H)])
    cols = torch.stack([edge_sizes(Skv, cspecial, KC, g) for _ in range(H)])
    m = torch.rand(H, QC, KC, generator=g) < 0.6
    for h in range(H):
        live_r = (rows[h] > 0).nonzero().flatten().tolist()
        live_c = (cols[h] > 0).nonzero().flatten().tolist()
        m[h, :, live_c[-1]] = True
        m[h, live_r[0], :] = False
        m[h, :, live_c[0]] = False
    return Rect(name, "varblock", Sq, Skv, H, bm=m, rows=rows, cols=cols,
                softmax=softmax or dict(L=256, C=4))


def wan720_text():
    """Wan 720p text cross-attention: 75 600 queries against 512 text keys, one head, dense.  The key regions are
    offset so that each row meets one cold chunk, is wiped in the next and rescales twice (t rising over 3 chunks)."""
    one = torch.ones(1, 1, 1, dtype=torch.bool)
    return Rect("wan720_text", "varblock", 75600, 512, 1, bm=one, rows=torch.tensor([[75600]]),
                cols=torch.tensor([[512]]), softmax=dict(L=384, C=2, offset=256), backward=False)


# --------------------------------------------------------------------------------------------
# the case list
# --------------------------------------------------------------------------------------------
def local(name, lq, lk, sink, left, right, L=384):
    return Rect(name, "local", sum(lq), sum(lk), cu_q=_cu(lq), cu_k=_cu(lk), args=(sink, left, right),
                softmax=dict(L=L, C=8))


def block(name, lq, lk, sink, C_, F, W, L=384):
    return Rect(name, "block", sum(lq), sum(lk), cu_q=_cu(lq), cu_k=_cu(lk), args=(sink, C_, F, W),
                softmax=dict(L=L, C=8))


def kvcache(name, Sq, L, page=0, sink=0, **mask):
    return Rect(name, "kvcache", Sq, L, kv=dict(page=page, sink=sink, **mask), softmax=dict(L=384, C=8),
                backward=False)


CASES = [
    # variable-block: Sq > Skv, Sq < Skv, and a key side shorter than one chunk
    varblock("vb_1000x600", 1000, 600, [0, 1, 128, 129, 255, 256], [0, 1, 64, 65, 127, 129], 9, 8, 11),
    varblock("vb_333x1200", 333, 1200, [0, 1, 64, 65, 127], [0, 1, 128, 129, 255, 256, 257], 8, 10, 12),
    varblock("vb_1151x65", 1151, 65, [0, 1, 127, 129, 256], [0, 1, 30], 8, 4, 13),
    # local mask in packed segments of unequal totals
    local("local_holes", [300, 500, 0, 77], [100, 900, 60, 0], 0, BIG, 0),
    local("local_sink_window", [1, 640, 333], [300, 2000, 333], 33, 517, 13),
    local("local_short_tail", [500, 651], [1200, 81], 0, 300, 0),
    # block-causal in packed segments: queries ahead of their keys (Lq > Lk), F < C with a window and a sink, one query
    block("block_ahead", [449, 384], [216, 1000], 0, 100, 40, -1),
    block("block_window_sink", [279, 1000], [1500, 1190], 33, 300, 77, 600),
    block("block_one_query", [1, 575], [705, 640], 7, 64, 64, 256),
    # 16-bit KV cache, single pass, Sq < L
    kvcache("kv_causal_contig", 1, 1300, mask="causal"),
    kvcache("kv_causal_paged", 300, 1279, page=256, mask="causal"),
    kvcache("kv_window_contig", 257, 1344, mask="window", left=300, sink=70),
    kvcache("kv_window_paged", 300, 1281, page=128, mask="window", left=517, sink=129),
    kvcache("kv_block_contig", 300, 1345, mask="block", C=100, F=45, W=400, sink=33),
    kvcache("kv_block_paged", 257, 1300, page=128, mask="block", C=300, F=77, W=-1),
]
BY_NAME = {c.name: c for c in CASES}
BACKWARD = [c.name for c in CASES if c.backward]
WAN720_TEXT = wan720_text()

# Wan 480p (1 560 tokens per latent frame): a 3-frame chunk against 22 frames as one block-causal segment; the chunk
# is exactly the last block, so every query sees the one-frame sink and the 9 frames before the chunk's end
FRAME = 1560
WAN480_CHUNK = block("wan480_chunk", [3 * FRAME], [22 * FRAME], FRAME, 3 * FRAME, FRAME, 9 * FRAME, L=4096)
