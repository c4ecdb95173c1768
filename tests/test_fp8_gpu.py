"""FP8 (e4m3) attention path (BASELINE config 5).  The reference has no FP8 sparse attention
(README.md:117; FlashInfer's fp8 sparse path asserts backend == "fa3"), so the oracle is fp32 attention
on the DEQUANTISED inputs and the tolerance is ours: P is rounded to e4m3 (3 mantissa bits, relative
step 2^-3..2^-4) before PV, which averages out over the keys of a row; we require rtol 8e-2 / atol 4e-2
on outputs of magnitude ~0.1-1 and report the measured error."""
import pytest
import torch

pytestmark = pytest.mark.gpu

# lse: Q K^T runs on e4m3 wgmma, whose accumulation is not full fp32 on sm_90 (about 2^-13 of the running sum); the
# logits of these inputs stay within ~10, so the lse is good to ~2e-3 against the fp64 logsumexp of the
# dequantised inputs
FP8_LSE = dict(rtol=1e-3, atol=5e-3)


def _check_lse(lse, ref_lse):
    lse, ref_lse = lse.cpu().double().reshape(ref_lse.shape), ref_lse.double()
    empty = ref_lse == float("-inf")
    assert torch.equal(lse == float("-inf"), empty), "-inf rows differ"
    torch.testing.assert_close(lse[~empty], ref_lse[~empty], **FP8_LSE)


def test_quantize_e4m3(cuda):
    """scale = absmax / 448 per head (1 for an all-zero head, whose bytes are all 0) and x8 = e4m3(fp32(x) *
    fp32(1 / scale)) round-to-nearest-even, bit for bit against torch's CPU float8_e4m3fn cast of the same fp32
    product; no scaled value exceeds 448 by more than its own rounding, so saturation cannot separate the two."""
    _quantize_case(cuda, torch.bfloat16)


def test_quantize_e4m3_fp16(cuda):
    """The same contract for fp16 input."""
    _quantize_case(cuda, torch.float16)


def _quantize_case(cuda, dtype):
    from svgb200 import core

    g = torch.Generator().manual_seed(0)
    x = (torch.randn(2, 3, 500, 128, generator=g) * torch.tensor([0.1, 1.0, 30.0]).view(1, 3, 1, 1)).to(dtype)
    x[1, 2] = 0  # an all-zero head
    x8, scale = core.quantize_e4m3(x.to(cuda))
    x8, scale = x8.cpu(), scale.cpu()
    amax = x.float().abs().amax(dim=(2, 3)).view(-1)
    ref_scale = torch.where(amax > 0, amax / 448.0, torch.ones_like(amax))
    assert torch.equal(scale, ref_scale)
    y = x.float() * torch.reciprocal(ref_scale).view(2, 3, 1, 1)
    assert float(y.abs().max()) <= 448 * (1 + 2 ** -21)  # three fp32 roundings: amax / 448, 1 / scale, x * inv
    ref8 = y.to(torch.float8_e4m3fn).view(torch.uint8)
    assert torch.equal(x8, ref8), f"{int((x8 != ref8).sum())} bytes differ"
    assert bool((x8[1, 2] == 0).all()) and float(scale[5]) == 1.0
    x = x.clone()
    x[1, 2] = torch.randn(500, 128, generator=g).to(dtype)  # the half-ulp bound below needs a non-zero head
    x8, scale = core.quantize_e4m3(x.to(cuda))
    deq = x8.view(torch.float8_e4m3fn).float().cpu() * scale.cpu().view(2, 3, 1, 1)
    amax = x.float().abs().amax(dim=(2, 3)).view(-1)
    torch.testing.assert_close(scale.cpu(), amax / 448.0, rtol=1e-6, atol=0)
    err = (deq - x.float()).abs()
    bound = torch.maximum(x.float().abs() * 2 ** -4, scale.cpu().view(2, 3, 1, 1) * 2 ** -10)  # half ulp (3 mantissa bits)
    assert bool((err <= bound * 1.001 + 1e-12).all())
    assert float(deq.abs().amax()) == pytest.approx(float(x.float().abs().amax()), rel=1e-6)


@pytest.mark.parametrize("S,MB,NB,density", [(1024, 5, 9, 0.4), (4096, 20, 100, 0.7)])
def test_fp8_variable_block_attention(cuda, S, MB, NB, density):
    from oracle.attention import dynamic_block_sparse_fwd
    from svgb200 import core

    g = torch.Generator().manual_seed(S)
    H, D = 2, 128
    q, k, v = (torch.randn(1, H, S, D, generator=g).bfloat16() for _ in range(3))

    def part(n):
        cuts = torch.sort(torch.randperm(S - 1, generator=g)[: n - 1] + 1)[0]
        return torch.diff(torch.cat([torch.tensor([0]), cuts, torch.tensor([S])])).to(torch.int32)
    row = torch.stack([part(MB) for _ in range(H)])
    col = torch.stack([part(NB) for _ in range(H)])
    bm = torch.rand(H, MB, NB, generator=g) > density
    (q8, sq), (k8, sk), (v8, sv) = (core.quantize_e4m3(t.to(cuda)) for t in (q, k, v))
    plan = core.plan_varblock(bm.to(cuda), row.to(cuda), col.to(cuda), S)
    o, lse = core.attn_fwd_fp8(q8, k8, v8, sq, sk, sv, plan, return_lse=True)
    o = o.float().cpu()

    def deq(x8, s):
        return x8.view(torch.float8_e4m3fn).double().cpu() * s.cpu().double().view(1, H, 1, 1)
    ref, ref_lse = dynamic_block_sparse_fwd(deq(q8, sq), deq(k8, sk), deq(v8, sv), bm[None], row[None], col[None],
                                            return_lse=True, dtype=torch.float64)
    ref = ref.float()
    _check_lse(lse, ref_lse)
    err = (o - ref).abs()
    print("fp8 attention max abs err", float(err.max()), "mean", float(err.mean()))
    torch.testing.assert_close(o, ref, rtol=8e-2, atol=4e-2)
    # and it stays close to the bf16 path on the original inputs
    o16 = core.attn_fwd(q.to(cuda), k.to(cuda), v.to(cuda), plan).float().cpu()
    assert float((o - o16).abs().mean()) < 2e-2


def test_fp8_band_attention(cuda):
    from oracle import attention as oa
    from svgb200 import core
    from svgb200.models import wan

    g = torch.Generator().manual_seed(5)
    H, F, P, D = 2, 6, 200, 128
    S = F * P
    q, k, v = (torch.randn(1, H, S, D, generator=g).bfloat16() for _ in range(3))
    bm = wan.prepare_flexattention(1, H, D, torch.bfloat16, cuda, 0, 0, F, P, diag_width=1.3, multiplier=1.3)
    (q8, sq), (k8, sk), (v8, sv) = (core.quantize_e4m3(t.to(cuda)) for t in (q, k, v))
    o, lse = core.attn_fwd_fp8(q8, k8, v8, sq, sk, sv, bm.plan, return_lse=True)
    o = o.float().cpu()

    def deq(x8, s):
        return x8.view(torch.float8_e4m3fn).double().cpu() * s.cpu().double().view(1, H, 1, 1)
    ref, ref_lse = oa.masked_attention_bhsd(deq(q8, sq)[0], deq(k8, sk)[0], deq(v8, sv)[0], oa.wan_mask_mod(F, P, 1.3),
                                            return_lse=True, dtype=torch.float64)
    torch.testing.assert_close(o, ref.float()[None], rtol=8e-2, atol=4e-2)
    _check_lse(lse, ref_lse)


@pytest.mark.parametrize("case", ["hy_band", "cog_band", "tails_o_rows"])
def test_fp8_masks_edges_and_head_scales(cuda, case):
    """FP8 under the HunyuanVideo and CogVideoX element masks, and on a variable-block plan with the dual-tail edge
    sizes, an empty q-block, a q-block that selects nothing (l = 0: output 0 whatever v_scale, lse -inf) and the
    output scattered through o_rows.  The two heads' q / v scales differ by ~300x (q x 0.03 | x 10, v x 10 | x 0.03),
    so a scale read from the wrong head fails; outputs are compared in units of each head's V magnitude."""
    from oracle import attention as oa
    from svgb200 import core

    g = torch.Generator().manual_seed(3)
    H, D = 2, 128
    fq, fv = torch.tensor([0.03, 10.0]), torch.tensor([10.0, 0.03])
    if case == "tails_o_rows":
        rows = [257, 15, 64, 128 + 33, 300, 48, 17, 0, 64 + 256, 1, 16, 33, 100, 128, 200]
        S, KC = sum(rows), 23
        row = torch.tensor([rows, rows[::-1]], dtype=torch.int32)
        col = torch.stack([torch.diff(torch.cat([torch.tensor([0]), torch.sort(torch.randperm(S - 1, generator=g)[:KC - 1] + 1)[0],
                                                 torch.tensor([S])])) for _ in range(H)]).to(torch.int32)
        bm = torch.rand(H, len(rows), KC, generator=g) < 0.45
        bm[0, 1, :] = False   # a tail that attends nothing
        bm[1, 3, :] = True
    else:
        if case == "hy_band":
            F, P, ctx, plen, mul = 6, 200, 48, 20, 1.4
            mod = oa.hy_mask_mod(ctx, plen, F, P, mul)
            args = (core.MASK_HY, F * P, F * P + plen, oa.hy_band_width(mul, P))
        else:
            F, P, ctx, plen, mul = 4, 260, 40, 40, 1.1
            mod = oa.cog_mask_mod(plen, F, P, mul)
            args = (core.MASK_COG, plen, plen, oa.hy_band_width(mul, P))
        S = ctx + F * P
    q = (torch.randn(1, H, S, D, generator=g) * fq.view(1, H, 1, 1)).bfloat16()
    k = torch.randn(1, H, S, D, generator=g).bfloat16()
    v = (torch.randn(1, H, S, D, generator=g) * fv.view(1, H, 1, 1)).bfloat16()
    (q8, sq), (k8, sk), (v8, sv) = (core.quantize_e4m3(t.to(cuda)) for t in (q, k, v))
    assert float(sq.max() / sq.min()) > 200 and float(sv.max() / sv.min()) > 200

    def deq(x8, s):
        return x8.view(torch.float8_e4m3fn).double().cpu() * s.cpu().double().view(1, H, 1, 1)
    qd, kd, vd = deq(q8, sq), deq(k8, sk), deq(v8, sv)
    if case == "tails_o_rows":
        plan = core.plan_varblock(bm.to(cuda), row.to(cuda), col.to(cuda), S)
        perm = torch.stack([torch.randperm(S, generator=g) for _ in range(H)]).to(torch.int32)
        o, lse = core.attn_fwd_fp8(q8, k8, v8, sq, sk, sv, plan, o_rows=perm.to(cuda), return_lse=True)
        o, lse = o.float().cpu(), lse.cpu()
        o = torch.stack([o[0, h][perm[h].long()] for h in range(H)])[None]  # undo the scatter
        lse = torch.stack([lse[h][perm[h].long()] for h in range(H)])
        ref, ref_lse = oa.dynamic_block_sparse_fwd(qd, kd, vd, bm[None], row[None], col[None], return_lse=True,
                                                   dtype=torch.float64)
        ref, ref_lse = ref, ref_lse[0]
        r0 = rows[0]
        assert torch.all(o[0, 0, r0:r0 + rows[1]] == 0)
    else:
        plan = core.plan_band(*args, H, S, cuda)
        o, lse = core.attn_fwd_fp8(q8, k8, v8, sq, sk, sv, plan, return_lse=True)
        o = o.float().cpu()
        ref, ref_lse = oa.masked_attention_bhsd(qd[0], kd[0], vd[0], mod, return_lse=True, dtype=torch.float64)
        ref = ref[None]
    for h in range(H):
        torch.testing.assert_close(o[0, h] / fv[h], (ref[0, h] / fv[h]).float(), rtol=8e-2, atol=4e-2)
    _check_lse(lse, ref_lse)
