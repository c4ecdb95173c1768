"""Exact census of the pre-attention backward on the GPU (oracle/rowwise_bwd.py): the standalone norm backwards, the
fused qkv_prep backward with per-head RMS / LayerNorm and with NORM_RMS_HIDDEN, and their autograd wiring, compared
bit for bit with a closed form on every element, at the shapes where the persistent grids, the hidden path's token
splits and the dead lanes come into play.

dx is compared bit for bit on every element (a row whose dn is 0 must give a zero of either sign: its -0 compares equal
to +0).  dgamma and dbeta are read in fp32 through the C entry points, as core calls them, and compared bit for bit:
dbeta and the hidden path's dgamma are exact in any summation order; dgamma on the rsqrtf paths is exact because
rsqrt.approx.f32 returns 2^-k for 4^k exactly, which `test_rsqrtf_is_exact_on_the_census_variances` pins.  Every
output goes into NaN-filled memory, so an element that is never written fails."""
import ctypes as C

import pytest
import torch

from oracle import rowwise as rw
from oracle import rowwise_bwd as rb

pytestmark = pytest.mark.gpu

CHUNK = 1 << 22   # elements per chunk of the builders and comparisons
NAN = float("nan")


def poison(cuda, nbytes=64 << 20):
    """Fill the caching allocator's free blocks with NaN so outputs the kernels never write show up."""
    t = torch.full((nbytes // 2 + 1,), NAN, dtype=torch.float16, device=cuda)
    del t


def assert_bits(got, want, what):
    """got == want bit for bit, with -0 taken as +0 (got + 0 changes nothing else); else the count and the first
    differing (row, column) of the [-1, last dim] view."""
    assert got.dtype == want.dtype and got.shape == want.shape, \
        f"{what}: {got.dtype} {got.shape} vs {want.dtype} {want.shape}"
    iv = {2: torch.int16, 4: torch.int32}[got.element_size()]
    got = got + 0
    ne = got.contiguous().view(iv) != want.contiguous().view(iv)
    if bool(ne.any()):
        r, c = (int(i) for i in ne.reshape(-1, got.shape[-1]).nonzero()[0])
        g, w = got.reshape(-1, got.shape[-1])[r, c].item(), want.reshape(-1, want.shape[-1])[r, c].item()
        raise AssertionError(f"{what}: {int(ne.sum())} elements differ; first at row {r}, column {c}: "
                             f"got {g}, want {w}")


def assert_rows(got, want, what):
    """assert_bits on [-1, N] views in row chunks (production sizes)."""
    N = got.shape[-1]
    got, want = got.reshape(-1, N), want.reshape(-1, N)
    step = max(1, CHUNK // N)
    for r0 in range(0, got.shape[0], step):
        assert_bits(got[r0:r0 + step], want[r0:r0 + step], f"{what}, rows from {r0}")


class Sums:
    """float64 dgamma / dbeta of a census and the sums of |terms| that bound their exactness."""

    def __init__(self, N, cuda):
        self.dg, self.db, self.ag, self.ab = (torch.zeros(N, dtype=torch.float64, device=cuda) for _ in range(4))

    def add(self, c, N):
        t = (c["dn"] * c["xh"]).reshape(-1, N)
        dn = c["dn"].reshape(-1, N)
        self.dg += t.sum(0)
        self.db += dn.sum(0)
        self.ag += t.abs().sum(0)
        self.ab += dn.abs().sum(0)

    def expect(self):
        """(dgamma, dbeta) as fp32, checking first that every fp32 sum of the terms is exact."""
        assert float(self.ag.max()) < rb.SUM_LIMIT * rb.Q_DG and float(self.ab.max()) < rb.SUM_LIMIT * rb.Q_DB, \
            "census premise: the dgamma / dbeta sums must stay below 2^24 quanta"
        return self.dg.float(), self.db.float()


def lib():
    from svgb200 import _lib

    return _lib.lib()


# ---- the C entry points, with fp32 parameter gradients ------------------------------------------------------------
def row_norm_bwd_f32(x, dy, g, layer):
    """svgb_rms_norm_bwd / svgb_layer_norm_bwd into NaN-filled dx, dgamma, dbeta (fp32, not rounded to 16 bits)."""
    from svgb200 import core

    n = x.shape[-1]
    m = x.numel() // n
    nbytes = C.c_size_t()
    core.check(lib().svgb_row_norm_bwd_bytes(m, n, C.byref(nbytes)), "svgb_row_norm_bwd_bytes")
    ws = torch.full((max(nbytes.value, 256) // 4,), NAN, dtype=torch.float32, device=x.device)
    dx = torch.full_like(x, NAN)
    dg, db = (torch.full((n,), NAN, dtype=torch.float32, device=x.device) for _ in range(2))
    if layer:
        core.check(lib().svgb_layer_norm_bwd(x.data_ptr(), dy.data_ptr(), g.data_ptr(), dx.data_ptr(), dg.data_ptr(),
                                             db.data_ptr(), m, n, core._dt(x), ws.data_ptr(), ws.numel() * 4,
                                             core._stream(x)), "svgb_layer_norm_bwd")
    else:
        core.check(lib().svgb_rms_norm_bwd(x.data_ptr(), dy.data_ptr(), g.data_ptr(), dx.data_ptr(), dg.data_ptr(), m,
                                           n, rb.RMS_EPS, core._dt(x), ws.data_ptr(), ws.numel() * 4,
                                           core._stream(x)), "svgb_rms_norm_bwd")
    return dx, dg, db


def prep_bwd_f32(dy, q_in, k_in, H, S, r0, norm, gq, gk, rope, cos, sin, lo, n):
    """svgb_qkv_prep_bwd as core.qkv_prep_bwd calls it, into NaN-filled outputs; dgamma / dbeta in fp32."""
    from svgb200 import core

    B, _, S_out, D = dy[0].shape
    nbytes = C.c_size_t()
    core.check(lib().svgb_qkv_prep_bwd_bytes(B, S, H, D, norm, C.byref(nbytes)), "svgb_qkv_prep_bwd_bytes")
    ws = torch.full((max(nbytes.value, 256) // 4,), NAN, dtype=torch.float32, device=q_in.device)
    dx = [torch.full((B, S, H * D), NAN, dtype=q_in.dtype, device=q_in.device) for _ in range(3)]
    gw = H * D if norm == 3 else D
    f32 = lambda: torch.full((gw,), NAN, dtype=torch.float32, device=q_in.device)  # noqa: E731
    dg = [f32(), f32()]
    db = [f32(), f32()] if norm == 2 else [None, None]
    core.check(lib().svgb_qkv_prep_bwd(
        dy[0].data_ptr(), dy[1].data_ptr(), dy[2].data_ptr(), S_out * D, H * S_out * D, q_in.data_ptr(),
        k_in.data_ptr(), q_in.stride(1), q_in.stride(0), dx[0].data_ptr(), dx[1].data_ptr(), dx[2].data_ptr(), B, S, H,
        D, r0, norm, gq.data_ptr(), gk.data_ptr(), rb.RMS_EPS, rope, core._p(cos), core._p(sin), lo, n,
        dg[0].data_ptr(), dg[1].data_ptr(), core._p(db[0]), core._p(db[1]), core._dt(q_in), ws.data_ptr(),
        ws.numel() * 4, core._stream(q_in)), "svgb_qkv_prep_bwd")
    return dx, dg, db


# ---- 0. the premise of the dgamma census on the rsqrtf paths ------------------------------------------------------
@pytest.mark.parametrize("n", rw.NORM_NS)
@pytest.mark.parametrize("layer", [False, True])
def test_rsqrtf_is_exact_on_the_census_variances(cuda, layer, n):
    """One standalone backward whose dn is a unit vector on each row: dgamma is a sum of the kernel's own x^ = x * r,
    exact only if rsqrtf(var + eps) returns r = 2^-(2+j) exactly for every census variance 16 * 4^j."""
    js = rb.LN_JS if layer else rw.JS
    m = 64
    x, rstd = rw.row_x(n, m, n, centred=layer, js=js)
    assert set(rstd.tolist()) == {2.0 ** -(2 + j) for j in js}
    xh = rw.xhat(x, rstd, layer)
    k = xh.abs().argmax(1)                                   # a column where x^ != 0
    dn = torch.zeros(m, n, dtype=torch.float64)
    dn[torch.arange(m), k] = 1.0
    want = torch.zeros(n, dtype=torch.float64).index_add_(0, k, xh[torch.arange(m), k])
    dtype = torch.bfloat16
    dx, dg, db = row_norm_bwd_f32(x.to(dtype).to(cuda), dn.to(dtype).to(cuda),
                                  torch.ones(n, dtype=dtype, device=cuda), layer)
    eq = dg.cpu().double() == want
    assert bool(eq.all()), (
        f"rsqrt.approx.f32 is not exact on the census variances {[16 * 4 ** j for j in js]}: dgamma column "
        f"{int((~eq).nonzero()[0])} is {dg.cpu()[~eq][0].item()!r}, want {want[~eq][0].item()!r}; the dgamma census "
        "on the rsqrtf paths needs a bound instead of bit equality")
    if layer:
        assert torch.equal(db.cpu().double(), dn.sum(0))


# ---- 1. standalone norm backward ----------------------------------------------------------------------------------
def run_row_norm(cuda, layer, m, n, dtype, seed):
    g = rb.gamma(seed, n, cuda)
    x, dy, want = (torch.empty(m, n, dtype=dtype, device=cuda) for _ in range(3))
    sums = Sums(n, cuda)
    step = max(1, CHUNK // n)
    for r0 in range(0, m, step):
        idx = torch.arange(r0, min(m, r0 + step), device=cuda)
        c = rb.rows(seed, idx, n, g, layer=layer, live=rb.row_live(seed, idx, m, n))
        x[idx], dy[idx], want[idx] = c["x"].to(dtype), c["dn"].to(dtype), c["dx"].to(dtype)
        sums.add(c, n)
        del c
    dg, db = sums.expect()
    got, gdg, gdb = row_norm_bwd_f32(x, dy, g.to(dtype), layer)
    what = f"{'layer' if layer else 'rms'}_norm_bwd m {m} n {n} {dtype}"
    assert_rows(got, want, f"{what}: dx")
    assert_bits(gdg, dg, f"{what}: dgamma")
    if layer:
        assert_bits(gdb, db, f"{what}: dbeta")


@pytest.mark.parametrize("layer, n, dtype, m, seed", rb.ROW_CASES)
def test_row_norm_bwd_census(cuda, layer, n, dtype, m, seed):
    """Every width and dtype at m = 1, m below RPB (one CTA, partly dead), and m just below and just above the row
    count where the 592-CTA walk takes a second pass (rb.row_norm_rows)."""
    run_row_norm(cuda, layer, m, n, rw.DT[dtype], seed)


@pytest.mark.parametrize("layer, n, dtype, m, seed", rb.ROW_CASES_HY)
def test_row_norm_bwd_census_hunyuan720p(cuda, layer, n, dtype, m, seed):
    """HunyuanVideo 720p's QK norm: 2 857 344 head rows of 128 (the 592-CTA walk takes 76 passes)."""
    run_row_norm(cuda, layer, m, n, rw.DT[dtype], seed)


# ---- 2. fused qkv_prep backward ------------------------------------------------------------------------------------
def prep_census(cuda, B, S, H, D, norm, rope, lo, n, dtype, seed, *, qkv=None):
    """The census of one qkv_prep call: q_in / k_in (and v_in, small integers) as strided views of one packed
    [B, S, 3HD] tensor, norm weights and tables, the gradient rows the call reads (dq, dk, dv [B, H, S, D]: dy = RoPE(dn)
    on the rotated tokens) and the expected dq_in, dk_in, dv_in [B, S, HD] and fp32 dgamma / dbeta of q and k."""
    layer, HD = norm == 2, H * D
    N = HD if norm == 3 else D
    gen = torch.Generator(device=cuda).manual_seed(seed)
    g = [rb.gamma(seed * 3 + i, N, cuda) for i in range(2)]
    cos, sin = rb.quarter_tables(seed, n, D, rope, cuda) if rope else (None, None)
    tok_live = rb.prep_live(seed, B, S, H, D, norm, lo, n).to(cuda)
    packed = torch.randint(-64, 65, (B, S, 3 * HD), generator=gen, device=cuda).to(dtype)
    dy = [torch.empty(B, H, S, D, dtype=dtype, device=cuda) for _ in range(2)]
    dy.append(torch.randint(-64, 65, (B, H, S, D), generator=gen, device=cuda).to(dtype))
    want = [torch.empty(B, S, HD, dtype=dtype, device=cuda) for _ in range(2)]
    want.append(dy[2].transpose(1, 2).reshape(B, S, HD))
    sums = [Sums(N, cuda), Sums(N, cuda)]
    step = max(1, CHUNK // HD)
    for i in range(2):
        for b in range(B):
            for t0 in range(0, S, step):
                t1 = min(S, t0 + step)
                tk = b * S + torch.arange(t0, t1, device=cuda)
                idx = tk if norm == 3 else (tk[:, None] * H + torch.arange(H, device=cuda)).reshape(-1)
                lv = tok_live[tk] if norm == 3 else tok_live[tk].repeat_interleave(H)
                c = rb.rows(seed * 3 + i, idx, N, g[i], layer=layer, live=lv)
                packed[b, t0:t1, i * HD:(i + 1) * HD] = c["x"].view(t1 - t0, HD).to(dtype)
                want[i][b, t0:t1] = c["dx"].view(t1 - t0, HD).to(dtype)
                dn = c["dn"].view(t1 - t0, H, D).transpose(0, 1)
                a, e = max(t0, lo), min(t1, lo + n)
                if rope and a < e:
                    dn = dn.clone()
                    tab = slice(a - lo, e - lo)
                    dn[:, a - t0:e - t0] = rb.rotate(dn[:, a - t0:e - t0], cos[tab], sin[tab], rope)
                dy[i][b, :, t0:t1] = dn.to(dtype)
                sums[i].add(c, N)
                del c, dn
    ins = [packed[..., i * HD:(i + 1) * HD] for i in range(3)]
    exp = [s.expect() for s in sums]
    return dict(packed=packed, ins=ins, g=[t.to(dtype) for t in g], cos=cos, sin=sin, dy=dy, want=want,
                dg=[e[0] for e in exp], db=[e[1] for e in exp])


def run_prep_bwd(cuda, B, S, H, D, norm, rope, lo, n, dtype, seed, r0=0, tail=0):
    """The census through svgb_qkv_prep_bwd, reading rows [r0, r0 + S) of NaN-filled gradients of r0 + S + tail
    rows: any read outside that range turns the result into NaN."""
    cs = prep_census(cuda, B, S, H, D, norm, rope, lo, n, dtype, seed)
    dy = []
    for t in cs["dy"]:
        full = torch.full((B, H, r0 + S + tail, D), NAN, dtype=dtype, device=cuda)
        full[:, :, r0:r0 + S] = t
        dy.append(full)
    del cs["dy"]
    dx, dg, db = prep_bwd_f32(dy, cs["ins"][0], cs["ins"][1], H, S, r0, norm, cs["g"][0], cs["g"][1], rope, cs["cos"],
                              cs["sin"], lo, n if rope else 0)
    what = f"qkv_prep_bwd B {B} S {S} H {H} D {D} norm {norm} rope {rope} lo {lo} n {n} r0 {r0} {dtype}"
    for i in range(3):
        assert_rows(dx[i], cs["want"][i], f"{what}: d{'qkv'[i]}_in")
    for i in range(2):
        assert_bits(dg[i], cs["dg"][i], f"{what}: dgamma_{'qk'[i]}")
        if norm == 2:
            assert_bits(db[i], cs["db"][i], f"{what}: dbeta_{'qk'[i]}")


CASE = "B, S, H, D, norm, rope, lo, n, dtype, seed, r0, tail"


@pytest.mark.parametrize(CASE, rb.PREP_CASES)
def test_prep_bwd_census_per_head(cuda, B, S, H, D, norm, rope, lo, n, dtype, seed, r0, tail):
    """Per-head RMS / LayerNorm x RoPE (none, text last, text first, complex) x D x dtype, B = 2, packed strided
    inputs, reading rows [37, 37 + S) of NaN-filled gradients of 37 + S + 11 rows."""
    run_prep_bwd(cuda, B, S, H, D, norm, rope, lo, n, rw.DT[dtype], seed, r0, tail)


@pytest.mark.parametrize(CASE, rb.PREP_CASES_THRESHOLD)
def test_prep_bwd_census_persistent_threshold(cuda, B, S, H, D, norm, rope, lo, n, dtype, seed, r0, tail):
    """B = 2, S_in just below and just above RPB * (592 // B), the token count where the persistent walk takes a
    second pass; neither a multiple of RPB, so the last CTA has dead lanes that must add nothing to dgamma."""
    run_prep_bwd(cuda, B, S, H, D, norm, rope, lo, n, rw.DT[dtype], seed, r0, tail)


@pytest.mark.parametrize(CASE, rb.HIDDEN_CASES)
def test_prep_bwd_census_hidden(cuda, B, S, H, D, norm, rope, lo, n, dtype, seed, r0, tail):
    """NORM_RMS_HIDDEN: H*D/8 not a multiple of 128 (threads past H*LPR return early), B*S below 592 / cols (one
    token per split) and well above it, splits that cross the batch boundary (rb.HIDDEN_CASES)."""
    run_prep_bwd(cuda, B, S, H, D, norm, rope, lo, n, rw.DT[dtype], seed, r0, tail)


@pytest.mark.parametrize(CASE, rb.PREP_CASES_FULL, ids=["wan720p", "hunyuan720p"])
def test_prep_bwd_census_720p(cuda, B, S, H, D, norm, rope, lo, n, dtype, seed, r0, tail):
    """Wan 2.1 720p (S = 75 600, RMS over the hidden row of 40 * 128, complex RoPE on every token) and HunyuanVideo
    720p's single block (S = 119 056, H = 24, D = 128, per-head RMS, RoPE on all but the last 256 tokens)."""
    run_prep_bwd(cuda, B, S, H, D, norm, rope, lo, n, rw.DT[dtype], seed, r0, tail)


# ---- 3. autograd wiring ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layer", [False, True])
def test_row_norm_autograd_on_a_view(cuda, layer):
    """rms_norm_ / layer_norm_ in place on a .view(-1, n) of a non-leaf: x, gamma (and beta) get the census
    gradients."""
    from svgb200 import core

    _, n, dtype, m, seed = rb.AUTOGRAD_ROW_CASES[layer]
    dtype, shape = rw.DT[dtype], (2, 7, 3)
    assert m == 2 * 7 * 3
    g = rb.gamma(seed, n, cuda)
    c = rb.rows(seed, torch.arange(m, device=cuda), n, g, layer=layer)
    x0 = c["x"].view(*shape, n).to(dtype).requires_grad_()
    w = g.to(dtype).requires_grad_()
    b = torch.zeros(n, dtype=dtype, device=cuda).requires_grad_()
    y = x0.clone()
    if layer:
        core.layer_norm_(y.view(-1, n), w, b)
    else:
        core.rms_norm_(y.view(-1, n), w, rb.RMS_EPS)
    poison(cuda)
    y.backward(c["dn"].to(dtype).view(*shape, n))
    assert_bits(x0.grad, c["dx"].to(dtype).view(*shape, n), "dx")
    # the wrappers round the fp32 parameter gradients once to the weight dtype
    assert_bits(w.grad, (c["dn"] * c["xh"]).sum(0).float().to(dtype), "dgamma")
    if layer:
        assert_bits(b.grad, c["dn"].sum(0).float().to(dtype), "dbeta")


def check_prep_grads(cs, packed_grad, wg, what, norm):
    HD = cs["want"][0].shape[-1]
    for i in range(3):
        assert_bits(packed_grad[..., i * HD:(i + 1) * HD], cs["want"][i], f"{what}: d{'qkv'[i]}_in")
    for i in range(2):
        assert_bits(wg[i], cs["dg"][i].to(wg[i].dtype), f"{what}: dgamma_{'qk'[i]}")
        if norm == 2:
            assert_bits(wg[2 + i], cs["db"][i].to(wg[i].dtype), f"{what}: dbeta_{'qk'[i]}")


def test_qkv_prep_autograd(cuda):
    """core.qkv_prep under autograd (LayerNorm, interleaved RoPE text first, rows [5, 5 + S) of S + 9): the packed
    projection and all four weights get the census gradients."""
    from svgb200 import core

    B, S, H, D, norm, rope, txt, n, dtype, seed = rb.AUTOGRAD_PREP_CASES[0]
    dtype, r0 = rw.DT[dtype], 5
    cs = prep_census(cuda, B, S, H, D, norm, rope, txt, n, dtype, seed)
    packed = cs["packed"].requires_grad_()
    qi, ki, vi = (packed[..., i * H * D:(i + 1) * H * D] for i in range(3))
    w = [t.clone().requires_grad_() for t in cs["g"]]
    bias = [torch.zeros(D, dtype=dtype, device=cuda).requires_grad_() for _ in range(2)]
    outs = core.qkv_prep(qi, ki, vi, H, out_row0=r0, out_rows=S + 9, norm=core.NORM_LAYER, gamma_q=w[0],
                         gamma_k=w[1], beta_q=bias[0], beta_k=bias[1], rope=1, cos=cs["cos"], sin=cs["sin"],
                         rope_lo=txt, rope_n=n)
    grads = []
    for t in cs["dy"]:
        full = torch.full((B, H, S + 9, D), NAN, dtype=dtype, device=cuda)
        full[:, :, r0:r0 + S] = t
        grads.append(full)
    poison(cuda)
    torch.autograd.backward(outs, grads)
    check_prep_grads(cs, packed.grad, [w[0].grad, w[1].grad, bias[0].grad, bias[1].grad], "qkv_prep", 2)


def test_wan_qkv_autograd(cuda):
    """prep.wan_qkv: RMS over the hidden row of 40 * 128, complex RoPE on every token."""
    from svgb200 import prep

    B, S, H, D, norm, rope, lo, n, dtype, seed = rb.AUTOGRAD_PREP_CASES[1]
    cs = prep_census(cuda, B, S, H, D, norm, rope, lo, n, rw.DT[dtype], seed)
    packed = cs["packed"].requires_grad_()
    qi, ki, vi = (packed[..., i * H * D:(i + 1) * H * D] for i in range(3))
    w = [t.clone().requires_grad_() for t in cs["g"]]
    outs = prep.wan_qkv(qi, ki, vi, H, w[0], w[1], rb.RMS_EPS, cs["cos"], cs["sin"])
    poison(cuda)
    torch.autograd.backward(outs, cs["dy"])
    check_prep_grads(cs, packed.grad, [w[0].grad, w[1].grad], "wan_qkv", 3)


def test_hunyuan_double_block_autograd(cuda):
    """prep.hunyuan_double_block_qkv: the video stream (RMS + RoPE, rows [0, Sv)) and the prompt stream (its own RMS
    weights, no RoPE, rows [Sv, Sv + St)) write one output and read their own rows of its gradient."""
    from svgb200 import prep

    vid, txt = (prep_census(cuda, *c[:8], rw.DT[c[8]], c[9]) for c in rb.AUTOGRAD_PREP_CASES[2:])
    H, D = rb.AUTOGRAD_PREP_CASES[2][2:4]
    leaves = [cs["packed"].requires_grad_() for cs in (vid, txt)]
    ins = [p[..., i * H * D:(i + 1) * H * D] for p in leaves for i in range(3)]
    w = [t.clone().requires_grad_() for cs in (vid, txt) for t in cs["g"]]
    outs = prep.hunyuan_double_block_qkv(*ins, H, w[0], w[1], w[2], w[3], rb.RMS_EPS, vid["cos"], vid["sin"])
    assert "_QkvPrep" in outs[0].grad_fn.name()
    grads = [torch.cat([vid["dy"][i], txt["dy"][i]], 2) for i in range(3)]
    poison(cuda)
    torch.autograd.backward(outs, grads)
    check_prep_grads(vid, leaves[0].grad, [w[0].grad, w[1].grad], "double block, video stream", 1)
    check_prep_grads(txt, leaves[1].grad, [w[2].grad, w[3].grad], "double block, prompt stream", 1)
