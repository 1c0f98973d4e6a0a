"""GPU: the element-wise and reduction kernels between the backward GEMMs (csrc/backward.cu) at their edges against
float64 autograd / einsum on the bf16 / fp32 values the kernels read (tests/kernel_check.py bounds; NaN-filled regions
must stay untouched; one sensitivity test per family).

Every op is called the way training.py calls it: FiLM and dFiLM as column windows of a per-layer table, the residual
gradient accumulated in place, dFiLM / dgamma starting non-zero.  Table columns outside the window hold random values
(the kernels add into the table) and must come back exactly unchanged.  Gradient tables accumulate with atomicAdd, so
their bound is acc_eps(total rows), not bit-exactness.

  ops.rmsnorm_film_bwd   every dim 128..1024, rows_per_batch 32 / 100 / 129 (partial 64-row CTAs), FiLM / gamma /
                         gamma without dgamma
  ops.geglu_bwd          Dp 128..1024, saturated gates, enough rows that the grid-stride loop wraps
  ops.wavenet_gate_bwd   every row-lane layout (8, 4, 2, 1 lanes; idle threads at dim 384 / 640), 4 groups, strided
                         c / dy / dc windows, |z| past the +-20 clamp
  ops.film_wgrad         B > 32 (chunked: overwrite then accumulate), cols % 4 != 0, rows off 64
  ops.colsum             partial 512-column blocks, rows around the 256-row chunk
  ops.group_sum, accum_bf16, mse_bwd
"""
import math

import pytest
import torch

from kernel_check import (U_BF16, U_F32, acc_eps, assert_close, assert_nan, assert_rejects, gen as _gen,
                          nan_buf as _nan_buf)

pytestmark = pytest.mark.gpu
bf = torch.bfloat16
dev = "cuda"
NAN = float("nan")
DIMS = [128 * v for v in range(1, 9)]


def _assert_outside_unchanged(table, before, lo, hi, what):
    assert torch.equal(table[:, :lo], before[:, :lo]) and torch.equal(table[:, hi:], before[:, hi:]), \
        f"{what}: table columns outside the window changed"


# ---------------------------------------------------------------------------------------------------------------
# rmsnorm_film_bwd
# ---------------------------------------------------------------------------------------------------------------
def _rms_bwd_case(mode, B, N, D, seed):
    from naturalspeech2_pytorch_b200 import ops
    g = _gen(seed)
    x = torch.randn(B, N, D, device=dev, generator=g) * 2
    dh = torch.randn(B, N, D, device=dev, generator=g).to(bf)
    dxr0 = torch.randn(B, N, D, device=dev, generator=g)
    fo, total = 2 * D, 6 * D + 4                                       # layer 1 of a 3-layer table, 4 spare columns
    table = torch.randn(B, total, device=dev, generator=g) * 0.5 + 1
    dtable = torch.randn(B, total, device=dev, generator=g)
    dtable0 = dtable.clone()
    gamma = torch.randn(D, device=dev, generator=g) * 0.3 + 1
    gbuf, dgamma = _nan_buf((D,))
    dgamma.copy_(torch.randn(D, device=dev, generator=g))
    dgamma0 = dgamma.clone()
    xbuf, dxr = _nan_buf((B, N, D))
    dxr.copy_(dxr0)
    bbuf, dxr_bf = _nan_buf((B, N, D), bf)
    film = table[:, fo:fo + 2 * D]
    if mode == "film":
        ops.rmsnorm_film_bwd(x, dh, dxr, dxr_bf, rows_per_batch=N, film=film, dfilm=dtable[:, fo:fo + 2 * D])
    else:
        ops.rmsnorm_film_bwd(x, dh, dxr, dxr_bf, rows_per_batch=N, gamma=gamma,
                             dgamma=dgamma if mode == "gamma" else None)
    assert_nan(xbuf[dxr.numel():], "past dxr")
    assert_nan(bbuf[dxr.numel():], "past dxr_bf")
    assert_nan(gbuf[D:], "past dgamma")
    assert torch.equal(dxr_bf, dxr.to(bf)), "dxr_bf is bf16(dxr)"
    if mode == "film":
        _assert_outside_unchanged(dtable, dtable0, fo, fo + 2 * D, "dfilm")
    else:
        assert torch.equal(dtable, dtable0), "no FiLM: the table is not touched"
    if mode != "gamma":
        assert torch.equal(dgamma, dgamma0), "no dgamma requested: dgamma is not touched"
    return dict(x=x, dh=dh, dxr0=dxr0, dxr=dxr, film=film, dfilm=dtable[:, fo:fo + 2 * D],
                dfilm0=dtable0[:, fo:fo + 2 * D], gamma=gamma, dgamma=dgamma, dgamma0=dgamma0)


def _rms_bwd_ref(mode, c, drop_projection=False):
    """fp64 autograd of h = normalize(x) sqrt(D) * gamma * fg + fb, and the bound of each gradient: the fp32 sum of
    squares and the u . du sum over D (acc_eps(D)) plus a few roundings relative to s (|du| + |u| (|dot| + mean|u du|));
    the column sums over the rows (acc_eps(rows)) relative to sum |dh u g| and sum |dh|."""
    x, dh = c["x"], c["dh"].double()
    B, N, D = x.shape
    x64 = x.double().requires_grad_(True)
    u = x64 / x64.norm(dim=-1, keepdim=True).clamp_min(1e-12) * math.sqrt(D)
    f64 = c["film"].double().requires_grad_(True)
    g64 = c["gamma"].double().requires_grad_(True)
    h = u * f64[:, None, :D] + f64[:, None, D:] if mode == "film" else u * g64
    h.backward(dh)
    with torch.no_grad():
        u = u.detach()
        s = math.sqrt(D) / x.double().norm(dim=-1, keepdim=True)
        gam = f64[:, None, :D] if mode == "film" else g64
        du = dh * gam
        dot = (u * du).sum(-1, keepdim=True) / D
        mdot = (u * du).abs().sum(-1, keepdim=True) / D
        eps = acc_eps(D) + 2.0 ** -20
        dx = s * du if drop_projection else x64.grad
        dx_bound = 2 * eps * s * (du.abs() + u.abs() * (dot.abs() + mdot))
        out = dict(dx=dx, dx_bound=dx_bound, dx_rel=4 * eps)
        if mode == "film":
            out["dfilm"] = f64.grad
            mag = torch.cat(((dh * u).abs().sum(1), dh.abs().sum(1)), dim=-1)
            out["dfilm_bound"] = (acc_eps(N) + eps) * mag
            out["dfilm_rel"] = 4 * (acc_eps(N) + eps)
        else:
            out["dgamma"] = g64.grad
            out["dgamma_bound"] = (acc_eps(B * N) + eps) * (dh * u).abs().sum((0, 1))
            out["dgamma_rel"] = 4 * (acc_eps(B * N) + eps)
    return out


@pytest.mark.parametrize("D", DIMS)
@pytest.mark.parametrize("mode", ["film", "gamma", "gamma-no-dgamma"])
def test_rmsnorm_film_bwd(mode, D):
    for N in (32, 100, 129):      # the perceiver's M = 32; 100 / 129 rows leave a partial 64-row CTA per batch
        c = _rms_bwd_case(mode, 3, N, D, seed=D + N)
        r = _rms_bwd_ref(mode, c)
        what = f"{mode} D={D} N={N}"
        got_dx = c["dxr"].double() - c["dxr0"].double()
        assert_close(got_dx, r["dx"], r["dx_bound"] + U_F32 * (c["dxr"].double().abs() + c["dxr0"].double().abs()),
                     r["dx_rel"], f"{what}: dx")
        if mode == "film":
            got = c["dfilm"].double() - c["dfilm0"].double()
            bound = r["dfilm_bound"] + U_F32 * (c["dfilm"].double().abs() + c["dfilm0"].double().abs())
            assert_close(got, r["dfilm"], bound, r["dfilm_rel"], f"{what}: dfilm")
        elif mode == "gamma":
            got = c["dgamma"].double() - c["dgamma0"].double()
            bound = r["dgamma_bound"] + U_F32 * (c["dgamma"].double().abs() + c["dgamma0"].double().abs())
            assert_close(got, r["dgamma"], bound, r["dgamma_rel"], f"{what}: dgamma")


def test_rmsnorm_film_bwd_sensitivity():
    c = _rms_bwd_case("film", 3, 100, 512, seed=1)
    r = _rms_bwd_ref("film", c)
    wrong = _rms_bwd_ref("film", c, drop_projection=True)
    got_dx = c["dxr"].double() - c["dxr0"].double()
    bound = r["dx_bound"] + U_F32 * (c["dxr"].double().abs() + c["dxr0"].double().abs())
    assert_rejects(got_dx, wrong["dx"], bound, r["dx_rel"], "u . du projection term dropped")


# ---------------------------------------------------------------------------------------------------------------
# geglu_bwd
# ---------------------------------------------------------------------------------------------------------------
def _geglu_case(rows, dp, seed):
    from naturalspeech2_pytorch_b200 import ops
    g = _gen(seed)
    pre = (torch.randn(rows, 2 * dp, device=dev, generator=g) * 2).to(bf)
    sat = torch.tensor([-30., -10., -6., 6., 10., 30.], device=dev).to(bf)
    pre[0, 128:134] = sat                                               # saturated gates: cdf 0 / 1, pdf 0
    dg = torch.randn(rows, dp, device=dev, generator=g).to(bf)
    buf, p = _nan_buf((rows, 2 * dp), bf)
    p.copy_(pre)
    ops.geglu_bwd(p, dg)
    assert_nan(buf[p.numel():], "past pre")
    return pre, dg, p


def _geglu_ref(pre, dg, drop_pdf=False):
    """d val = dg gelu(gate), d gate = dg val (Phi(gate) + gate phi(gate)) in fp64; bound: bf16 output rounding plus
    erff / expf (2 ulp each, CUDA Math API) and the fp32 products - erff's error is absolute near Phi = 0."""
    rows, dp = dg.shape
    t = pre.double().view(rows, dp // 128, 2, 128)
    v, gt = t[:, :, 0], t[:, :, 1]
    d = dg.double().view(rows, dp // 128, 128)
    cdf = 0.5 * (1 + torch.erf(gt / math.sqrt(2)))
    pdf = torch.exp(-0.5 * gt * gt) / math.sqrt(2 * math.pi)
    dval = d * gt * cdf
    dgate = d * v * (cdf if drop_pdf else cdf + gt * pdf)
    bval = U_BF16 * dval.abs() + (d * gt).abs() * (2.0 ** -22 + 2.0 ** -21 * cdf)
    bgate = U_BF16 * dgate.abs() + (d * v).abs() * (2.0 ** -22 + 2.0 ** -21 * cdf
                                                    + gt.abs() * pdf * (2.0 ** -21 + 2.0 ** -24 * gt * gt))
    pack = lambda a, b: torch.stack((a, b), dim=2).reshape(rows, 2 * dp)
    return pack(dval, dgate), pack(bval, bgate)


@pytest.mark.parametrize("rows,dp", [(1, 128), (300, 384), (37, 1024), (10007, 128)])   # 10007 x 64 pairs > 2368 CTAs
def test_geglu_bwd(rows, dp):
    pre, dg, got = _geglu_case(rows, dp, seed=rows + dp)
    ref, bound = _geglu_ref(pre, dg)
    assert_close(got, ref, bound, 2.0 ** -8, f"rows={rows} dp={dp}")


def test_geglu_bwd_sensitivity():
    pre, dg, got = _geglu_case(300, 384, seed=2)
    _, bound = _geglu_ref(pre, dg)
    wrong, _ = _geglu_ref(pre, dg, drop_pdf=True)
    assert_rejects(got, wrong, bound, 2.0 ** -8, "gate * pdf(gate) term dropped")


# ---------------------------------------------------------------------------------------------------------------
# wavenet_gate_bwd
# ---------------------------------------------------------------------------------------------------------------
def _wn_case(B, N, D, G, seed):
    from naturalspeech2_pytorch_b200 import ops
    g = _gen(seed)
    cols, pad = G * D, 12
    cw = torch.full((B, N, cols + pad), NAN, device=dev, dtype=bf)
    cw[..., :cols] = (torch.randn(B, N, cols, device=dev, generator=g) * 2).to(bf)
    cw[0, :4, :4] = torch.tensor([[-40., -21., 21., 40.]], device=dev).to(bf)    # |z| past the +-20 clamp
    dyw = torch.full((B, N, cols + pad), NAN, device=dev, dtype=bf)
    dyw[..., 4:4 + cols] = torch.randn(B, N, cols, device=dev, generator=g).to(bf)
    dcw = torch.full((B, N, cols + pad), NAN, device=dev, dtype=bf)
    c, dy, dc = cw[..., :cols], dyw[..., 4:4 + cols], dcw[..., 8:8 + cols]
    fo = 6 * D                                                          # after three 2D-wide FiLM layers
    total = fo + G * 2 * D + 8
    table = torch.randn(B, total, device=dev, generator=g) * 0.5 + 0.5
    table[0, fo:fo + 4] = 1.0                                           # fg = 1 where c = +-40 / +-21
    table[0, fo + D:fo + D + 4] = 0.0
    dtable = torch.randn(B, total, device=dev, generator=g)
    dtable0 = dtable.clone()
    ops.wavenet_gate_bwd(c, dy, dc, table[:, fo:], dtable[:, fo:], dim=D, groups=G, film_group_stride=2 * D)
    assert_nan(dcw[..., :8], "left of dc")
    assert_nan(dcw[..., 8 + cols:], "right of dc")
    _assert_outside_unchanged(dtable, dtable0, fo, fo + G * 2 * D, "dfilm")
    return dict(c=c, dy=dy, dc=dc, film=table[:, fo:fo + G * 2 * D], dfilm=dtable[:, fo:fo + G * 2 * D],
                dfilm0=dtable0[:, fo:fo + G * 2 * D])


def _wn_ref(c, D, G, swap=False):
    """y = tanh(z) sigmoid(z), z = c fg + fb, in fp64 without the clamp.  Bound: __expf has 2 + floor(1.173 |z|) ulp
    and __fdividef 2 ulp (CUDA Math API, intrinsic functions), so the derivative factor is within 8 (e_u + 2^-22)
    absolutely; the fma of z adds 2^-24 |z|; past |z| = 20 the kernel's clamped factor (< 3e-9) replaces the true one."""
    B, N, _ = c["c"].shape
    cv = c["c"].double().view(B, N, G, D)
    dv = c["dy"].double().view(B, N, G, D)
    f = c["film"].double().view(B, G, 2, D)
    ga, be = f[:, None, :, 0], f[:, None, :, 1]
    z = cv * ga + be
    th, sg = torch.tanh(z), torch.sigmoid(z)
    F = (1 - th * th) * sg + th * sg * (1 - sg)
    dz = dv * F
    dc = dz * ga
    dgam, dbeta = (dz * cv).sum(1), dz.sum(1)                          # (B, G, D)
    e_u = (2 + 1.173 * z.abs().clamp_max(20)) * 2.0 ** -23
    dF = 8 * (e_u + 2.0 ** -22) + 2.0 ** -24 * z.abs() + torch.where(z.abs() > 20, 1e-8, 0.0)
    bdz = dv.abs() * dF
    dc_bound = (U_BF16 + 2.0 ** -23) * dc.abs() + ga.abs() * bdz
    N_ = N
    bgam = acc_eps(N_) * (dz * cv).abs().sum(1) + (cv.abs() * bdz).sum(1)
    bbeta = acc_eps(N_) * dz.abs().sum(1) + bdz.sum(1)
    first, second = (dbeta, dgam) if swap else (dgam, dbeta)
    dfilm = torch.stack((first, second), dim=2).reshape(B, G * 2 * D)
    dfilm_bound = torch.stack((bgam, bbeta), dim=2).reshape(B, G * 2 * D)
    return dc.reshape(B, N, G * D), dc_bound.reshape(B, N, G * D), dfilm, dfilm_bound, 4 * acc_eps(N) + 2.0 ** -15


@pytest.mark.parametrize("D", [128, 256, 384, 512, 640, 1024])   # 8, 4, 2 (64 idle threads), 2, 1 (96 idle), 1 row lanes
@pytest.mark.parametrize("G", [1, 4])
def test_wavenet_gate_bwd(D, G):
    c = _wn_case(2, 70, D, G, seed=D + G)
    dc, dc_bound, dfilm, dfilm_bound, rel = _wn_ref(c, D, G)
    assert_close(c["dc"], dc, dc_bound, 2.0 ** -8, f"D={D} G={G}: dc")
    got = c["dfilm"].double() - c["dfilm0"].double()
    bound = dfilm_bound + U_F32 * (c["dfilm"].double().abs() + c["dfilm0"].double().abs())
    assert_close(got, dfilm, bound, rel, f"D={D} G={G}: dfilm")


def test_wavenet_gate_bwd_sensitivity():
    c = _wn_case(2, 70, 256, 2, seed=3)
    _, _, _, dfilm_bound, rel = _wn_ref(c, 256, 2)
    _, _, wrong, _, _ = _wn_ref(c, 256, 2, swap=True)
    got = c["dfilm"].double() - c["dfilm0"].double()
    bound = dfilm_bound + U_F32 * (c["dfilm"].double().abs() + c["dfilm0"].double().abs())
    assert_rejects(got, wrong, bound, rel, "dfilm gamma and beta halves swapped")


# ---------------------------------------------------------------------------------------------------------------
# film_wgrad
# ---------------------------------------------------------------------------------------------------------------
def _fw_case(B, rows, cols, accumulate, seed):
    from naturalspeech2_pytorch_b200 import ops
    g = _gen(seed)
    wide = torch.randn(B, rows + 40, device=dev, generator=g)
    dfilm = wide[:, 16:16 + rows]                                       # a column window of the per-layer table
    t = torch.randn(B, cols, device=dev, generator=g)
    buf, dw = _nan_buf((rows, cols))
    start = torch.zeros(rows, cols, device=dev)
    if accumulate:
        start = torch.randn(rows, cols, device=dev, generator=g)
        dw.copy_(start)                                                 # overwrite mode leaves dw NaN: never read
    ops.film_wgrad(dfilm, t, dw, accumulate=accumulate)
    assert_nan(buf[dw.numel():], "past dw")
    return dfilm, t, start, dw


def _fw_bound(dfilm, t, got, start):
    B = dfilm.shape[0]
    return acc_eps(B) * (dfilm.double().abs().T @ t.double().abs()) + U_F32 * (got.double().abs() + start.double().abs())


@pytest.mark.parametrize("B", [5, 32, 33, 70])
@pytest.mark.parametrize("rows,cols", [(64, 256), (100, 300), (130, 301), (7, 5)])
def test_film_wgrad(B, rows, cols):
    for accumulate in (True, False):
        dfilm, t, start, got = _fw_case(B, rows, cols, accumulate, seed=B * 1000 + rows + cols)
        ref = dfilm.double().T @ t.double()
        assert_close(got.double() - start.double(), ref, _fw_bound(dfilm, t, got, start), 4 * acc_eps(B),
                     f"B={B} rows={rows} cols={cols} accumulate={accumulate}")


def test_film_wgrad_sensitivity():
    dfilm, t, start, got = _fw_case(33, 100, 300, False, seed=4)
    wrong = dfilm[:32].double().T @ t[:32].double()
    assert_rejects(got.double() - start.double(), wrong, _fw_bound(dfilm, t, got, start), 4 * acc_eps(33),
                   "33rd batch row left out")


# ---------------------------------------------------------------------------------------------------------------
# colsum, group_sum
# ---------------------------------------------------------------------------------------------------------------
def _colsum_case(rows, cols, seed):
    from naturalspeech2_pytorch_b200 import ops
    g = _gen(seed)
    wide = torch.full((rows, cols + 10), NAN, device=dev, dtype=bf)
    wide[:, 2:2 + cols] = torch.randn(rows, cols, device=dev, generator=g).to(bf)
    t = wide[:, 2:2 + cols]                                             # row-strided window, NaN around it
    buf, out = _nan_buf((cols,))
    out.copy_(torch.randn(cols, device=dev, generator=g))
    start = out.clone()
    ops.colsum(t, out)
    assert_nan(buf[cols:], "past out")
    bound = acc_eps(rows) * t.double().abs().sum(0) + U_F32 * (out.double().abs() + start.double().abs())
    return t, start, out, bound


@pytest.mark.parametrize("rows", [1, 255, 256, 257, 513])
@pytest.mark.parametrize("cols", [6, 514, 1000])
def test_colsum(rows, cols):
    t, start, got, bound = _colsum_case(rows, cols, seed=rows * 7 + cols)
    assert_close(got.double() - start.double(), t.double().sum(0), bound, 4 * acc_eps(rows), f"rows={rows} cols={cols}")


def test_colsum_sensitivity():
    t, start, got, bound = _colsum_case(513, 514, seed=5)
    keep = torch.ones(513, dtype=torch.bool, device=dev)
    keep[256] = False
    assert_rejects(got.double() - start.double(), t.double()[keep].sum(0), bound, 4 * acc_eps(513), "row 256 left out")


@pytest.mark.parametrize("rows,dim,groups", [(1, 2, 1), (90, 128, 4), (33, 130, 8)])
def test_group_sum(rows, dim, groups):
    from naturalspeech2_pytorch_b200 import ops
    t = torch.randn(rows, groups * dim, device=dev, generator=_gen(rows + dim)).to(bf)
    buf, out = _nan_buf((rows, dim), bf)
    ops.group_sum(t, out, dim=dim, groups=groups)
    assert_nan(buf[out.numel():], "past out")
    tg = t.double().view(rows, groups, dim)
    ref = tg.sum(1)
    assert_close(out, ref, U_BF16 * ref.abs() + groups * 2.0 ** -24 * tg.abs().sum(1), 2.0 ** -8, "group_sum")


# ---------------------------------------------------------------------------------------------------------------
# accum_bf16, mse_bwd: one fp32 add / product each, bit-exact
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("count", [4, 1000, 2_500_004])   # 2.5M: past 2368 CTAs x 256 float4, the loop wraps
def test_accum_bf16_exact(count):
    from naturalspeech2_pytorch_b200 import ops
    g = _gen(count)
    acc0 = torch.randn(count, device=dev, generator=g)
    t = torch.randn(count, device=dev, generator=g).to(bf)
    for with_bf in (False, True):
        buf, acc = _nan_buf((count,))
        acc.copy_(acc0)
        bbuf, acc_bf = _nan_buf((count,), bf)
        ops.accum_bf16(acc, t, acc_bf if with_bf else None)
        assert_nan(buf[count:], "past acc")
        assert torch.equal(acc, acc0 + t.float()), f"count={count}"
        if with_bf:
            assert torch.equal(acc_bf, acc.to(bf))
        else:
            assert_nan(bbuf, "acc_bf not requested")


@pytest.mark.parametrize("B,per", [(1, 4), (9, 1000), (3, 70004)])
def test_mse_bwd_exact(B, per):
    from naturalspeech2_pytorch_b200 import ops
    g = _gen(B + per)
    p, t = torch.randn(B, per, device=dev, generator=g), torch.randn(B, per, device=dev, generator=g)
    coef = torch.randn(B, device=dev, generator=g)
    ref = coef[:, None] * (p - t)
    bf_buf, ob = _nan_buf((B, per), bf)
    f_buf, of = _nan_buf((B, per))
    ops.mse_bwd(p, t, coef, out_bf=ob, out_f32=of)
    assert_nan(bf_buf[ob.numel():], "past out_bf")
    assert_nan(f_buf[of.numel():], "past out_f32")
    assert torch.equal(of, ref), "fp32 seed"
    assert torch.equal(ob, ref.to(bf)), "bf16 seed"
    of2 = torch.full_like(p, NAN)
    ops.mse_bwd(p, t, coef, out_f32=of2)
    assert torch.equal(of2, ref), "fp32 output alone"
