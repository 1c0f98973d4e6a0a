"""GPU: the element-wise kernels of csrc/elementwise.cu at their edges against float64 references
(tests/kernel_check.py bounds; NaN-filled regions must stay untouched; one sensitivity test per family).

  ops.rmsnorm_film / rmsnorm_f32   every dim 128..1024 (VEC 1..8) in both kernel variants, zero rows, FiLM as a
                                   column window of a wider table; bit-identical across variants and SM limits
  ops.time_cond / small_linear     batches around the 8-row blocking and the 64-row launch limit, k up to the shared
                                   memory chunking, n_out off the warps per CTA, act / bias on and off, strided x / out
  q_sample, x_start, ddim_step,    all three objectives, alpha = 0 / sigma = 0 samples, batch > 8 (quarter grid),
  mse_rows, cfg_combine            grid-stride wrap-around; mse_rows deterministic
  groupnorm_silu                   channels per group = 4, a constant group, a mean offset of 1000
  rowdot, mean_rows                dims off the float4 / warp tiling, rows off the 8-row CTAs
  casts, cond_inject, select_rows, copies, casts and single fp32 adds: bit-exact against the same torch fp32 expression
  transpose_cast, embedding_bf16,
  expand_encodings

Most tests run under `sm2` (every persistent grid sized for 2 SMs), so the streaming RMSNorm variant and the
grid-stride loops are reached at small sizes.  The results must not depend on the limit.
"""
import math

import pytest
import torch

from kernel_check import (U_BF16, U_F32, acc_eps, assert_close, assert_nan, assert_rejects, gen as _gen,
                          nan_buf as _nan_buf, sm_limit)

pytestmark = pytest.mark.gpu
bf = torch.bfloat16
dev = "cuda"
NAN = float("nan")
DIMS = [128 * v for v in range(1, 9)]
TINY = float(torch.tensor(1e-10, dtype=torch.float32))   # safe_div's clamp as the kernels hold it (fp32)


@pytest.fixture(scope="module")
def sm2():
    """Every kernel's persistent grid sized for 2 SMs; yields the previous limit."""
    with sm_limit(2) as prev:
        yield prev


def _silu64(z):
    return z * torch.sigmoid(z)


# ---------------------------------------------------------------------------------------------------------------
# RMSNorm (+gamma) (+FiLM)
# ---------------------------------------------------------------------------------------------------------------
def _rms_inputs(B, N, D, seed):
    g = _gen(seed)
    x = torch.randn(B, N, D, device=dev, generator=g) * 3
    x[0, 0] = 0                                                        # all-zero row: the 1e-12 clamp
    x[-1, -1] *= 1e-3
    gamma = torch.randn(D, device=dev, generator=g) * 0.5 + 1
    table = torch.full((B, 4 * D), NAN, device=dev)                   # [.. | gamma_b | beta_b | ..]: only the window is read
    table[:, D:3 * D] = torch.randn(B, 2 * D, device=dev, generator=g) * 0.5 + 1
    return x, gamma, table[:, D:3 * D]


def _rms_run(mode, x, gamma, film):
    from naturalspeech2_pytorch_b200 import ops
    dt = torch.float32 if mode.startswith("f32") else bf
    buf, out = _nan_buf(tuple(x.shape), dt)
    if mode == "film":
        ops.rmsnorm_film(x, out, film=film)
    elif mode == "gamma":
        ops.rmsnorm_film(x, out, gamma=gamma)
    elif mode == "f32":
        ops.rmsnorm_f32(x, out, gamma)
    else:
        ops.rmsnorm_f32(x, out, None)
    assert_nan(buf[out.numel():], f"{mode}: past the output")
    return out


def _rms_ref(mode, x, gamma, film, skip_last4=False):
    """(reference, bound, rel-L2): fp32 sum of squares over D (acc_eps) and a few roundings (sqrt, div, scale, gamma,
    FiLM fma) relative to |u * gamma * fg|, plus the output rounding."""
    D = x.shape[-1]
    x64 = x.double()
    sq = (x64 * x64)[..., :D - 4] if skip_last4 else x64 * x64
    u = x64 / sq.sum(-1, keepdim=True).sqrt().clamp_min(1e-12) * math.sqrt(D)
    if mode == "film":
        scaled = u * film[:, None, :D].double()
        ref = scaled + film[:, None, D:].double()
    elif mode in ("gamma", "f32"):
        scaled = ref = u * gamma.double()
    else:
        scaled = ref = u
    u_out = U_F32 if mode.startswith("f32") else U_BF16
    bound = u_out * ref.abs() + (acc_eps(D) + 2.0 ** -21) * scaled.abs()
    return ref, bound, u_out + 4 * acc_eps(D)


@pytest.mark.parametrize("D", DIMS)
@pytest.mark.parametrize("mode", ["film", "gamma", "f32"])
def test_rmsnorm(sm2, mode, D):
    # 74 rows: one row per warp with a partial last CTA; 123 and 1055 rows: the streaming variant (>= 121 rows at 2 SMs)
    # with a partial last pass of its 32 / 96 warps
    for B, N in ((2, 37), (3, 41), (5, 211)):
        x, gamma, film = _rms_inputs(B, N, D, seed=D + N)
        got = _rms_run(mode, x, gamma, film)
        ref, bound, rel = _rms_ref(mode, x, gamma, film)
        assert_close(got, ref, bound, rel, f"{mode} D={D} rows={B * N}")
        if mode == "film":
            assert torch.equal(got[0, 0], film[0, D:].to(bf)), "a zero row gives exactly the FiLM shift"
        else:
            assert torch.count_nonzero(got[0, 0]) == 0, "a zero row gives exactly zero"


@pytest.mark.parametrize("D", DIMS)
def test_rmsnorm_variants_bit_identical(sm2, D):
    """rmsnorm_row is shared by both kernels, so a row's bits do not depend on the variant the problem size selects:
    320 rows stream at 2 SMs and take one row per warp with every SM; 40-row slices take one row per warp."""
    B, N = 8, 40
    x, gamma, film = _rms_inputs(B, N, D, seed=7 * D)
    for mode in ("film", "gamma", "f32", "f32-plain"):
        full = _rms_run(mode, x, gamma, film)
        for b in range(B):
            part = _rms_run(mode, x[b:b + 1].contiguous(), gamma, film[b:b + 1])
            assert torch.equal(full[b:b + 1], part), f"{mode} D={D}: slice {b} differs from the full problem"
        with sm_limit(sm2):
            assert torch.equal(full, _rms_run(mode, x, gamma, film)), f"{mode} D={D}: differs across SM limits"


def test_rmsnorm_sensitivity(sm2):
    x, gamma, film = _rms_inputs(3, 41, 512, seed=3)
    got = _rms_run("f32", x, gamma, film)
    _, bound, rel = _rms_ref("f32", x, gamma, film)
    wrong, _, _ = _rms_ref("f32", x, gamma, film, skip_last4=True)
    wrong[0, 0] = 0
    assert_rejects(got, wrong, bound, rel, "last float4 of each row left out of the sum of squares")


# ---------------------------------------------------------------------------------------------------------------
# conditioning-vector layers: time_cond, small_linear
# ---------------------------------------------------------------------------------------------------------------
def _linear_bound(pre_err, ref, act):
    """Bound of act(z) given the bound of z: |silu'| <= 1.1; expf (2 ulp, CUDA Math API), the add and the IEEE divide
    of x / (1 + e^-x) add <= 8 ulp of the result; then the fp32 output rounding."""
    if act:
        return 1.1 * pre_err + (2.0 ** -20 + U_F32) * ref.abs()
    return pre_err + U_F32 * ref.abs()


def _time_feat(times, freqs, swap=False):
    """The kernel's fp32 argument ((t * w) * 2) * pi (pi rounded to fp32), then sin / cos of that fp32 value in fp64:
    the reference of the kernel's sinf / cosf rather than of the range reduction of a large |t * w|."""
    pi32 = torch.tensor(math.pi, dtype=torch.float32, device=dev)
    fr = ((times[:, None] * freqs[None]) * 2.0) * pi32
    s, c = fr.double().sin(), fr.double().cos()
    if swap:
        s, c = c, s
    return torch.cat((times[:, None].double(), s, c), dim=-1)


def _time_case(batch, half, n_out, seed):
    from naturalspeech2_pytorch_b200 import ops
    g = _gen(seed)
    times = torch.rand(batch, device=dev, generator=g)
    freqs = torch.randn(half, device=dev, generator=g) * 8
    freqs[:4] = torch.tensor([60.0, -75.0, 110.0, -150.0], device=dev)   # |2 pi t w| up to ~900
    W = torch.randn(n_out, 2 * half + 1, device=dev, generator=g) / math.sqrt(2 * half + 1)
    bias = torch.randn(n_out, device=dev, generator=g)
    wide = torch.full((batch, n_out + 9), NAN, device=dev)
    out = wide[:, 4:4 + n_out]                                           # a column window of a wider matrix
    ops.time_cond(times, freqs, W, bias, out)
    assert_nan(wide[:, :4], "columns left of out")
    assert_nan(wide[:, 4 + n_out:], "columns right of out")
    return times, freqs, W, bias, out


def _time_ref(times, freqs, W, bias, swap=False):
    """sinf / cosf: 2 ulp over the full range (CUDA C++ Programming Guide, Mathematical Functions, single-precision
    table), i.e. <= 2^-22 |feature|; the fp32 dot product over k = 2 half + 1 terms (acc_eps)."""
    feat = _time_feat(times, freqs, swap)
    z = feat @ W.double().T + bias.double()
    mag = feat.abs() @ W.double().abs().T
    ref = _silu64(z)
    k = feat.shape[1]
    return ref, _linear_bound((acc_eps(k) + 2.0 ** -22) * mag + U_F32 * bias.double().abs(), ref, 1), \
        4 * acc_eps(k) + 2.0 ** -20


@pytest.mark.parametrize("batch", [1, 7, 9, 65, 130])
@pytest.mark.parametrize("half", [8, 64, 1024])
def test_time_cond(sm2, batch, half):
    # half = 1024 -> k = 2049: 24 rows per launch (200 KB of shared memory); 65 / 130 rows: 64 rows per launch
    for n_out in (9, 2048):
        times, freqs, W, bias, got = _time_case(batch, half, n_out, seed=batch * 100 + half + n_out)
        ref, bound, rel = _time_ref(times, freqs, W, bias)
        assert_close(got, ref, bound, rel, f"batch={batch} half={half} n_out={n_out}")


def test_time_cond_sensitivity(sm2):
    times, freqs, W, bias, got = _time_case(9, 64, 2048, seed=11)
    _, bound, rel = _time_ref(times, freqs, W, bias)
    wrong, _, _ = _time_ref(times, freqs, W, bias, swap=True)
    assert_rejects(got, wrong, bound, rel, "sin and cos halves swapped")


def _small_case(batch, k, W, bias, act, n_out, seed):
    from naturalspeech2_pytorch_b200 import ops
    g = _gen(seed)
    xw = torch.full((batch, k + 5), NAN, device=dev)
    xw[:, 2:2 + k] = torch.randn(batch, k, device=dev, generator=g)
    x = xw[:, 2:2 + k]                                                   # row-strided window, NaN around it
    wide = torch.full((batch, n_out + 8), NAN, device=dev)
    out = wide[:, 3:3 + n_out]
    ops.small_linear(x, W[:n_out], bias, out, act=act)
    assert_nan(wide[:, :3], "columns left of out")
    assert_nan(wide[:, 3 + n_out:], "columns right of out")
    return x, out


def _small_ref(x, W, bias, act, drop_last_col=False):
    x64, w64 = x.double(), W.double()
    if drop_last_col:
        x64, w64 = x64[:, :-1], w64[:, :-1]
    z = x64 @ w64.T
    mag = x64.abs() @ w64.abs().T
    pre_err = acc_eps(x.shape[1]) * mag
    if bias is not None:
        z = z + bias.double()
        pre_err = pre_err + U_F32 * bias.double().abs()
    ref = _silu64(z) if act else z
    bound = _linear_bound(pre_err, ref, act)
    # a few outputs (n_out * batch = 1) can sit near a cancellation of the dot product: the rel-L2 bound is at least
    # twice the one the element-wise bound implies
    return ref, bound, max(4 * acc_eps(x.shape[1]) + 2.0 ** -20, 2 * float(bound.norm() / ref.norm()))


@pytest.mark.parametrize("batch", [1, 7, 8, 9, 64, 65, 130])
@pytest.mark.parametrize("k", [1, 31, 33, 512, 2049])
def test_small_linear(sm2, batch, k):
    g = _gen(batch * 10000 + k)
    W = torch.randn(2048, k, device=dev, generator=g) / math.sqrt(k)
    b = torch.randn(2048, device=dev, generator=g)
    for n_out in (1, 7, 9, 2048):
        for act, bias in ((0, b), (1, b), (0, None), (1, None)):
            x, got = _small_case(batch, k, W, None if bias is None else bias[:n_out], act, n_out, seed=n_out + act)
            ref, bound, rel = _small_ref(x, W[:n_out], None if bias is None else bias[:n_out], act)
            assert_close(got, ref, bound, rel, f"batch={batch} k={k} n_out={n_out} act={act} bias={bias is not None}")


def test_small_linear_sensitivity(sm2):
    g = _gen(12)
    W = torch.randn(300, 33, device=dev, generator=g)
    bias = torch.randn(300, device=dev, generator=g)
    x, got = _small_case(9, 33, W, bias, 1, 300, seed=13)
    _, bound, rel = _small_ref(x, W, bias, 1)
    wrong, _, _ = _small_ref(x, W, bias, 1, drop_last_col=True)
    assert_rejects(got, wrong, bound, rel, "last input column left out")


# ---------------------------------------------------------------------------------------------------------------
# diffusion element-wise ops
# ---------------------------------------------------------------------------------------------------------------
OBJECTIVES = ["v", "eps", "x0"]
BATCHES = [1, 8, 9, 33]
PERS = [4, 1000, 70004]   # 70004: grid-stride wrap at 2 SMs in every launch (and in mse_rows' fixed 64-CTA grid)


def _alpha_sigma(B, g):
    """Per-sample (alpha, sigma) on the unit circle; the first samples are (0, 1), (1, 0) and (1/sqrt 2, 1/sqrt 2)."""
    th = torch.rand(B, device=dev, generator=g, dtype=torch.float64) * (math.pi / 2 - 0.2) + 0.1
    a, s = th.cos(), th.sin()
    r = math.sqrt(0.5)
    for i, (ai, si) in enumerate(((0.0, 1.0), (1.0, 0.0), (r, r))[:B]):
        a[i], s[i] = ai, si
    return a.float().contiguous(), s.float().contiguous()


def _diff_inputs(B, per, seed):
    g = _gen(seed)
    x = torch.randn(B, per, device=dev, generator=g)
    y = torch.randn(B, per, device=dev, generator=g)
    a, s = _alpha_sigma(B, g)
    return g, x, y, a, s


@pytest.mark.parametrize("per", PERS)
@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("objective", OBJECTIVES)
def test_q_sample(sm2, objective, B, per):
    from naturalspeech2_pytorch_b200 import ops
    _, x0, noise, a, s = _diff_inputs(B, per, seed=B * 7 + per)
    bx, xt = _nan_buf((B, per))
    bt, target = _nan_buf((B, per))
    ops.q_sample(x0, noise, a, s, xt, target, objective=objective)
    assert_nan(bx[xt.numel():], "past x_t")
    assert_nan(bt[target.numel():], "past target")
    a64, s64, x64, e64 = a.double()[:, None], s.double()[:, None], x0.double(), noise.double()
    # one fma + one product: <= 2 half-ulps of |a x| + |s e|
    assert_close(xt, a64 * x64 + s64 * e64, U_F32 * ((a64 * x64).abs() + (s64 * e64).abs()), 2.0 ** -22, "x_t")
    if objective == "v":
        assert_close(target, a64 * e64 - s64 * x64, U_F32 * ((a64 * e64).abs() + (s64 * x64).abs()), 2.0 ** -22, "v")
    else:
        assert torch.equal(target, noise if objective == "eps" else x0), f"{objective} target is a copy"


def _x_start_ref(objective, x, p, a, s):
    """(x_start, bound) of ns2.py:1673-1680 in fp64 from the fp32 operands; eps divides by max(alpha, 1e-10)."""
    a64, s64, x64, p64 = a.double()[:, None], s.double()[:, None], x.double(), p.double()
    if objective == "v":
        return a64 * x64 - s64 * p64, U_F32 * ((a64 * x64).abs() + (s64 * p64).abs())
    if objective == "eps":
        a_safe = a64.clamp_min(TINY)
        ref = (x64 - s64 * p64) / a_safe
        return ref, U_F32 * (x64.abs() + (s64 * p64).abs()) / a_safe + U_F32 * ref.abs()
    return p64, torch.zeros_like(p64)


@pytest.mark.parametrize("per", PERS)
@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("objective", OBJECTIVES)
def test_x_start(sm2, objective, B, per):
    from naturalspeech2_pytorch_b200 import ops
    _, x, pred, a, s = _diff_inputs(B, per, seed=B * 11 + per)
    buf, out = _nan_buf((B, per))
    ops.x_start_from_pred(x, pred, a, s, out, objective=objective)
    assert_nan(buf[out.numel():], "past out")
    if objective == "x0":
        assert torch.equal(out, pred), "x0 objective: a copy"
        return
    ref, bound = _x_start_ref(objective, x, pred, a, s)
    assert_close(out, ref, bound, 2.0 ** -20, objective)


def _ddim_ref(objective, x, v, a, s, an, sn):
    """DDIM update (ns2.py:1412-1429) in fp64 with its bound propagated through the kernel's fp32 steps:
    x0 from the model output, eps = (x - a x0) / max(sigma, 1e-10), out = x0 an + eps sn."""
    x64 = x.double()
    a64, s64 = a.double()[:, None], s.double()[:, None]
    an64, sn64 = an.double()[:, None], sn.double()[:, None]
    x0, dx0 = _x_start_ref(objective, x, v, a, s)
    s_safe = s64.clamp_min(TINY)
    eps = (x64 - a64 * x0) / s_safe
    deps = (U_F32 * (x64.abs() + (a64 * x0).abs()) + a64 * dx0) / s_safe + U_F32 * eps.abs()
    out = x0 * an64 + eps * sn64
    dout = U_F32 * ((x0 * an64).abs() + (eps * sn64).abs()) + an64 * dx0 + sn64 * deps
    return out, dout


@pytest.mark.parametrize("per", PERS)
@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("objective", OBJECTIVES)
def test_ddim_step(sm2, objective, B, per):
    from naturalspeech2_pytorch_b200 import ops
    g, x, v, a, s = _diff_inputs(B, per, seed=B * 13 + per)
    an, sn = _alpha_sigma(B, g)
    an, sn = an.flip(0).contiguous(), sn.flip(0).contiguous()
    buf, xx = _nan_buf((B, per))
    xx.copy_(x)
    ops.ddim_step(xx, v, a, s, an, sn, objective=objective)
    assert_nan(buf[xx.numel():], "past x")
    ref, bound = _ddim_ref(objective, x, v, a, s, an, sn)
    for b in range(B):   # per sample: the sigma = 0 sample's bound (amplified by 1e10) must not mask the others' rel-L2
        assert_close(xx[b], ref[b], bound[b], 2.0 ** -16, f"{objective} B={B} per={per} sample {b}")
    _assert_ddim_safe_div_edges(objective, xx, x, v, an, sn)


def _assert_ddim_safe_div_edges(objective, got, x, v, an, sn):
    """Where safe_div's clamp is hit, the kernel's intermediates are known exactly in fp32, so the generic bound (scaled
    by 1e10) is replaced by an exact or one-rounding check.  Sample 0 has alpha = 0, sigma = 1; sample 1 (if any)
    alpha = 1, sigma = 0 (see `_alpha_sigma`)."""
    B = x.shape[0]
    an0, sn0 = an[:, None], sn[:, None]
    if B > 1 and objective in ("v", "eps"):
        # alpha = 1, sigma = 0: x_start is x itself, eps = (x - x) / 1e-10 = 0 exactly, so out = x * alpha_next
        assert torch.equal(got[1], x[1] * an0[1]), f"{objective}: sigma = 0 sample"
    if B > 1 and objective == "x0":
        # x_start = pred; eps = fp32(x - pred) / 1e-10, rounded once more; out = x0 an + eps sn (<= 2 more roundings)
        eps = (x[1] - v[1]).double() / TINY
        ref = v[1].double() * an0[1].double() + eps * sn0[1].double()
        bound = U_F32 * ((v[1].double() * an0[1].double()).abs() + 2 * (eps * sn0[1].double()).abs())
        assert_close(got[1], ref, bound, 2.0 ** -21, "x0: sigma = 0 sample")
    if objective == "eps":
        # alpha = 0: x_start = fp32(x - pred) / 1e-10, rounded once more; eps = x exactly; out = x0 an + x sn
        x0 = (x[0] - v[0]).double() / TINY
        ref = x0 * an0[0].double() + x[0].double() * sn0[0].double()
        bound = U_F32 * (2 * (x0 * an0[0].double()).abs() + (x[0].double() * sn0[0].double()).abs())
        assert_close(got[0], ref, bound, 2.0 ** -21, "eps: alpha = 0 sample")


def test_ddim_step_sensitivity(sm2):
    from naturalspeech2_pytorch_b200 import ops
    g, x, v, a, s = _diff_inputs(9, 1000, seed=17)
    a[1], s[1] = math.cos(0.7), math.sin(0.7)      # no sigma = 0 sample: its 1e10-amplified bound accepts anything
    an, sn = _alpha_sigma(9, g)
    an, sn = an.flip(0).contiguous(), sn.flip(0).contiguous()
    xx = x.clone()
    ops.ddim_step(xx, v, a, s, an, sn)
    _, bound = _ddim_ref("v", x, v, a, s, an, sn)
    wrong, _ = _ddim_ref("v", x, v, a, s, sn, an)
    assert_rejects(xx, wrong, bound, 2.0 ** -16, "alpha_next and sigma_next swapped")


@pytest.mark.parametrize("per", PERS)
@pytest.mark.parametrize("B", BATCHES)
def test_mse_rows(sm2, B, per):
    from naturalspeech2_pytorch_b200 import ops
    _, p, t, _, _ = _diff_inputs(B, per, seed=B * 17 + per)
    bo, out = _nan_buf((B,))
    bm, mean = _nan_buf((1,))
    ops.mse_rows(p, t, out, mean_out=mean)
    assert_nan(bo[B:], "past out")
    assert_nan(bm[1:], "past mean_out")
    d2 = (p.double() - t.double()) ** 2
    ref = d2.mean(1)
    # fp32 difference and square (<= 3 roundings), fp32 sum of per terms, the division
    bound = (acc_eps(per) + 2.0 ** -21) * ref + U_F32 * ref
    assert_close(out, ref, bound, 4 * acc_eps(per), "per-sample mse")
    mref = ref.mean()
    assert_close(mean, mref.reshape(1), bound.mean() + (acc_eps(B) + U_F32) * mref, 4 * acc_eps(per * B), "mean")
    out2, mean2 = torch.empty(B, device=dev), torch.empty(1, device=dev)
    ops.mse_rows(p, t, out2, mean_out=mean2)
    assert torch.equal(out, out2) and torch.equal(mean, mean2), "fixed grid, no float atomics: bit-identical"


@pytest.mark.parametrize("count", [4, 1000, 70004])
def test_cfg_combine(sm2, count):
    from naturalspeech2_pytorch_b200 import ops
    g = _gen(count)
    c, n = torch.randn(count, device=dev, generator=g), torch.randn(count, device=dev, generator=g)
    scale = 2.5
    ref = n.double() + (c.double() - n.double()) * scale
    bound = U_F32 * (ref.abs() + scale * (c.double() - n.double()).abs())
    buf, out = _nan_buf((count,))
    ops.cfg_combine(c, n, scale, out)
    assert_nan(buf[count:], "past out")
    assert_close(out, ref, bound, 2.0 ** -22, "out of place")
    ops.cfg_combine(c, n, scale, c)
    assert torch.equal(c, out), "in place into cond gives the same bits"


def test_flat_wrappers_reject_bad_tensors():
    """The element-wise diffusion kernels and rmsnorm_f32 read their tensors as flat float4 arrays: a strided view
    (also one whose last dimension is unit-stride, i.e. a row window of a wider buffer), a view that is not 16-byte
    aligned, a wrong dtype or a wrong element count is rejected on the host and nothing is launched."""
    from naturalspeech2_pytorch_b200 import ops
    B, N, D = 2, 8, 128
    g = _gen(0)
    x, y = torch.randn(B, N, D, device=dev, generator=g), torch.randn(B, N, D, device=dev, generator=g)
    a, s = torch.rand(B, device=dev, generator=g), torch.rand(B, device=dev, generator=g)
    bad = {
        "strided": torch.randn(B, D, N, device=dev, generator=g).transpose(1, 2),
        "row window": torch.randn(B, N, D + 4, device=dev, generator=g)[..., :D],     # stride(-1) == 1
        "misaligned": torch.randn(B * N * D + 4, device=dev, generator=g)[1:1 + B * N * D].view(B, N, D),
        "float64": y.double(),
        "bfloat16": y.to(bf),
        "numel": y[:, :N - 1].contiguous(),
    }
    bad_scalar = {"strided": torch.rand(2 * B, device=dev, generator=g)[::2],
                  "row window": torch.rand(B, 2, device=dev, generator=g)[:, :1],        # (B, 1), stride (2, 1)
                  "float64": a.double(),
                  "numel": torch.rand(B + 1, device=dev, generator=g)}
    e = torch.empty_like
    calls = {
        "q_sample": lambda t: ops.q_sample(x, t, a, s, e(x), e(x)),
        "q_sample alpha": lambda t: ops.q_sample(x, y, t, s, e(x), e(x)),
        "ddim_step x": lambda t: ops.ddim_step(t, y, a, s, a, s),
        "ddim_step v": lambda t: ops.ddim_step(x.clone(), t, a, s, a, s),
        "ddim_step sigma_next": lambda t: ops.ddim_step(x.clone(), y, a, s, a, t),
        "x_start_from_pred": lambda t: ops.x_start_from_pred(x, t, a, s, e(x)),
        "x_start_from_pred sigma": lambda t: ops.x_start_from_pred(x, y, a, t, e(x)),
        "cfg_combine": lambda t: ops.cfg_combine(x, t, 2.0, e(x)),
        "cfg_combine out": lambda t: ops.cfg_combine(x, y, 2.0, t),
        "mse_bwd": lambda t: ops.mse_bwd(x, t, a, out_f32=e(x)),
        "mse_bwd out": lambda t: ops.mse_bwd(x, y, a, out_f32=t),
        "mse_bwd coef": lambda t: ops.mse_bwd(x, y, t, out_f32=e(x)),
        "rmsnorm_f32 x": lambda t: ops.rmsnorm_f32(t, e(x), None),
        "rmsnorm_f32 out": lambda t: ops.rmsnorm_f32(x, t, None),
    }
    before = ops.launch_count()
    ops.cfg_combine(x, y, 2.0, e(x))
    torch.cuda.synchronize()
    assert ops.launch_count() == before + 1, "launch_count counts a valid call"
    assert bad["row window"].stride(-1) == 1 and not bad["row window"].is_contiguous()
    assert bad["misaligned"].is_contiguous() and bad["misaligned"].data_ptr() % 16
    for name, call in calls.items():
        for kind, t in (bad_scalar if name.split()[-1] in ("alpha", "sigma", "sigma_next", "coef") else bad).items():
            before = ops.launch_count()
            with pytest.raises(ValueError):
                call(t)
            assert ops.launch_count() == before, f"{name} with a {kind} tensor launched a kernel"


# ---------------------------------------------------------------------------------------------------------------
# groupnorm_silu
# ---------------------------------------------------------------------------------------------------------------
def _gn_ref(x, w, b, groups, eps, resid, one_pass=False):
    """(reference, bound).  Bound from the kernel's arithmetic: the group mean is an fp32 sum (a serial run of
    ceil(n/256) terms per thread, then two 8-level trees: <= (ceil(n/256) + 9) roundings of sum |x|); the centred
    variance is insensitive to that mean error to first order; __expf in SiLU: 2 + 1.173 |y| ulp (CUDA Math API,
    intrinsic functions table).  `one_pass`: the variance as E[x^2] - E[x]^2 in torch fp32."""
    B, N, C = x.shape
    cpg = C // groups
    n = N * cpg
    xg = x.view(B, N, groups, cpg).double()
    m = xg.mean(dim=(1, 3), keepdim=True)
    var = ((xg - m) ** 2).mean(dim=(1, 3), keepdim=True)
    if one_pass:
        xf = x.view(B, N, groups, cpg)
        m32 = xf.mean(dim=(1, 3), keepdim=True)
        var = ((xf * xf).mean(dim=(1, 3), keepdim=True) - m32 * m32).clamp_min(0).double()
    rstd = (var + eps).rsqrt()
    w64, b64 = w.double().view(groups, cpg), b.double().view(groups, cpg)
    y = (xg - m) * rstd * w64 + b64
    ref = _silu64(y)
    red = math.ceil(n / 256) + 9
    dm = red * 2.0 ** -24 * xg.abs().mean(dim=(1, 3), keepdim=True)
    ev = (red + 3) * 2.0 ** -23
    dy = w64.abs() * rstd * (dm + (xg - m).abs() * (ev / 2 + 2.0 ** -22)) + 2.0 ** -23 * (y.abs() + b64.abs())
    bound = 1.1 * dy + (4 + 1.2 * y.abs()) * 2.0 ** -23 * ref.abs()
    if resid is not None:
        ref = ref + resid.double().view(B, N, groups, cpg)
    # rel-L2 from the groups with spread: a constant group's worst-case mean error is amplified by 1/sqrt(eps), so its
    # element-wise bound (checked all the same) would dominate the norm
    spread = (var > 0).expand_as(ref)
    rel = float(bound[spread].norm() / ref[spread].norm())
    return ref.reshape(B, N, C), bound.reshape(B, N, C), rel


def _gn_case(B, N, C, groups, with_resid, seed, constant_group=True):
    from naturalspeech2_pytorch_b200 import ops
    g = _gen(seed)
    x = 1000 + torch.randn(B, N, C, device=dev, generator=g)
    if constant_group:
        x[0, :, :C // groups] = 1000.0                 # group 0 of sample 0 is constant: zero variance
    w = torch.randn(C, device=dev, generator=g)
    b = torch.randn(C, device=dev, generator=g)
    resid = torch.randn(B, N, C, device=dev, generator=g) if with_resid else None
    bf32, o32 = _nan_buf((B, N, C))
    bb16, o16 = _nan_buf((B, N, C), bf)
    ops.groupnorm_silu(x, w, b, groups, resid=resid, out_f32=o32, out_bf16=o16)
    assert_nan(bf32[o32.numel():], "past out_f32")
    assert_nan(bb16[o16.numel():], "past out_bf16")
    return x, w, b, resid, o32, o16


@pytest.mark.parametrize("B,N,C,groups,with_resid", [
    (2, 200, 32, 8, False),     # 4 channels per group: one float4 per row
    (2, 77, 128, 4, True),
    (1, 300, 512, 8, True),
])
def test_groupnorm_silu(B, N, C, groups, with_resid):
    x, w, b, resid, o32, o16 = _gn_case(B, N, C, groups, with_resid, seed=N + C)
    ref, bound, rel = _gn_ref(x, w, b, groups, 1e-5, resid)
    assert_close(o32, ref, bound + U_F32 * ref.abs(), rel, "f32")
    assert_close(o16, ref, bound + U_BF16 * ref.abs(), rel + U_BF16, "bf16")


def test_groupnorm_silu_two_pass_variance():
    """With a mean of 1000 the one-pass variance E[x^2] - E[x]^2 in fp32 is off by O(0.1): the bound accepts the
    kernel's centred variance and rejects the one-pass formula."""
    x, w, b, _, o32, _ = _gn_case(2, 200, 32, 8, False, seed=5, constant_group=False)
    ref, bound, rel = _gn_ref(x, w, b, 8, 1e-5, None)
    wrong, _, _ = _gn_ref(x, w, b, 8, 1e-5, None, one_pass=True)
    assert_rejects(o32, wrong, bound + U_F32 * ref.abs(), rel, "one-pass fp32 variance")


# ---------------------------------------------------------------------------------------------------------------
# rowdot, mean_rows
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows", [1, 13, 1001])
@pytest.mark.parametrize("dim", [4, 132, 1000])
def test_rowdot(rows, dim):
    from naturalspeech2_pytorch_b200 import ops
    g = _gen(rows + dim)
    x = torch.randn(rows, dim, device=dev, generator=g)
    w = torch.randn(dim, device=dev, generator=g)
    bias = torch.randn(1, device=dev, generator=g)
    for relu, bb in ((True, bias), (False, bias), (False, None), (True, None)):
        buf, out = _nan_buf((rows,))
        ops.rowdot(x, w, bb, out, relu=relu)
        assert_nan(buf[rows:], "past out")
        z = x.double() @ w.double() + (0 if bb is None else bb.double())
        ref = z.clamp_min(0) if relu else z
        bound = acc_eps(dim) * (x.double().abs() @ w.double().abs()) + U_F32 * (z.abs() + (0 if bb is None else bb.double().abs()))
        assert_close(out, ref, bound, 4 * acc_eps(dim), f"rows={rows} dim={dim} relu={relu} bias={bb is not None}")


def test_rowdot_sensitivity():
    from naturalspeech2_pytorch_b200 import ops
    g = _gen(21)
    x, w = torch.randn(13, 132, device=dev, generator=g), torch.randn(132, device=dev, generator=g)
    out = ops.rowdot(x, w, None, torch.empty(13, device=dev))
    bound = acc_eps(132) * (x.double().abs() @ w.double().abs()) + U_F32 * (x.double() @ w.double()).abs()
    wrong = x.double()[:, :128] @ w.double()[:128]
    assert_rejects(out, wrong, bound, 4 * acc_eps(132), "dim tail past the last full 128 left out")


@pytest.mark.parametrize("B,N,D", [(1, 1, 5), (3, 77, 300), (2, 1000, 64)])
def test_mean_rows(B, N, D):
    from naturalspeech2_pytorch_b200 import ops
    x = torch.randn(B, N, D, device=dev, generator=_gen(N + D)) + 0.5
    buf, out = _nan_buf((B, D))
    ops.mean_rows(x, out)
    assert_nan(buf[B * D:], "past out")
    ref = x.double().mean(1)
    # a serial fp32 sum of N terms: <= N roundings of sum |x|, then the division
    assert_close(out, ref, N * 2.0 ** -24 * x.double().abs().mean(1) + U_F32 * ref.abs(), N * 2.0 ** -22, "mean_rows")


# ---------------------------------------------------------------------------------------------------------------
# copies, casts and single fp32 adds: bit-exact
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("count", [4, 1000, 70004])
def test_cast_bf16_exact(sm2, count):
    from naturalspeech2_pytorch_b200 import ops
    g = _gen(count)
    x, add = torch.randn(count, device=dev, generator=g) * 100, torch.randn(count, device=dev, generator=g)
    for a in (None, add):
        buf, out = _nan_buf((count,), bf)
        ops.cast_bf16(x, out, add=a)
        assert_nan(buf[count:], "past out")
        assert torch.equal(out, (x if a is None else x + a).to(bf)), f"count={count} add={a is not None}"


@pytest.mark.parametrize("L", [20, 50, 70])   # zero-padded, equal, curtailed
@pytest.mark.parametrize("D", [4, 132])
def test_cond_inject_exact(L, D):
    from naturalspeech2_pytorch_b200 import ops
    B, N = 3, 50
    g = _gen(L + D)
    x = torch.randn(B, N, D, device=dev, generator=g)
    cproj = torch.randn(B, L, D, device=dev, generator=g)
    null = torch.randn(D, device=dev, generator=g)
    drop = torch.tensor([True, False, True], device=dev)
    for mask in (None, drop):
        c = torch.zeros(B, N, D, device=dev)
        m = min(L, N)
        c[:, :m] = cproj[:, :m]
        if mask is not None:
            c[mask, :m] = null
        buf, out = _nan_buf((B, N, D), bf)
        ops.cond_inject(x, cproj, out, drop_mask=mask, null_cond=None if mask is None else null)
        assert_nan(buf[out.numel():], "past out")
        assert torch.equal(out, (x + c).to(bf)), f"L={L} D={D} mask={mask is not None}"


@pytest.mark.parametrize("row_len", [3, 1000, 20000])
def test_select_rows_exact(row_len):
    from naturalspeech2_pytorch_b200 import ops
    B = 4
    g = _gen(row_len)
    src = torch.randn(B, row_len, device=dev, generator=g)
    null = torch.randn(row_len, device=dev, generator=g)
    drop = torch.tensor([False, True, True, False], device=dev)
    ref = torch.where(drop[:, None], null[None], src)
    for dt in (torch.float32, bf):
        wide = torch.full((B, row_len + 9), NAN, device=dev, dtype=dt)
        out = wide[:, 5:5 + row_len]                     # a column window of a wider matrix
        ops.select_rows(drop, null, src, out)
        assert_nan(wide[:, :5], "left of out")
        assert_nan(wide[:, 5 + row_len:], "right of out")
        assert torch.equal(out, ref.to(dt)), f"row_len={row_len} {dt}"


@pytest.mark.parametrize("B,C,L", [(1, 1, 1), (2, 33, 65), (3, 80, 333)])
def test_transpose_cast_exact(B, C, L):
    from naturalspeech2_pytorch_b200 import ops
    x = torch.randn(B, C, L, device=dev, generator=_gen(C + L))
    buf, out = _nan_buf((B, L, C), bf)
    ops.transpose_cast(x, out)
    assert_nan(buf[out.numel():], "past out")
    assert torch.equal(out, x.transpose(1, 2).to(bf))


@pytest.mark.parametrize("dim", [4, 132])
def test_embedding_bf16_exact(dim):
    from naturalspeech2_pytorch_b200 import ops
    rows, pad = 11, 3
    g = _gen(dim)
    table = torch.randn(rows, dim, device=dev, generator=g)
    ids = torch.randint(-2, rows + 3, (5, 37), device=dev, generator=g)
    ids[0, :4] = torch.tensor([-1, rows - 1, rows, 10 ** 6], device=dev)   # ids >= num_rows are clamped to the last row
    buf, out = _nan_buf((5, 37, dim), bf)
    ops.embedding_bf16(ids, table, out, pad)
    assert_nan(buf[out.numel():], "past out")
    idx = ids.masked_fill(ids < 0, pad).clamp_max(rows - 1)
    assert torch.equal(out, table[idx].to(bf))


@pytest.mark.parametrize("B,T,D,L", [(2, 7, 45, 70), (1, 40, 128, 33), (3, 5, 1, 1)])
def test_expand_encodings_exact(B, T, D, L):
    from naturalspeech2_pytorch_b200 import ops
    rows = 9
    g = _gen(T + D + L)
    phon = torch.randn(B, T, D, device=dev, generator=g)
    table = torch.randn(rows, D, device=dev, generator=g)
    coarse = torch.randint(-3, rows + 3, (B, T), device=dev, generator=g).int()   # out-of-range bins clamp
    idx = torch.randint(-2, T + 2, (B, L), device=dev, generator=g).int()         # < 0 and >= T give 0
    out = ops.expand_encodings(phon, coarse, table, idx)
    valid = (idx >= 0) & (idx < T)
    m = idx.long().clamp(0, T - 1)
    c = torch.gather(coarse.long().clamp(0, rows - 1), 1, m)
    val = torch.gather(phon, 1, m[..., None].expand(-1, -1, D)) + table[c]
    ref = torch.where(valid[..., None], val, torch.zeros_like(val)).transpose(1, 2)
    assert torch.equal(out, ref)
