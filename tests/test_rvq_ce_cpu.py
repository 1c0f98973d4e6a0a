"""CPU: the pieces of the RVQ cross-entropy gradient that need no GPU — the fp64 restatement of ResidualVQ-with-indices
(tests/rvq_ce_restatement.py) against the torch.cdist formula, the per-objective d x_start / d pred coefficient
against autograd of ns2.py:1673-1680, and the host-side argument checks of ns2_rvq_ce_bwd."""
import pytest
import torch
import torch.nn.functional as F

from rvq_ce_restatement import residual_vq_ce


def _cdist_loss(x, cb, codes, own):
    """The formula the reference's codec evaluates: -torch.cdist logits, cross_entropy (ignore_index -1), summed over
    stages, residual chain through `own`."""
    r, total = x, 0.
    for q in range(cb.shape[0]):
        total = total + F.cross_entropy(-torch.cdist(r, cb[q]), codes[:, q], ignore_index=-1)
        r = r - cb[q][own[:, q]]
    return total


def test_restatement_matches_cdist_formula_in_fp64():
    g = torch.Generator().manual_seed(3)
    Q, K, Fr = 3, 64, 90
    cb = torch.randn(Q, K, 128, generator=g, dtype=torch.float64)
    x = torch.randn(Fr, 128, generator=g, dtype=torch.float64)
    x[:4] = cb[0, :4]                                    # frames on a codeword: zero distance
    codes = torch.randint(0, K, (Fr, Q), generator=g)
    codes[::6, 1] = -1
    xa = x.clone().requires_grad_(True)
    quantized, loss, own = residual_vq_ce(xa, cb, codes)
    (ga,) = torch.autograd.grad(loss, xa)
    # own codes: the exact nearest codewords of the fp64 chain; quantized: their sum
    r, qsum = x.clone(), torch.zeros_like(x)
    for q in range(Q):
        d = torch.cdist(r, cb[q])
        assert torch.equal(own[:, q], d.argmin(-1)), q
        qsum, r = qsum + cb[q][own[:, q]], r - cb[q][own[:, q]]
    assert torch.allclose(quantized, qsum, rtol=0, atol=1e-12)
    xb = x.clone().requires_grad_(True)
    ref = _cdist_loss(xb, cb, codes, own)
    (gb,) = torch.autograd.grad(ref, xb)
    assert abs(loss.item() - ref.item()) < 1e-10 * abs(ref.item())
    assert bool(torch.isfinite(ga).all())
    assert float((ga - gb).abs().max()) < 1e-7 * float(gb.abs().max()), float((ga - gb).abs().max())


def test_restatement_all_ignored_stage_is_nan_with_zero_gradient():
    g = torch.Generator().manual_seed(4)
    cb = torch.randn(2, 32, 128, generator=g, dtype=torch.float64)
    x = torch.randn(10, 128, generator=g, dtype=torch.float64, requires_grad=True)
    codes = torch.randint(0, 32, (10, 2), generator=g)
    codes[:, 1] = -1
    _, loss, own = residual_vq_ce(x, cb, codes)
    assert torch.isnan(loss)
    (g_all,) = torch.autograd.grad(loss, x)
    xs = x.detach().clone().requires_grad_(True)
    _, loss0, _ = residual_vq_ce(xs, cb[:1], codes[:, :1])
    (g0,) = torch.autograd.grad(loss0, xs)
    assert torch.equal(torch.nan_to_num(g_all), g0)


@pytest.mark.parametrize("objective", ["v", "eps", "x0"])
def test_x_start_coefficient_matches_autograd(objective):
    """x_start_pred_coef is d x_start / d pred of ns2.py:1673-1680 per sample, including safe_div's clamp of alpha."""
    from naturalspeech2_pytorch_b200.diffusion import x_start_pred_coef
    B = 4
    alpha = torch.tensor([0.9, 0.3, 1e-12, 0.0], dtype=torch.float64)   # the last two hit the 1e-10 clamp
    sigma = torch.tensor([0.4, 0.95, 1.0, 1.0], dtype=torch.float64)
    audio = torch.randn(B, 5, 128, dtype=torch.float64)
    pred = torch.randn(B, 5, 128, dtype=torch.float64, requires_grad=True)
    a3, s3 = alpha.view(-1, 1, 1), sigma.view(-1, 1, 1)
    if objective == "x0":
        x_start = pred
    elif objective == "eps":
        x_start = (audio - s3 * pred) / a3.clamp(min=1e-10)     # safe_div, ns2.py:1122-1123
    else:
        x_start = a3 * audio - s3 * pred
    up = torch.randn_like(audio)
    (grad,) = torch.autograd.grad(x_start, pred, up)
    coef = x_start_pred_coef(alpha, sigma, objective)
    got = up if coef is None else up * coef.view(-1, 1, 1)
    assert torch.allclose(got, grad, rtol=1e-15, atol=0)


def test_rvq_ce_bwd_rejects_bad_arguments_before_launch():
    """Host-side checks: a clean error and no kernel launch (dummy non-NULL device pointers are never dereferenced)."""
    from naturalspeech2_pytorch_b200 import _lib, build, ops
    build.build()
    lib = _lib.load()
    before = lib.ns2_launch_count()
    p = 16
    assert lib.ns2_rvq_ce_bwd(p, 4, 64, p, p, 1, 256, p, p, p, None, 1, p, p, 128, None) < 0          # d != 128
    assert lib.ns2_rvq_ce_bwd(p, 4, 128, p, p, 1, 256, p, p, p, None, 1, p, p, 130, None) < 0         # out_stride % 4
    assert b"out_stride" in lib.ns2_last_error()
    assert lib.ns2_rvq_ce_bwd(p, 4, 128, p, p, 1, 256, p, p, None, None, 1, p, p, 128, None) < 0      # no d_loss
    assert lib.ns2_rvq_ce_bwd(p, 4, 128, p, p, 1, 256, p, p, p, p, 0, p, p, 128, None) < 0            # rows_per_sample
    assert lib.ns2_launch_count() == before
    with pytest.raises(ValueError):
        ops.rvq_ce_bwd(torch.zeros(4, 128), torch.zeros(1, 32, 128), torch.zeros(1, 32), torch.zeros(4, 1).long(),
                       torch.zeros(4, 1).long(), torch.ones(1))
