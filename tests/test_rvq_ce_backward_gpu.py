"""GPU: `ops.rvq_ce_bwd` (d loss / d frames of the RVQ cross-entropy head, ns2.py:1682) at its edges, against float64
torch autograd of rvq_ce_restatement.residual_vq_ce on the same fp32 inputs and the same residual chain.

Bound (the kernel_check protocol): our error against the fp64 reference may be at most ERR_MULT times the error of the
same torch formula run in fp32, element-wise max-abs and relative L2, plus an absolute floor of 2^-16 max|ref|.  A
reference that drops the target term, or one that never advances the residual chain, must fail both bounds."""
import pytest
import torch

from kernel_check import assert_close, assert_nan, assert_rejects
from rvq_ce_restatement import residual_vq_ce

pytestmark = pytest.mark.gpu

ERR_MULT = 8.0


def _problem(F, Q, K, seed, *, frame_scale=1.0, degenerate=False):
    g = torch.Generator().manual_seed(seed)
    cb = torch.randn(Q, K, 128, generator=g)
    if degenerate:   # every codeword within 1e-3 of one point: a nearly flat softmax
        cb = cb[:, :1] + 1e-3 * torch.randn(Q, K, 128, generator=g)
    x = torch.randn(F, 128, generator=g) * frame_scale
    return x, cb, g


def _own_codes(x, cb):
    with torch.no_grad():
        return residual_vq_ce(x.double().cuda(), cb.double().cuda(), torch.zeros(x.shape[0], cb.shape[0]))[2]


def _targets(own, K, g, *, scatter_ignored=True):
    """Half the targets equal the own code, half are random; some -1 scattered over every stage."""
    F, Q = own.shape
    tgt = torch.randint(0, K, (F, Q), generator=g).cuda()
    same = torch.rand(F, Q, generator=g).cuda() < 0.5
    tgt = torch.where(same, own, tgt)
    if scatter_ignored:
        tgt[torch.rand(F, Q, generator=g).cuda() < 0.1] = -1
    return tgt


def _ref_grad(x, cb, own, tgt, d_loss, row_scale, rps, dtype, *, drop_target=False, advance=True):
    """d loss / d x of residual_vq_ce in `dtype` (the fp32 / fp64 references), or a deliberately wrong variant."""
    import torch.nn.functional as Fn
    xx = x.cuda().to(dtype).requires_grad_(True)
    cbd = cb.cuda().to(dtype)
    if not drop_target and advance:
        _, loss, _ = residual_vq_ce(xx, cbd, tgt, own=own)
    else:
        loss, r = 0., xx
        for q in range(cb.shape[0]):
            d2 = ((r * r).sum(-1, keepdim=True) - 2 * r @ cbd[q].t() + (cbd[q] * cbd[q]).sum(-1)[None]).clamp_min(0)
            lg = -d2.clamp_min(1e-300 if dtype == torch.float64 else 1e-30).sqrt()
            valid = tgt[:, q] >= 0
            if drop_target:   # logsumexp only: the target term u_t missing
                loss = loss + lg.logsumexp(-1)[valid].sum() / valid.sum()
            else:
                loss = loss + Fn.cross_entropy(lg, tgt[:, q], ignore_index=-1)
            if advance:
                r = r - cbd[q][own[:, q]]
    (g,) = torch.autograd.grad(loss, xx, grad_outputs=d_loss.to(dtype).reshape(()))
    g = torch.nan_to_num(g, nan=0.0)
    if row_scale is not None:
        g = g * row_scale.to(dtype).repeat_interleave(rps)[: x.shape[0], None]
    return g.double()


def _run(x, cb, own, tgt, d_loss, row_scale=None, rps=1, out=None):
    from naturalspeech2_pytorch_b200 import ops
    cbc = cb.cuda().contiguous()
    cn2 = (cbc * cbc).sum(-1)   # same values as rvq_prepare's norms (fp32 sum of squares)
    return ops.rvq_ce_bwd(x.cuda(), cbc, cn2.contiguous(), own, tgt, d_loss, row_scale=row_scale, rows_per_sample=rps,
                          out=out)


def _check(got, x, cb, own, tgt, d_loss, row_scale=None, rps=1, what=""):
    r64 = _ref_grad(x, cb, own, tgt, d_loss, row_scale, rps, torch.float64)
    r32 = _ref_grad(x, cb, own, tgt, d_loss, row_scale, rps, torch.float32)
    floor = 2.0 ** -16 * float(r64.abs().max())
    bound = ERR_MULT * float((r32 - r64).abs().max()) + floor
    rel32 = float((r32 - r64).norm() / r64.norm().clamp_min(1e-300))
    assert_close(got, r64, bound, ERR_MULT * rel32 + 1e-6, what)
    return r64, bound, ERR_MULT * rel32 + 1e-6


@pytest.mark.parametrize("K", [32, 100, 128, 1000, 1024])
@pytest.mark.parametrize("Q", [1, 3, 8])
@pytest.mark.parametrize("F", [1, 31, 33, 4097])
def test_rvq_ce_bwd_shapes(F, Q, K):
    x, cb, g = _problem(F, Q, K, seed=F * 131 + Q * 17 + K)
    own = _own_codes(x, cb)
    tgt = _targets(own, K, g)
    d_loss = torch.tensor([0.75], device="cuda")
    got = _run(x, cb, own, tgt, d_loss)
    _check(got, x, cb, own, tgt, d_loss, what=f"F={F} Q={Q} K={K}")


def test_rvq_ce_bwd_ignored_stage_codeword_frames_and_saturation():
    """One stage with every target -1 (NaN loss, zero gradient from it), frames exactly on a codeword (finite, the
    cdist convention) and large-norm frames whose softmax is one-hot."""
    F, Q, K = 200, 3, 256
    x, cb, g = _problem(F, Q, K, seed=5)
    x[:10] = cb[0, 7:17]                         # on a codeword at stage 0
    x[10:20] *= 300.0                            # saturated softmax
    own = _own_codes(x, cb)
    tgt = _targets(own, K, g)
    tgt[:, 1] = -1                               # an all-ignored stage
    tgt[:5, 0] = own[:5, 0]                      # on-codeword frames whose target is that codeword
    d_loss = torch.tensor([1.0], device="cuda")
    got = _run(x, cb, own, tgt, d_loss)
    assert bool(torch.isfinite(got).all())
    _check(got, x, cb, own, tgt, d_loss, what="edges")
    # the check above holds because the ignored stage adds nothing (torch's gradient of that stage is all-zero); with
    # valid targets the same stage does contribute, so the kernel did not simply skip stage 1
    tgt2 = tgt.clone()
    tgt2[:, 1] = own[:, 1]
    with_stage = _run(x, cb, own, tgt2, d_loss)
    assert float((with_stage - got).abs().max()) > 1e-6, "stage 1 has gradient when its targets are valid"


def test_rvq_ce_bwd_degenerate_codebook():
    """Codewords within 1e-3 of each other: a nearly flat softmax, u_t - sum p u is a small difference."""
    x, cb, g = _problem(300, 2, 128, seed=6, degenerate=True)
    own = _own_codes(x, cb)
    tgt = _targets(own, 128, g)
    d_loss = torch.tensor([2.0], device="cuda")
    _check(_run(x, cb, own, tgt, d_loss), x, cb, own, tgt, d_loss, what="degenerate")


def test_rvq_ce_bwd_row_scale_guards_and_determinism():
    """Per-sample row scales (including 0 and negative ones), NaN guard rows and columns of a wider output buffer, and
    bit-identical results across two launches."""
    B, n, Q, K = 5, 70, 4, 1024
    F = B * n
    x, cb, g = _problem(F, Q, K, seed=7)
    own = _own_codes(x, cb)
    tgt = _targets(own, K, g)
    d_loss = torch.tensor([0.5], device="cuda")
    row_scale = torch.tensor([1.0, 0.0, -0.7, 3.5, -1e-3], device="cuda")
    buf = torch.full((F + 3, 136), float("nan"), device="cuda")
    got = _run(x, cb, own, tgt, d_loss, row_scale, n, out=buf[:F])
    assert_nan(buf[:F, 128:], "guard columns")
    assert_nan(buf[F:], "guard rows")
    assert torch.count_nonzero(got[n:2 * n, :128]) == 0, "row scale 0 gives exact zeros"
    _check(got[:, :128], x, cb, own, tgt, d_loss, row_scale, n, what="row scale")
    again = _run(x, cb, own, tgt, d_loss, row_scale, n)
    assert torch.equal(again, got[:, :128]), "two launches differ (the backward has no atomics)"


def test_rvq_ce_bwd_bounds_reject_wrong_references():
    """Sensitivity: the bounds above reject a reference without the target term and one whose residual chain is never
    advanced."""
    x, cb, g = _problem(257, 3, 256, seed=8)
    own = _own_codes(x, cb)
    tgt = _targets(own, 256, g)
    d_loss = torch.tensor([1.0], device="cuda")
    got = _run(x, cb, own, tgt, d_loss)
    _, bound, rel = _check(got, x, cb, own, tgt, d_loss, what="sensitivity baseline")
    for kw in (dict(drop_target=True), dict(advance=False)):
        wrong = _ref_grad(x, cb, own, tgt, d_loss, None, 1, torch.float64, **kw)
        assert_rejects(got, wrong, bound, rel, str(kw))


def test_rq_autograd_and_loss_bit_identity():
    """`EncodecRVQ.rq` is differentiable in x: its gradient is ops.rvq_ce_bwd's, its loss is bit-identical to the
    no-grad call, and quantized is a constant."""
    from naturalspeech2_pytorch_b200 import EncodecRVQ
    g = torch.Generator().manual_seed(21)
    Q, K = 4, 256
    cb = torch.randn(Q, K, 128, generator=g)
    x = torch.randn(3, 50, 128, generator=g).cuda()
    codes = torch.randint(0, K, (3, 50, Q), generator=g).cuda()
    codes[0, :5, 1] = -1
    codec = EncodecRVQ(cb).cuda()
    with torch.no_grad():
        q0, l0 = codec.rq(x, codes)
    xr = x.clone().requires_grad_(True)
    q1, l1 = codec.rq(xr, codes)
    assert l1.requires_grad and not q1.requires_grad
    assert torch.equal(l0, l1.detach()) and torch.equal(q0, q1)
    (2.5 * l1).backward()
    own, _ = codec.quantize(x.reshape(-1, 128))   # the codes rq follows
    tgt = codes.reshape(-1, Q)
    d_loss = torch.tensor([2.5], device="cuda")
    _check(xr.grad.reshape(-1, 128), x.cpu().reshape(-1, 128), cb, own, tgt, d_loss, what="rq autograd")
