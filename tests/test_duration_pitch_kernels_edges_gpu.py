"""GPU: the duration / pitch predictor's backward kernels at their edges, against float64 from the same operands
(tests/kernel_check.py: an element-wise max-abs bound and a rel-L2 bound, and a wrong reference both must reject).

  groupnorm_silu_bwd   channels per group 4 / 64, groups 1 / 8 / 32, rows 1 / 3 / 100 / 1000, batch up to 70; a
                       constant group (rstd = 1/sqrt(eps)), a mean of 1000, saturated SiLU; d weight / d bias
                       bit-identical across launches; rejects a reference without the x_hat * mean(dx_hat * x_hat) term
  rowdot_bwd           rows 1 ... 4097 (around the 32-row chunks), dim 4 ... 2048; exact-zero predictions take no
                       gradient; accumulation into a non-zero d x; bit-identical d w / d b across launches; rejects a
                       reference that ignores the ReLU gate
"""
import pytest
import torch

from kernel_check import U_BF16, U_F32, acc_eps, assert_close, assert_rejects, gen
from naturalspeech2_pytorch_b200 import ops

pytestmark = pytest.mark.gpu
EPS = 1e-5


# ---------------------------------------------------------------------------------------------------------------------
# groupnorm_silu_bwd
# ---------------------------------------------------------------------------------------------------------------------
def _gn_reference(x, w, b, groups, dy, drop_m2=False):
    """float64 backward of silu(GroupNorm(x) * w + b) -> (dx, dw, db, bound terms)."""
    B, N, C = x.shape
    cpg = C // groups
    xg = x.double().view(B, N, groups, cpg)
    mean = xg.mean(dim=(1, 3), keepdim=True)
    var = ((xg - mean) ** 2).mean(dim=(1, 3), keepdim=True)
    rstd = (var + EPS).rsqrt()
    xh = (xg - mean) * rstd
    wg, bg = w.double().view(groups, cpg), b.double().view(groups, cpg)
    z = xh * wg + bg
    s = torch.sigmoid(z)
    dz = dy.double().view(B, N, groups, cpg) * s * (1 + z * (1 - s))
    dxh = dz * wg
    m1 = dxh.mean(dim=(1, 3), keepdim=True)
    m2 = (dxh * xh).mean(dim=(1, 3), keepdim=True)
    dx = rstd * (dxh - m1 - (0.0 if drop_m2 else xh * m2))
    n = N * cpg
    # bf16 rounding of dx; fp32 rounding of dz (__expf) and of the group sums / statistics, scaled by rstd; the fp32
    # mean is off by ~2^-24 sqrt(n) |mean|, which shifts x_hat by that times rstd (the mean-1000 case)
    shift = 4 * 2.0 ** -24 * n ** 0.5 * mean.abs() * rstd
    bound_dx = (U_BF16 * dx.abs() + acc_eps(n) * dx.abs()
                + rstd * shift * (wg ** 2 * dy.double().view(B, N, groups, cpg).abs() + m2.abs())
                + rstd * (1e-5 * (dxh.abs() + (xh * m2).abs())
                          + acc_eps(n) * (dxh.abs().mean(dim=(1, 3), keepdim=True)
                                          + xh.abs() * (dxh * xh).abs().mean(dim=(1, 3), keepdim=True))))
    dw = (dz * xh).sum(dim=(0, 1)).reshape(C)
    db = dz.sum(dim=(0, 1)).reshape(C)
    sum_dz = dz.abs().sum(dim=(0, 1)).reshape(C)
    bound_dw = (1e-5 * dw.abs() + acc_eps(B * N) * (dz * xh).abs().sum(dim=(0, 1)).reshape(C)
                + 2 * (shift * dz.abs()).sum(dim=(0, 1)).reshape(C) + 1e-30)
    bound_db = 1e-5 * db.abs() + acc_eps(B * N) * sum_dz + 1e-30
    return dx.view(B, N, C), dw, db, bound_dx.view(B, N, C), bound_dw, bound_db


def _gn_case(B, N, C, groups, seed, *, mean=0.0, constant_group=False, saturate=False, correlated=False):
    g = gen(seed)
    x = torch.randn(B, N, C, device="cuda", generator=g) * 1.5 + mean
    if constant_group:
        x.view(B, N, groups, C // groups)[:, :, 0] = 0.75          # group 0 of every sample: zero variance
    w = torch.randn(C, device="cuda", generator=g)
    b = torch.randn(C, device="cuda", generator=g) * 0.5
    if saturate:
        w *= 20.0                                                    # |z| up to ~60: sigmoid at 0 and 1
    dy = torch.randn(B, N, C, device="cuda", generator=g)
    if correlated:                                                   # makes mean(dx_hat * x_hat) large
        dy += 2.0 * (x - x.mean()) / x.std()
    dx = torch.full((B, N, C), float("nan"), device="cuda", dtype=torch.bfloat16)
    dw, db = ops.groupnorm_silu_bwd(x, w, b, groups, dy, dx, eps=EPS)
    return (x, w, b, dy), (dx, dw, db)


GN_SHAPES = [
    # (B, N, C, groups): cpg = C / groups
    (1, 1, 4, 1),        # cpg 4, one element per row
    (2, 3, 32, 8),       # cpg 4
    (70, 3, 128, 32),    # cpg 4, batch 70
    (3, 100, 512, 8),    # the predictor's Block: cpg 64
    (2, 1000, 512, 8),   # cpg 64, 1000 rows
    (1, 1000, 64, 1),    # one group of 64 channels
    (4, 100, 2048, 32),  # cpg 64, 32 groups
    (70, 100, 512, 8),   # batch 70
]


@pytest.mark.parametrize("B,N,C,groups", GN_SHAPES)
def test_groupnorm_silu_bwd(B, N, C, groups):
    ops_in, (dx, dw, db) = _gn_case(B, N, C, groups, seed=B * 1000 + N + C + groups)
    rdx, rdw, rdb, bdx, bdw, bdb = _gn_reference(*ops_in[:3], groups, ops_in[3])
    what = f"B{B} N{N} C{C} G{groups}"
    assert_close(dx, rdx, bdx, 5e-3, what + " dx")
    assert_close(dw, rdw, bdw, 1e-5, what + " dw")
    assert_close(db, rdb, bdb, 1e-5, what + " db")


@pytest.mark.parametrize("kind", ["constant_group", "mean_1000", "saturated"])
def test_groupnorm_silu_bwd_special_inputs(kind):
    B, N, C, groups = 3, 100, 512, 8
    kw = {"constant_group": dict(constant_group=True), "mean_1000": dict(mean=1000.0),
          "saturated": dict(saturate=True)}[kind]
    ops_in, (dx, dw, db) = _gn_case(B, N, C, groups, seed=17, **kw)
    for t in (dx, dw, db):
        assert bool(torch.isfinite(t.float()).all()), kind
    rdx, rdw, rdb, bdx, bdw, bdb = _gn_reference(*ops_in[:3], groups, ops_in[3])
    rel_w = 1e-4 if kind == "mean_1000" else 1e-5     # x_hat carries the fp32 mean's error (measured 3.1e-5)
    assert_close(dx, rdx, bdx, 5e-3, kind + " dx")
    assert_close(dw, rdw, bdw, rel_w, kind + " dw")
    assert_close(db, rdb, bdb, rel_w, kind + " db")


def test_groupnorm_silu_bwd_is_deterministic():
    ops_in, (dx, dw, db) = _gn_case(70, 100, 512, 8, seed=5)
    dx2 = torch.empty_like(dx)
    dw2, db2 = ops.groupnorm_silu_bwd(*ops_in[:3], 8, ops_in[3], dx2, eps=EPS)
    assert torch.equal(dw, dw2) and torch.equal(db, db2) and torch.equal(dx, dx2)


def test_groupnorm_silu_bwd_sensitivity():
    """The x_hat * mean(dx_hat * x_hat) term left out of the reference must fail both bounds."""
    ops_in, (dx, _, _) = _gn_case(3, 100, 512, 8, seed=9, correlated=True)
    rdx, _, _, bdx, _, _ = _gn_reference(*ops_in[:3], 8, ops_in[3])
    assert_close(dx, rdx, bdx, 5e-3, "correlated dy")
    wrong = _gn_reference(*ops_in[:3], 8, ops_in[3], drop_m2=True)[0]
    assert_rejects(dx, wrong, bdx, 5e-3, "no x_hat * mean(dx_hat * x_hat)")


# ---------------------------------------------------------------------------------------------------------------------
# rowdot_bwd
# ---------------------------------------------------------------------------------------------------------------------
def _rowdot_case(rows, dim, seed):
    g = gen(seed)
    x = torch.randn(rows, dim, device="cuda", generator=g)
    w = torch.randn(dim, device="cuda", generator=g) / dim ** 0.5
    pred = torch.relu(torch.randn(rows, device="cuda", generator=g))   # about half the rows exactly 0
    pred[::7] = 0.0
    dpred = torch.randn(rows, device="cuda", generator=g)
    dx0 = torch.randn(rows, dim, device="cuda", generator=g)            # the caller's residual gradient so far
    dx = dx0.clone()
    dw, db = ops.rowdot_bwd(x, w, pred, dpred, dx)
    return (x, w, pred, dpred, dx0), (dx, dw, db)


def _rowdot_reference(x, w, pred, dpred, dx0, ignore_gate=False):
    d = dpred.double() if ignore_gate else torch.where(pred > 0, dpred.double(), torch.zeros((), dtype=torch.float64,
                                                                                               device=pred.device))
    dx = dx0.double() + d[:, None] * w.double()
    dw = (d[:, None] * x.double()).sum(0)
    db = d.sum().reshape(1)
    rows = x.shape[0]
    bound_dx = U_F32 * (dx.abs() + (d[:, None] * w.double()).abs())
    bound_dw = U_F32 * dw.abs() + acc_eps(rows) * (d[:, None] * x.double()).abs().sum(0)
    bound_db = U_F32 * db.abs() + acc_eps(rows) * d.abs().sum().reshape(1)
    return (dx, dw, db), (bound_dx, bound_dw, bound_db)


@pytest.mark.parametrize("rows,dim", [(1, 4), (31, 12), (32, 512), (33, 2048), (100, 512), (257, 4), (4097, 512),
                                      (3200, 512), (4097, 2048)])
def test_rowdot_bwd(rows, dim):
    ops_in, got = _rowdot_case(rows, dim, seed=rows + dim)
    ref, bounds = _rowdot_reference(*ops_in)
    for name, o, r, bnd in zip(("dx", "dw", "db"), got, ref, bounds):
        assert_close(o, r, bnd, 1e-5, f"rows {rows} dim {dim} {name}")


def test_rowdot_bwd_exact_zero_prediction_takes_no_gradient():
    """pred == 0 exactly (ReLU at 0): d pre = 0, as torch's threshold_backward; the row's d x stays as it was."""
    x = torch.randn(64, 128, device="cuda")
    w = torch.randn(128, device="cuda")
    pred = torch.zeros(64, device="cuda")
    pred[5] = 1e-30                                                   # the smallest positive still passes
    dpred = torch.randn(64, device="cuda")
    dx0 = torch.randn(64, 128, device="cuda")
    dx = dx0.clone()
    dw, db = ops.rowdot_bwd(x, w, pred, dpred, dx)
    rows = torch.arange(64, device="cuda") != 5
    assert torch.equal(dx[rows], dx0[rows])
    assert torch.equal(db, dpred[5:6])
    assert torch.equal(dw, dpred[5] * x[5])


def test_rowdot_bwd_is_deterministic():
    ops_in, (_, dw, db) = _rowdot_case(4097, 2048, seed=3)
    dx = ops_in[4].clone()
    dw2, db2 = ops.rowdot_bwd(*ops_in[:4], dx)
    assert torch.equal(dw, dw2) and torch.equal(db, db2)


def test_rowdot_bwd_sensitivity():
    """A reference that ignores the ReLU gate must fail both bounds on d w."""
    ops_in, (_, dw, _) = _rowdot_case(1000, 512, seed=11)
    _, bounds = _rowdot_reference(*ops_in)
    (_, wrong, _), _ = _rowdot_reference(*ops_in, ignore_gate=True)
    assert_rejects(dw, wrong, bounds[1], 1e-5, "ReLU gate ignored")
