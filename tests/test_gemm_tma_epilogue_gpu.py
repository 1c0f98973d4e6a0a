"""GPU: the GEMM epilogue's TMA stores at the tile edges, against a float64 reference.

The epilogue (csrc/gemm.cu) stages every consumer warpgroup's 64 rows in shared-memory boxes of 128 bytes per row
(64 bf16 or 32 fp32 columns) and writes them with TMA stores clipped at n (inside every group) and at a_rows (inside
every batch).  An F32 epilogue whose residual is `out` itself adds acc + bias into `out` with a TMA reduce-add at L2
and never reads the residual; a residual held elsewhere is read by the epilogue and stored with the sum.  Both must
give the same bits.
"""
import math

import pytest
import torch

from kernel_check import U_BF16, U_F32, acc_eps, assert_close, assert_nan

pytestmark = pytest.mark.gpu
bf = torch.bfloat16
dev = "cuda"


def _gen(seed):
    return torch.Generator(device=dev).manual_seed(seed)


def _operands(B, N, K, n, groups, seed):
    g = _gen(seed)
    a = (torch.randn(B, N, groups * K, device=dev, generator=g) * 0.5).to(bf)
    w = (torch.randn(groups * n, K, device=dev, generator=g) / math.sqrt(K)).to(bf)
    bias = torch.randn(groups * n, device=dev, generator=g)
    return a, w, bias


def _ref(a, w, bias, K, n, groups, silu):
    """float64 (value, error magnitude) per group: acc + bias (SiLU'd), and acc_eps(K) sum |a||w| + |bias|."""
    vals, mags = [], []
    for gi in range(groups):
        a64 = a[..., gi * K:(gi + 1) * K].double()
        w64 = w[gi * n:(gi + 1) * n].double()
        pre = a64 @ w64.T + bias[gi * n:(gi + 1) * n].double()
        mag = a64.abs() @ w64.abs().T + bias[gi * n:(gi + 1) * n].double().abs()
        vals.append(pre * torch.sigmoid(pre) if silu else pre)
        mags.append((1.1 if silu else 1.0) * acc_eps(K) * mag)
    return vals, mags


def _buffer(B, N, width, dtype):
    """NaN-filled (B, N, width) rows plus one spare 128-row tile after the last batch."""
    store = torch.full((B * N + 128, width), float("nan"), device=dev, dtype=dtype)
    return store, store[:B * N].view(B, N, width)


def _gemm(a, w, out, n, K, groups, gcs, **kw):
    from naturalspeech2_pytorch_b200 import ops
    return ops.gemm(a, w, out, n=n, groups=groups, a_group_col_stride=K, b_group_row_stride=n,
                    out_group_col_stride=gcs, segs=[(0, 0, K, 0, 0)], **kw)


def _f32_resid_case(B, N, K, n, *, groups=1, gap=64, flags=0, seed=0):
    """In-place and out-of-place F32 + residual into a row-strided window of a NaN-filled wider buffer."""
    from naturalspeech2_pytorch_b200 import ops
    gcs = n + gap if groups > 1 else 0
    width = groups * (n + gap) + 32
    a, w, bias = _operands(B, N, K, n, groups, seed)
    vals, mags = _ref(a, w, bias, K, n, groups, bool(flags & 4))
    resid = torch.randn(B, N, width, device=dev, generator=_gen(seed + 1))

    store, full = _buffer(B, N, width, torch.float32)
    win = full[..., :width - 32]
    for gi in range(groups):   # the residual lives in the output's own columns; gaps between groups stay NaN
        c0 = gi * gcs
        win[..., c0:c0 + n] = resid[..., c0:c0 + n]
    _gemm(a, w, win, n, K, groups, gcs, epilogue=ops.EPI_F32, bias=bias, resid=win, flags=flags)

    store2, full2 = _buffer(B, N, width, torch.float32)
    win2 = full2[..., :width - 32]
    res2 = torch.full_like(resid, float("nan"))
    for gi in range(groups):
        c0 = gi * gcs
        res2[..., c0:c0 + n] = resid[..., c0:c0 + n]
    _gemm(a, w, win2, n, K, groups, gcs, epilogue=ops.EPI_F32, bias=bias, resid=res2[..., :width - 32], flags=flags)

    for gi in range(groups):
        c0 = gi * gcs
        r = resid[..., c0:c0 + n].double()
        ref = vals[gi] + r
        bound = U_F32 * (ref.abs() + r.abs()) + mags[gi]
        assert_close(full[..., c0:c0 + n], ref, bound, acc_eps(K) * 4, f"in place, group {gi}")
        assert torch.equal(full[..., c0:c0 + n], full2[..., c0:c0 + n]), f"group {gi}: in place != out of place"
        if groups > 1 and gi < groups - 1:
            assert_nan(full[..., c0 + n:c0 + gcs], f"in place: gap after group {gi}")
            assert_nan(full2[..., c0 + n:c0 + gcs], f"out of place: gap after group {gi}")
    last = (groups - 1) * gcs + n
    for st, fu, what in ((store, full, "in place"), (store2, full2, "out of place")):
        assert_nan(fu[..., last:], f"{what}: columns past n")
        assert_nan(st[B * N:], f"{what}: rows past the last batch")
    return a, w, bias, resid, full


N_COLS = [32, 96, 160, 256, 288, 480, 512]   # BN=128 full / partial tiles; BN=256 full, 32-, 224-wide last tiles
N_ROWS = [1, 33, 65, 129, 200]               # empty second warpgroup, partial warpgroups, a second row tile


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("N", N_ROWS)
@pytest.mark.parametrize("n", N_COLS)
def test_f32_resid_in_place_tile_edges(n, N, B):
    _f32_resid_case(B, N, 192, n, seed=n * 1000 + N * 10 + B)


@pytest.mark.parametrize("n", [96, 160])
def test_f32_resid_in_place_silu(n):
    _f32_resid_case(2, 77, 128, n, flags=4, seed=n)   # NS2_GEMM_FLAG_SILU: out += silu(acc + bias)


@pytest.mark.parametrize("n,N", [(96, 65), (160, 200), (288, 129)])
def test_f32_resid_in_place_groups(n, N):
    _f32_resid_case(2, N, 64, n, groups=3, gap=32, seed=7 * n + N)


@pytest.mark.parametrize("n,N", [(96, 65), (32, 1), (352, 200)])
def test_bf16_groups_partial_box(n, N):
    """groups > 1 with n not a multiple of the 64-column bf16 box: each group's last box is clipped at n, so nothing
    lands in the gap before the next group's columns."""
    from naturalspeech2_pytorch_b200 import ops
    B, K, groups, gap = 2, 64, 3, 32
    gcs = n + gap
    a, w, bias = _operands(B, N, K, n, groups, seed=n + N)
    vals, mags = _ref(a, w, bias, K, n, groups, False)
    store, full = _buffer(B, N, groups * gcs + 64, bf)
    _gemm(a, w, full[..., :groups * gcs], n, K, groups, gcs, epilogue=ops.EPI_BF16, bias=bias)
    for gi in range(groups):
        c0 = gi * gcs
        assert_close(full[..., c0:c0 + n], vals[gi], U_BF16 * vals[gi].abs() + mags[gi], U_BF16 + acc_eps(K),
                     f"group {gi}")
        assert_nan(full[..., c0 + n:c0 + gcs], f"gap after group {gi}")
    assert_nan(full[..., groups * gcs:], "columns past the last group")
    assert_nan(store[B * N:], "rows past the last batch")


def test_f32_resid_in_place_two_launches_bit_identical():
    from naturalspeech2_pytorch_b200 import ops
    B, N, K, n = 3, 200, 512, 512
    a, w, bias = _operands(B, N, K, n, 1, seed=11)
    x0 = torch.randn(B, N, n, device=dev, generator=_gen(12))
    outs = []
    for _ in range(2):
        x = x0.clone()
        ops.gemm(a, w, x, n=n, epilogue=ops.EPI_F32, bias=bias, resid=x)
        outs.append(x)
    assert torch.equal(outs[0], outs[1])
