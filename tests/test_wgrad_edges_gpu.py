"""GPU: the weight-gradient GEMM (`ops.wgrad`) at its tile edges against a float64 reference.

Tile geometry (csrc/wgrad.cu): 128 dW rows (n) x BN dW columns (k) per tile, BN = 256 when k % 256 == 0 or k > 1024
and 128 otherwise; the position range runs in 64-row blocks and is split across CTAs (`splits`), whose partial sums
meet in dW through fp32 atomic adds.  The call accumulates into dW.
"""
import pytest
import torch

from kernel_check import U_F32, acc_eps, assert_close, assert_nan, assert_rejects, shifted

pytestmark = pytest.mark.gpu
bf = torch.bfloat16
dev = "cuda"


def _case(B, N, n, k, *, shift=0, x_col_off=0, splits=0, seed=0):
    """dy (B, N, n), x = NaN-padded window [x_col_off, x_col_off + k) of a wider (B, N, x_col_off + k + 64) buffer, dW
    (n + 8, k + 32) starting random with NaN in the rows / columns outside (n, k).  Returns (dy, x, dW before, after)."""
    from naturalspeech2_pytorch_b200 import ops
    g = torch.Generator(device=dev).manual_seed(seed)
    dy = torch.randn(B, N, n, device=dev, generator=g).to(bf)
    x = torch.full((B, N, x_col_off + k + 64), float("nan"), device=dev, dtype=bf)
    x[..., x_col_off:x_col_off + k] = torch.randn(B, N, k, device=dev, generator=g).to(bf)
    dw = torch.full((n + 8, k + 32), float("nan"), device=dev)
    dw[:n, :k] = torch.randn(n, k, device=dev, generator=g)
    start = dw[:n, :k].clone()
    ops.wgrad(dy, x, dw, n=n, k=k, shift_units=1 if shift else 0, dil=[max(shift, 1)], x_col_off=x_col_off,
              splits=splits)
    assert_nan(dw[n:], "dW rows past n")
    assert_nan(dw[:, k:], "dW columns past k")
    return dy, x[..., x_col_off:x_col_off + k], start, dw[:n, :k]


def _ref(dy, x, shift):
    """float64 dW increment and sum |dy||x| over the B*N positions."""
    xs = shifted(x.double(), shift)
    dyd = dy.double()
    return torch.einsum("bmn,bmk->nk", dyd, xs), torch.einsum("bmn,bmk->nk", dyd.abs(), xs.abs())


def _assert_increment(got, start, ref, mag, positions, what):
    # fp32 accumulation over the positions, 2^-20 sqrt(B N) sum |dy||x| (kernel_check.acc_eps), + fp32 rounding of
    # the sum with the starting value (recovered by subtracting it again)
    inc = got.double() - start.double()
    bound = acc_eps(positions) * mag + U_F32 * (got.double().abs() + start.double().abs())
    assert_close(inc, ref, bound, acc_eps(positions) * 4, what)
    return bound


@pytest.mark.parametrize("k", [
    32,     # BN=128, the only tile is 32 wide
    96,     # BN=128, the only tile is 96 wide
    224,    # BN=128, last tile 96 wide
    512,    # BN=256 (k % 256 == 0), two full tiles
    1056,   # k > 1024 with k % 256 != 0: BN=256, last tile 32 wide
    1408,   # BN=256 (k > 1024), last tile 128 wide
])
@pytest.mark.parametrize("n", [
    32,     # one 128-row tile, 32 valid rows: warpgroup 2 (rows 64..127) stores nothing
    96,     # warpgroup 2 stores 32 rows
    128,    # exactly one tile
    160,    # second tile with 32 rows
])
def test_wgrad_n_k_edges(n, k):
    B, N = 2, 300
    dy, x, start, got = _case(B, N, n, k, shift=2, seed=n * 10000 + k)
    ref, mag = _ref(dy, x, 2)
    _assert_increment(got, start, ref, mag, B * N, f"n={n} k={k}")


@pytest.mark.parametrize("shift", [
    0,      # no shift
    1,      # one row
    64,     # exactly one 64-position block
    130,    # more than two position blocks
    400,    # >= N for every N here: the tap reads only zero padding, dW must not change
])
@pytest.mark.parametrize("N", [
    1,      # a single position
    63,     # one partial position block
    65,     # one full block + one position
    300,    # 4 full blocks + 44 positions
])
def test_wgrad_rows_and_shifts(N, shift):
    B = 3
    dy, x, start, got = _case(B, N, 128, 224, shift=shift, seed=N * 1000 + shift)
    ref, mag = _ref(dy, x, shift)
    _assert_increment(got, start, ref, mag, B * N, f"N={N} shift={shift}")
    if shift >= N:
        assert torch.equal(got, start), "a tap entirely in the padding must add exactly zero"


@pytest.mark.parametrize("x_col_off", [
    0,      # window at the start of x
    64,     # one 64-channel TMA box in
    192,    # three boxes in; the last partial k-tile reads NaN columns past the window (masked on store)
])
def test_wgrad_x_col_off(x_col_off):
    B, N = 2, 200
    dy, x, start, got = _case(B, N, 128, 96, shift=1, x_col_off=x_col_off, seed=x_col_off)
    ref, mag = _ref(dy, x, 1)
    _assert_increment(got, start, ref, mag, B * N, f"x_col_off={x_col_off}")


def test_wgrad_splits_agree_and_single_split_is_deterministic():
    B, N, n, k = 3, 700, 160, 224        # 3 * 11 = 33 position blocks
    results = {}
    for splits in (
        0,     # automatic
        1,     # one CTA per tile walks every position block
        7,     # uneven: 5 blocks per split, the last split holds 3
        40,    # more splits than position blocks: 7 CTAs per tile have nothing to add and return early
    ):
        dy, x, start, got = _case(B, N, n, k, shift=1, splits=splits, seed=77)
        ref, mag = _ref(dy, x, 1)
        _assert_increment(got, start, ref, mag, B * N, f"splits={splits}")
        results[splits] = got.clone()
    _, _, _, again = _case(B, N, n, k, shift=1, splits=1, seed=77)
    assert torch.equal(again, results[1]), "splits=1 adds each dW element once: two runs must be bit-identical"


def test_wgrad_grouped_strided():
    """groups = 8 with x_group_col_stride wider than k (NaN in the gaps) and dW rows wider than k."""
    from naturalspeech2_pytorch_b200 import ops
    B, N, n, k, G, xgs = 2, 150, 128, 96, 8, 160
    g = torch.Generator(device=dev).manual_seed(8)
    dils = [2 ** i for i in range(G)]
    dy = torch.randn(B, N, G * n, device=dev, generator=g).to(bf)
    x = torch.full((B, N, G * xgs), float("nan"), device=dev, dtype=bf)
    for gi in range(G):
        x[..., gi * xgs:gi * xgs + k] = torch.randn(B, N, k, device=dev, generator=g).to(bf)
    dw = torch.full((G * n + 16, k + 32), float("nan"), device=dev)
    dw[:G * n, :k] = torch.randn(G * n, k, device=dev, generator=g)
    start = dw[:G * n, :k].clone()
    ops.wgrad(dy, x, dw, n=n, k=k, shift_units=2, groups=G, dy_group_col_stride=n, x_group_col_stride=xgs,
              dw_group_row_stride=n, dil=dils)
    assert_nan(dw[:, k:], "dW columns past k")
    assert_nan(dw[G * n:], "dW rows past the last group")
    for gi in range(G):
        ref, mag = _ref(dy[..., gi * n:(gi + 1) * n], x[..., gi * xgs:gi * xgs + k], 2 * dils[gi])
        _assert_increment(dw[gi * n:(gi + 1) * n, :k], start[gi * n:(gi + 1) * n], ref, mag, B * N, f"group {gi}")


def test_wgrad_sensitivity_tap_shift():
    """The wgrad tolerance rejects a reference whose tap is shifted by one extra row."""
    B, N = 2, 300
    dy, x, start, got = _case(B, N, 128, 224, shift=2, seed=3)
    ref, mag = _ref(dy, x, 2)
    bound = _assert_increment(got, start, ref, mag, B * N, "exact reference")
    wrong, _ = _ref(dy, x, 3)
    assert_rejects(got.double() - start.double(), wrong, bound, acc_eps(B * N) * 4, "tap shifted by one row")
