"""GPU: the GEMM epilogue's column vectors and its GELU against float64.

The epilogue reads each tile's bias (and for WAVENET its FiLM slice) from a shared-memory copy made under the tile's
mainloop; the copy is overwritten by every tile a persistent CTA takes.  These cases run many tiles per CTA over
several groups and a partial last n-tile, with a bias large enough that a slice from the wrong tile, group or column
cannot pass.  The GEGLU case sweeps the gate densely, tails past |x| = 5 included, with the accumulator exactly 0 so
that the output is the kernel's GELU of the bias alone.
"""
import math

import pytest
import torch

from kernel_check import U_BF16, U_F32, acc_eps, assert_close, assert_rejects, sm_limit

pytestmark = pytest.mark.gpu
bf = torch.bfloat16
dev = "cuda"


def _gen(seed):
    return torch.Generator(device=dev).manual_seed(seed)


@pytest.mark.parametrize("epi", ["bf16", "f32"])
@pytest.mark.parametrize("n", [1408, 224])   # BN 256 with a half-full last tile; BN 128 with a 96-column last tile
def test_bias_slices_across_tiles_and_groups(epi, n):
    from naturalspeech2_pytorch_b200 import ops
    B, N, K, G = 2, 300, 128, 3
    g = _gen(n + G)
    a = (torch.randn(B, N, G * K, device=dev, generator=g) * 0.5).to(bf)
    w = (torch.randn(G * n, K, device=dev, generator=g) / math.sqrt(K)).to(bf)
    bias = torch.randn(G * n, device=dev, generator=g) * 4
    f32 = epi == "f32"
    out = torch.full((B, N, G * n), float("nan"), device=dev, dtype=torch.float32 if f32 else bf)
    with sm_limit(2):   # 2 persistent CTAs: every CTA takes tiles of all groups and n-tiles in turn
        ops.gemm(a, w, out, n=n, epilogue=ops.EPI_F32 if f32 else ops.EPI_BF16, bias=bias, groups=G,
                 a_group_col_stride=K, b_group_row_stride=n, out_group_col_stride=n)
    a64, w64, b64 = a.double(), w.double(), bias.double()
    ref = torch.cat([a64[..., gi * K:(gi + 1) * K] @ w64[gi * n:(gi + 1) * n].T + b64[gi * n:(gi + 1) * n]
                     for gi in range(G)], dim=-1)
    mag = torch.cat([a64[..., gi * K:(gi + 1) * K].abs() @ w64[gi * n:(gi + 1) * n].abs().T
                     + b64[gi * n:(gi + 1) * n].abs() for gi in range(G)], dim=-1)
    u = U_F32 if f32 else U_BF16
    bound = u * ref.abs() + acc_eps(K) * mag
    assert_close(out, ref, bound, u + acc_eps(K), f"{epi} n={n}")
    # the same bias shifted by one 4-column piece, as a wrong slice would give
    wrong = ref - b64 + b64.view(G, n).roll(4, dims=1).flatten()
    assert_rejects(out, wrong, bound, u + acc_eps(K), f"{epi} n={n}: shifted bias")


def test_geglu_gelu_sweep_fp64():
    """out = value * gelu(gate) with value = 1 and gate = its bias: 4096 gate values in [-12, 12], one per column."""
    from naturalspeech2_pytorch_b200 import ops
    B, N, K, Dp = 2, 130, 64, 4096
    x = torch.zeros(B, N, K, device=dev, dtype=bf)
    W = torch.zeros(2 * Dp, K, device=dev, dtype=bf)
    gate = torch.linspace(-12.0, 12.0, Dp, device=dev)
    # packed layout: tile pair t holds value rows [256 t, 256 t + 128) and gate rows [256 t + 128, 256 t + 256)
    bp = torch.stack((torch.ones(Dp // 128, 128, device=dev), gate.view(-1, 128)), dim=1).reshape(2 * Dp)
    out = torch.full((B, N, Dp), float("nan"), device=dev, dtype=bf)
    with sm_limit(4):
        ops.gemm(x, W, out, n=2 * Dp, epilogue=ops.EPI_GEGLU, bias=bp.contiguous())
    g64 = gate.double()
    ref = (0.5 * g64 * (1.0 + torch.erf(g64 / math.sqrt(2.0)))).expand(B, N, Dp)
    # bf16 rounding of the output + an fp32 erf within 1e-6 of the true one (0.5 |x| |d erf|)
    bound = U_BF16 * ref.abs() + 0.5e-6 * g64.abs().expand(B, N, Dp)
    assert_close(out, ref, bound, U_BF16, "geglu gelu sweep")
    # the sigmoid approximation x sigmoid(1.702 x) must not pass for the exact-erf GELU (|x| <= 3, where they differ)
    mid = g64.abs() <= 3.0
    assert_rejects(out[..., mid], (g64 * torch.sigmoid(1.702 * g64))[mid].expand(B, N, -1), bound[..., mid], U_BF16,
                   "sigmoid GELU")
