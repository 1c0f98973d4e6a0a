"""GPU: the denoiser's feed-forward sublayer as `Model._forward_impl` runs it, x += W2 conv3(GEGLU(W1 h + b1)) + b2
(ns2.py:1009-1025), where the causal k=3 conv and W2 are ONE conv GEMM whose tap t is W2 @ Wc[:, :, t]
(`model._fold_conv_linear`), reduce-added into the fp32 residual stream.  Checked against float64 of the unfolded
reference math, and the GEMM configuration the fold uses (F32 in-place reduce-add over three shifted conv segments)
at partial row tiles inside NaN-guarded wider buffers.  Bounds and helpers: tests/kernel_check.py."""
import math

import pytest
import torch
import torch.nn.functional as F

from kernel_check import U_BF16, U_F32, acc_eps, assert_close, assert_nan, assert_rejects, shifted

pytestmark = pytest.mark.gpu
bf = torch.bfloat16
dev = "cuda"


def _gen(seed):
    return torch.Generator(device=dev).manual_seed(seed)


def _conv3(x, taps, shift_error=0):
    """sum_t shifted(x, 2 - t) @ taps[t]^T (float64), the causal k=3 conv; `shift_error` moves tap 1 by extra rows."""
    return sum(shifted(x, 2 - t + (shift_error if t == 1 else 0)) @ taps[t].T for t in range(3))


@pytest.fixture(scope="module")
def model():
    """One transformer layer at the denoiser's dims (dim 512, inner width 1365 padded to 1408) with bf16-representable
    parameters, so that the packs hold the parameters exactly except the folded taps, which are products."""
    from naturalspeech2_pytorch_b200 import Model
    torch.manual_seed(0)
    m = Model(dim=512, depth=1, heads=8, wavenet_layers=1, wavenet_stacks=1).to(dev)
    with torch.no_grad():
        for p in m.parameters():
            p.copy_(p.bfloat16().float())
    return m


def _sublayer(m, B, N, seed):
    from naturalspeech2_pytorch_b200 import ops
    P, D, Di = m.packed(), m.dim, m.ff_inner
    Dp = P["l0_ff_wo"].shape[1] // 3
    g = _gen(seed)
    h = torch.randn(B, N, D, device=dev, generator=g).to(bf)
    x = torch.randn(B, N, D, device=dev, generator=g)
    xr = x.clone()
    ff_g = torch.empty(B, N, Dp, device=dev, dtype=bf)
    ops.gemm(h, P["l0_ff_w1"], ff_g, n=2 * Dp, epilogue=ops.EPI_GEGLU, bias=P["l0_ff_b1"])
    ops.gemm(ff_g, P["l0_ff_wo"], xr, n=D, epilogue=ops.EPI_F32, bias=P["l0_ff_bo"], resid=xr, segs=ops.conv3_segs(Dp))

    ff = m.transformer.layers[0][5]
    W1, b1 = ff[0].weight.double(), ff[0].bias.double()
    Wc, bc = ff[2][1].weight.double(), ff[2][1].bias.double()
    W2, b2 = ff[-1].weight.double(), ff[-1].bias.double()
    h64 = h.double()
    pre, pmag = h64 @ W1.T + b1, h64.abs() @ W1.abs().T + b1.abs()
    v, gate, mv, mg = pre[..., :Di], pre[..., Di:], pmag[..., :Di], pmag[..., Di:]
    gel = F.gelu(gate)
    g64 = gel * v
    # the GEGLU output's error (tests/test_gemm_edges_gpu.py::test_gemm_geglu): bf16 rounding + accumulation of K = D
    g_err = U_BF16 * g64.abs() + acc_eps(D) * (1.13 * mg * v.abs() + gel.abs() * mv)
    c = _conv3(g64, [Wc[:, :, t] for t in range(3)]) + bc
    y = c @ W2.T + b2
    ref = x.double() + y
    folded = [W2 @ Wc[:, :, t] for t in range(3)]
    # through the folded taps: the GEGLU error, the taps' one bf16 rounding, fp32 accumulation of K = 3 Dp, and the
    # fp32 bias / residual adds
    mag = _conv3(g64.abs(), [w.abs() for w in folded])
    bound = (_conv3(g_err, [w.abs() for w in folded]) + (U_BF16 + acc_eps(3 * Dp)) * mag
             + U_F32 * (ref.abs() + x.double().abs() + y.abs()))
    rel = 2 * U_BF16 + acc_eps(3 * Dp)   # two bf16 roundings (g and the taps) reach the output
    return xr, x, ref, y, bound, rel, (g64, folded, W2 @ bc + b2)


@pytest.mark.parametrize("N", [1, 2, 3, 65, 1024])
def test_ff_sublayer_matches_fp64(model, N):
    B = 3   # an odd batch: the conv's zero padding is per sample
    xr, x, ref, y, bound, rel, _ = _sublayer(model, B, N, seed=N)
    inc = xr.double() - x.double()   # the sublayer's own output, exactly
    assert_close(inc, y, bound, rel, f"ff increment N={N}")
    assert_close(xr, ref, bound, rel, f"residual N={N}")
    # rows 0 and 1: their first taps read the causal padding, not the previous sample's last rows
    assert_close(inc[:, :2], y[:, :2], bound[:, :2], rel, f"rows 0-1 N={N}")


def test_ff_sublayer_sensitivity_tap_shift(model):
    """The sublayer's bounds reject a reference whose middle tap reads one row too early."""
    xr, x, ref, y, bound, rel, (g64, folded, bias) = _sublayer(model, 3, 65, seed=7)
    wrong = _conv3(g64, folded, shift_error=1) + bias
    assert_rejects(xr.double() - x.double(), wrong, bound, rel, "tap 1 shifted by one row")


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("N", [1, 2, 33, 65, 129, 200])
@pytest.mark.parametrize("n", [96, 288, 512])   # BN 128 partial tile; BN 256 with a 32-wide last tile; two full tiles
def test_f32_in_place_conv3_segments_partial_tiles(n, N, B):
    """F32 out += conv3(a) + bias by TMA reduce-add, the output a column window of a NaN-filled wider buffer with a
    spare row tile after the last batch, the input a column window of a NaN-filled wider buffer: columns past n,
    rows past the last batch and the input's outer columns must never be touched or read."""
    from naturalspeech2_pytorch_b200 import ops
    C = 192
    g = _gen(n * 100 + N * 10 + B)
    a_full = torch.full((B, N, C + 128), float("nan"), device=dev, dtype=bf)
    a = a_full[..., 64:64 + C]
    a.copy_(torch.randn(B, N, C, device=dev, generator=g) * 0.5)
    w = (torch.randn(n, 3 * C, device=dev, generator=g) / math.sqrt(3 * C)).to(bf)
    bias = torch.randn(n, device=dev, generator=g)
    resid = torch.randn(B, N, n, device=dev, generator=g)
    store = torch.full((B * N + 128, n + 64), float("nan"), device=dev)
    full = store[:B * N].view(B, N, n + 64)
    out = full[..., :n]
    out.copy_(resid)
    ops.gemm(a, w, out, n=n, epilogue=ops.EPI_F32, bias=bias, resid=out, segs=ops.conv3_segs(C))

    a64, w64 = a.double(), w.double()
    taps = [w64[:, t * C:(t + 1) * C] for t in range(3)]
    conv = _conv3(a64, taps) + bias.double()
    mag = _conv3(a64.abs(), [t.abs() for t in taps]) + bias.double().abs()
    ref = resid.double() + conv
    bound = U_F32 * (ref.abs() + resid.double().abs()) + acc_eps(3 * C) * mag
    assert_close(out, ref, bound, acc_eps(3 * C) * 4, f"n={n} N={N} B={B}")
    assert_nan(full[..., n:], "columns past n")
    assert_nan(store[B * N:], "rows past the last batch")
    if N > 2:
        wrong = resid.double() + _conv3(a64, taps, shift_error=1) + bias.double()
        assert_rejects(out, wrong, bound, acc_eps(3 * C) * 4, "tap 1 shifted by one row")


def _fold_ref(w2, wc, bc, b2):
    """float64 (taps (L, T, O, I), their magnitudes, bias, its magnitude) of `ops.fold_conv_linear`'s operands."""
    w2d, wcd = w2.double(), wc.double()
    taps = torch.einsum("lod,ldit->ltoi", w2d, wcd)
    mag = torch.einsum("lod,ldit->ltoi", w2d.abs(), wcd.abs())
    bias = torch.einsum("lod,ld->lo", w2d, bc.double()) + b2.double()
    bmag = torch.einsum("lod,ld->lo", w2d.abs(), bc.double().abs()) + b2.double().abs()
    return taps, mag, bias, bmag


@pytest.mark.parametrize("L,O,K,I,T,i_pad", [
    (12, 512, 1365, 1365, 3, 1408),   # the denoiser's feed-forwards (the bias column completes the last 128-wide tile)
    (2, 200, 77, 70, 3, 128),         # partial output-channel tile, K not a multiple of the 16-wide stage
    (3, 64, 16, 128, 2, 128),         # no padding columns, the bias column alone in its tile
    (1, 129, 300, 41, 5, 64),         # one row past a tile, five taps
])
def test_fold_kernel_matches_fp64(L, O, K, I, T, i_pad):
    """ns2_fold_conv_linear against float64: one bf16 rounding + fp32 accumulation of K products, padding exactly 0."""
    from naturalspeech2_pytorch_b200 import ops
    g = _gen(L * 1000 + O + K)
    w2 = torch.randn(L, O, K, device=dev, generator=g) / math.sqrt(K)
    wc = torch.randn(L, K, I, T, device=dev, generator=g) / math.sqrt(I * T)
    bc = torch.randn(L, K, device=dev, generator=g)
    b2 = torch.randn(L, O, device=dev, generator=g)
    wo, bo = ops.fold_conv_linear(w2, wc, bc, b2, i_pad)
    assert wo.shape == (L, O, T * i_pad) and bo.shape == (L, O)
    taps, mag, bias, bmag = _fold_ref(w2, wc, bc, b2)
    got = wo.view(L, O, T, i_pad).permute(0, 2, 1, 3)
    assert torch.equal(got[..., I:], torch.zeros_like(got[..., I:])), "padding columns must be exactly 0"
    bound = U_BF16 * taps.abs() + acc_eps(K) * mag
    assert_close(got[..., :I], taps, bound, U_BF16 + acc_eps(K), "folded taps")
    bbound = U_F32 * (bias.abs() + b2.double().abs()) + acc_eps(K) * bmag
    assert_close(bo, bias, bbound, acc_eps(K) * 4, "folded bias")
    wrong = taps.flip(1)   # the taps in the wrong order
    assert_rejects(got[..., :I], wrong, bound, U_BF16 + acc_eps(K), "taps reversed")


def test_model_fold_on_cuda_matches_the_cpu_fold():
    """The packs `Model` builds on the GPU (the kernel) and on the CPU (float64) agree to one bf16 rounding."""
    from naturalspeech2_pytorch_b200 import Model
    torch.manual_seed(0)
    m = Model(dim=256, depth=3, heads=4, wavenet_layers=1, wavenet_stacks=1)
    P_cpu = {k: v for k, v in m.packed().items() if "_ff_wo" in k or "_ff_bo" in k}
    mags = {}
    for l, layer in enumerate(m.transformer.layers):   # sum |w2| |wc| of each folded weight: fp32 accumulation's scale
        ff = layer[5]
        w2, wc = ff[-1].weight.detach().double().abs(), ff[2][1].weight.detach().double().abs()
        mag = torch.zeros_like(P_cpu[f"l{l}_ff_wo"], dtype=torch.float64).view(w2.shape[0], 3, -1)
        mag[:, :, :wc.shape[1]] = torch.einsum("od,dit->oti", w2, wc)
        mags[f"l{l}_ff_wo"] = mag.view(w2.shape[0], -1)
        mags[f"l{l}_ff_bo"] = w2 @ ff[2][1].bias.detach().double().abs() + ff[-1].bias.detach().double().abs()
    P_gpu = m.to(dev).packed()
    for k, v in P_cpu.items():
        a, b = P_gpu[k].double().cpu(), v.double()
        # at most one bf16 rounding apart, where fp32 accumulation moved the value across a rounding boundary
        assert bool(((a - b).abs() <= 2.0 ** -7 * b.abs() + acc_eps(m.ff_inner) * mags[k]).all()), k
        if k.endswith("_wo"):   # bf16: nearly all of them round to the same value
            assert (a == b).double().mean() > 0.99, k
