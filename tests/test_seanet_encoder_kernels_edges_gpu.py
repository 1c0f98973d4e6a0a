"""GPU: the SEANet encoder's new operations at their edges against float64 references on the same operands: the
full-rate head kernel (tile and halo edges, the reflected rows, a strided batch, determinism) and the strided-conv
GEMM mapping for each of the encoder's four (stride, channels) shapes.  Each has a sensitivity case: a subtly wrong
reference must fail the tolerance."""
import math

import pytest
import torch
import torch.nn.functional as F

from kernel_check import U_BF16, U_F32, acc_eps, assert_close, assert_rejects, gen

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------
# head: conv7 (1 -> 32), ResnetBlock(32), ELU, reflect pad 2, bf16
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def head_params():
    from naturalspeech2_pytorch_b200 import SEANetEncoder
    from naturalspeech2_pytorch_b200.seanet import pack_head
    enc = SEANetEncoder()
    g = torch.Generator().manual_seed(60)
    sd = {k: (torch.randn(v.shape, generator=g, dtype=torch.float64) * (0.1 if "bias" in k else 1.0))
          for k, v in enc.state_dict().items() if k.startswith(("layers.0.", "layers.1."))}
    fold = lambda pre: (sd[pre + ".parametrizations.weight.original0"] * sd[pre + ".parametrizations.weight.original1"]
                        / sd[pre + ".parametrizations.weight.original1"].norm(dim=(1, 2), keepdim=True),
                        sd[pre + ".bias"])
    parts = [fold(p) for p in ("layers.0.conv", "layers.1.block.1.conv", "layers.1.block.3.conv",
                               "layers.1.shortcut.conv")]
    packed = pack_head(*(t.float() for pair in parts for t in pair)).cuda()
    # fp32-representable weights, so the fp64 reference sees exactly what the kernel multiplies by
    sd = {k: v.float().double().cuda() for k, v in sd.items()}
    return sd, packed


def _reflect_off_by_one(x, p):
    """A wrong reflect pad that repeats the edge sample: xpad[i] = x[p - 1 - i]."""
    return torch.cat([x[..., :p].flip(-1), x], dim=-1) if p else x


def _head_ref(x, sd, pad=None):
    """(B, T) -> (B, T + 2, 32) float64: ELU(ResnetBlock(conv7(x))) reflect-padded by 2 (or by `pad`, a wrong one)."""
    import seanet_oracle
    orig = seanet_oracle.reflect_pad_left
    if pad is not None:
        seanet_oracle.reflect_pad_left = pad
    try:
        z0 = seanet_oracle.conv(x.double()[:, None], sd, "layers.0.conv", False)
        z1 = seanet_oracle.resnet_block(z0, sd, "layers.1")
        y = seanet_oracle.reflect_pad_left(F.elu(z1), 2)
    finally:
        seanet_oracle.reflect_pad_left = orig
    return y.transpose(1, 2)


HEAD_REL = 4e-3   # bf16 output rounding (~1.1e-3 rel-L2) with margin


def _run_head(x, packed):
    from naturalspeech2_pytorch_b200 import ops
    B, T = x.shape
    buf = torch.full((B, T + 2, 48), float("nan"), device="cuda").to(torch.bfloat16)
    ops.seanet_head(x, packed, buf[..., 8:40])           # row stride 48, column offset 8 (16-byte aligned)
    torch.cuda.synchronize()
    assert torch.isnan(buf[..., :8].float()).all() and torch.isnan(buf[..., 40:].float()).all()
    return buf[..., 8:40]


@pytest.mark.parametrize("T", [1, 2, 3, 7, 9, 125, 126, 127, 252, 253, 320, 1000, 4099])
def test_head_kernel(head_params, T):
    sd, packed = head_params
    B = 3
    base = torch.rand(B, T + 9, device="cuda", generator=gen(70 + T)) * 2 - 1
    x = base[:, 5:5 + T]                                  # batch stride T + 9
    out = _run_head(x, packed)
    ref = _head_ref(x, sd)
    bound = U_BF16 * ref.abs() + 1e-5 * (1 + ref.abs())
    assert_close(out, ref, bound, HEAD_REL, f"head T={T}")
    if T >= 3:   # the two reflected output rows repeat rows 3 and 4 (z1 at 1 and 2) bit for bit
        assert torch.equal(out[:, 0], out[:, 4]) and torch.equal(out[:, 1], out[:, 3])
    if T == 9:
        assert_rejects(out, _head_ref(x, sd, pad=lambda t, p: F.pad(t, (p, 0))), bound, HEAD_REL,
                       "zero instead of reflect")
        assert_rejects(out, _head_ref(x, sd, pad=_reflect_off_by_one), bound, HEAD_REL, "reflect off by one")


def test_head_two_launches_bit_identical(head_params):
    _, packed = head_params
    x = torch.rand(5, 32000, device="cuda", generator=gen(80)) * 2 - 1
    assert torch.equal(_run_head(x, packed), _run_head(x, packed))


# ------------------------------------------------------------------------------------------------
# strided convolution (k = 2s, stride s, reflect pad s) as a 2-segment GEMM
# ------------------------------------------------------------------------------------------------
def _strided_ref(a, w, b, s):
    """a: the (B, L + s, C) padded bf16 operand; fp64 F.conv1d(stride=s) -> (B, L / s, C_out)."""
    y = F.conv1d(a.double().transpose(1, 2), w.double(), None if b is None else b.double(), stride=s)
    return y.transpose(1, 2)


@pytest.mark.parametrize("s,c_in", [(2, 32), (4, 64), (5, 128), (8, 256)])
@pytest.mark.parametrize("N", [1, 2, 129])
def test_strided_conv_gemm_mapping(s, c_in, N):
    from naturalspeech2_pytorch_b200 import ops
    from naturalspeech2_pytorch_b200.seanet import pack_strided_conv, strided_conv_segs
    g = gen(90 + s + N)
    B, L, c_out = 2, s * N, 2 * c_in
    x = torch.randn(B, L, c_in, device="cuda", generator=g)
    w = (torch.randn(c_out, c_in, 2 * s, device="cuda", generator=g) / math.sqrt(2 * s * c_in)).to(torch.bfloat16).float()
    b = torch.randn(c_out, device="cuda", generator=g) * 0.1
    a = torch.empty(B, L + s, c_in, device="cuda", dtype=torch.bfloat16)
    ops.elu_pad(x, a, pad=s, elu=True)
    y = torch.full((B, N + 1, c_out), float("nan"), device="cuda")
    ops.gemm(a.view(B, N + 1, s * c_in), pack_strided_conv(w), y, n=c_out, epilogue=ops.EPI_F32,
             segs=strided_conv_segs(s, c_in), bias=b)
    torch.cuda.synchronize()
    got = y[:, 1:]
    ref = _strided_ref(a, w, b, s)
    bound = acc_eps(2 * s * c_in) * _strided_ref(a.abs(), w.abs(), None, s) + U_F32 * ref.abs() + 1e-6
    assert_close(got, ref, bound, 1e-5, f"strided conv s={s} C={c_in} N={N}")
    if N == 129:
        w_swapped = torch.cat([w[..., s:], w[..., :s]], dim=-1)
        assert_rejects(got, _strided_ref(a, w_swapped, b, s), bound, 1e-5, "taps swapped between the segments")
