"""GPU: the SEANet decoder's kernels at their edges against float64 references on the same rounded operands:
the LSTM recurrence (cluster batch groups, saturated gates, skip, strided input, determinism), the ELU + reflect-pad
operand kernel (bit-exact), the transposed-conv GEMM mapping and the 32-channel tail kernel.  Each family has a
sensitivity case: a subtly wrong reference must fail the tolerance."""
import math

import pytest
import torch
import torch.nn.functional as F

from kernel_check import U_F32, acc_eps, assert_close, assert_rejects, gen

pytestmark = pytest.mark.gpu


def _bf(t):
    return t.to(torch.bfloat16)


# ------------------------------------------------------------------------------------------------
# LSTM
# ------------------------------------------------------------------------------------------------
def _lstm_inputs(B, T, seed, gate_scale=1.0):
    g = gen(seed)
    xp = torch.randn(B, T, 2048, device="cuda", generator=g) * gate_scale          # PyTorch gate order
    whh = _bf(torch.randn(2048, 512, device="cuda", generator=g) / math.sqrt(512))
    return xp, whh


def _lstm_ref(xp, whh, skip=None, swap_if=False):
    """float64 nn.LSTM recurrence from the precomputed projection; h_{t-1} rounded to bf16 like the kernel's operand."""
    xp, w = xp.double(), whh.double()
    B, T, _ = xp.shape
    h = xp.new_zeros(B, 512)
    c = xp.new_zeros(B, 512)
    out = []
    for t in range(T):
        g = xp[:, t] + h.to(torch.bfloat16).double() @ w.t()
        i, f, gg, o = g.chunk(4, dim=-1)
        if swap_if:
            i, f = f, i
        c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(gg)
        h = torch.sigmoid(o) * torch.tanh(c)
        out.append(h)
    y = torch.stack(out, dim=1)
    return y + skip.double() if skip is not None else y


def _run_lstm(xp, whh, skip=None, strided=False):
    from naturalspeech2_pytorch_b200 import ops
    from naturalspeech2_pytorch_b200.seanet import lstm_gate_perm
    perm = lstm_gate_perm().cuda()
    B, T, _ = xp.shape
    xk = xp[..., perm].contiguous()
    if strided:   # rows of 2048 + 64 values inside a wider buffer, a column window
        buf = torch.full((B, T, 2048 + 64), float("nan"), device="cuda")
        buf[..., 32:32 + 2048] = xk
        xk = buf[..., 32:32 + 2048]
    out = torch.full((B, T, 512), float("nan"), device="cuda")
    out_bf = torch.empty(B, T, 512, device="cuda", dtype=torch.bfloat16)
    ops.lstm_seq(xk, whh[perm].contiguous(), skip=skip, out=out, out_bf16=out_bf)
    torch.cuda.synchronize()
    return out, out_bf


LSTM_BOUND, LSTM_REL = 2e-2, 5e-3   # fp32 gates vs fp64 + the occasional flipped bf16 rounding of h fed back


@pytest.mark.parametrize("T", [1, 2, 37, 1024])
@pytest.mark.parametrize("B", [1, 31, 64, 65, 130])
def test_lstm_batch_groups_and_lengths(B, T):
    xp, whh = _lstm_inputs(B, T, seed=100 + B + T)
    out, out_bf = _run_lstm(xp, whh)
    ref = _lstm_ref(xp, whh)
    assert_close(out, ref, LSTM_BOUND, LSTM_REL, f"lstm B={B} T={T}")
    assert torch.equal(out_bf, out.to(torch.bfloat16))


def test_lstm_saturated_gates():
    xp, whh = _lstm_inputs(33, 40, seed=7, gate_scale=30.0)
    out, _ = _run_lstm(xp, whh)
    assert_close(out, _lstm_ref(xp, whh), LSTM_BOUND, LSTM_REL, "saturated")


def test_lstm_skip_and_strided_input():
    xp, whh = _lstm_inputs(66, 50, seed=8)
    skip_buf = torch.randn(66, 50, 512 + 16, device="cuda", generator=gen(9))
    skip = skip_buf[..., 8:8 + 512]
    out, _ = _run_lstm(xp, whh, skip=skip, strided=True)
    assert_close(out, _lstm_ref(xp, whh, skip=skip), LSTM_BOUND, LSTM_REL, "skip + strided")
    out0, _ = _run_lstm(xp, whh, strided=True)
    assert_close(out0, _lstm_ref(xp, whh), LSTM_BOUND, LSTM_REL, "no skip + strided")


def test_lstm_two_launches_bit_identical():
    xp, whh = _lstm_inputs(70, 300, seed=10)
    a, _ = _run_lstm(xp, whh)
    b, _ = _run_lstm(xp, whh)
    assert torch.equal(a, b)


def test_lstm_sensitivity_gate_order():
    xp, whh = _lstm_inputs(31, 37, seed=11)
    out, _ = _run_lstm(xp, whh)
    assert_rejects(out, _lstm_ref(xp, whh, swap_if=True), LSTM_BOUND, LSTM_REL, "i/f swapped")


# ------------------------------------------------------------------------------------------------
# ELU + reflect pad + bf16 cast (bit-exact)
# ------------------------------------------------------------------------------------------------
def _reflect_ref(x, p):
    """(B, T, C) -> (B, p + T, C): rows r < p hold x_ext[p - r] (x zero-extended to >= p + 1 rows)."""
    if p == 0:
        return x
    T = x.shape[1]
    xe = F.pad(x, (0, 0, 0, max(0, p + 1 - T)))
    return torch.cat([xe[:, 1:p + 1].flip(1), x], dim=1)


@pytest.mark.parametrize("p", [0, 2, 6])
@pytest.mark.parametrize("T_kind", ["1", "2", "p", "p+1", "4097"])
@pytest.mark.parametrize("elu", [False, True])
def test_elu_pad_bit_exact(p, T_kind, elu):
    from naturalspeech2_pytorch_b200 import ops
    T = {"1": 1, "2": 2, "p": max(p, 1), "p+1": p + 1, "4097": 4097}[T_kind]
    B, C = 3, 64
    g = gen(20 + p + T)
    base = torch.randn(B, T + 3, C + 8, device="cuda", generator=g) * 2
    x = base[:, 3:, 4:4 + C]                       # row offset 3, row stride C + 8
    out_buf = torch.full((B, p + T, 3 * C), float("nan"), device="cuda").to(torch.bfloat16)
    ops.elu_pad(x, out_buf, pad=p, elu=elu, raw=True)
    torch.cuda.synchronize()
    xp = _reflect_ref(x, p)
    act = F.elu(xp) if elu else xp
    assert torch.equal(out_buf[..., :C], act.to(torch.bfloat16))
    assert torch.equal(out_buf[..., C:2 * C], xp.to(torch.bfloat16))
    assert torch.isnan(out_buf[..., 2 * C:].float()).all()


# ------------------------------------------------------------------------------------------------
# transposed convolution as a 2-segment GEMM
# ------------------------------------------------------------------------------------------------
def _convt_ref(x, w, b, s):
    y = F.conv_transpose1d(x.double().transpose(1, 2), w.double(), None if b is None else b.double(), stride=s)
    return y[..., :s * x.shape[1]].transpose(1, 2)


@pytest.mark.parametrize("s,c_in,c_out", [(8, 512, 256), (5, 256, 128), (4, 128, 64), (2, 64, 32)])
@pytest.mark.parametrize("N", [1, 2, 129])
def test_conv_transpose_gemm_mapping(s, c_in, c_out, N):
    from naturalspeech2_pytorch_b200 import ops
    from naturalspeech2_pytorch_b200.seanet import pack_conv_transpose
    g = gen(30 + s + N)
    B = 2
    x = _bf(torch.randn(B, N, c_in, device="cuda", generator=g))
    w = _bf(torch.randn(c_in, c_out, 2 * s, device="cuda", generator=g) / math.sqrt(2 * c_in)).float()
    b = torch.randn(c_out, device="cuda", generator=g) * 0.1
    pw, pb = pack_conv_transpose(w, b, s)
    out = torch.empty(B, N, s * c_out, device="cuda")
    ops.gemm(x, pw, out, n=s * c_out, epilogue=ops.EPI_F32, segs=[(0, 0, c_in, 0, 0), (0, c_in, c_in, 1, 0)], bias=pb)
    torch.cuda.synchronize()
    got = out.view(B, s * N, c_out)
    ref = _convt_ref(x, w, b, s)
    bound = acc_eps(2 * c_in) * _convt_ref(x.abs(), w.abs(), None, s) + U_F32 * ref.abs() + 1e-6
    assert_close(got, ref, bound, 1e-5, f"convT s={s} N={N}")
    if N == 129:
        w_swapped = torch.cat([w[..., s:], w[..., :s]], dim=-1)
        assert_rejects(got, _convt_ref(x, w_swapped, b, s), bound, 1e-5, "tap halves swapped")


# ------------------------------------------------------------------------------------------------
# 32-channel tail
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def tail_params():
    from naturalspeech2_pytorch_b200 import SEANetDecoder
    from naturalspeech2_pytorch_b200.seanet import pack_tail
    dec = SEANetDecoder()
    g = torch.Generator().manual_seed(40)
    sd = {k: (torch.randn(v.shape, generator=g, dtype=torch.float64) * (0.1 if "bias" in k else 1.0))
          for k, v in dec.state_dict().items() if k.startswith(("layers.13.", "layers.15."))}
    fold = lambda pre: (sd[pre + ".parametrizations.weight.original0"] * sd[pre + ".parametrizations.weight.original1"]
                        / sd[pre + ".parametrizations.weight.original1"].norm(dim=(1, 2), keepdim=True),
                        sd[pre + ".bias"])
    w3, b3 = fold("layers.13.block.1.conv")
    w1, b1 = fold("layers.13.block.3.conv")
    wsc, bsc = fold("layers.13.shortcut.conv")
    wf, bf = fold("layers.15.conv")
    # fp32-representable weights, so the fp64 reference sees exactly what the kernel multiplies by
    sd = {k: v.float().double().cuda() for k, v in sd.items()}
    packed = pack_tail(*(t.float() for t in (w3, b3, w1, b1, wsc, bsc, wf, bf))).cuda()
    return sd, packed


def _tail_ref(x, sd, zero_pad=False):
    import seanet_oracle
    xc = x.double().transpose(1, 2)
    if zero_pad:
        orig = seanet_oracle.reflect_pad_left
        seanet_oracle.reflect_pad_left = lambda t, p: F.pad(t, (p, 0))
    try:
        z = seanet_oracle.resnet_block(xc, sd, "layers.13")
        y = seanet_oracle.conv(F.elu(z), sd, "layers.15.conv", False)
    finally:
        if zero_pad:
            seanet_oracle.reflect_pad_left = orig
    return y[:, 0]


TAIL_REL = 1e-5


@pytest.mark.parametrize("T", [1, 3, 6, 7, 9, 121, 122, 123, 244, 245, 1000, 4099])
def test_tail_kernel(tail_params, T):
    from naturalspeech2_pytorch_b200 import ops
    sd, packed = tail_params
    B = 3
    base = torch.randn(B, T, 40, device="cuda", generator=gen(50 + T))
    x = base[..., 4:36]                                   # row stride 40
    out = torch.full((B, T + 5), float("nan"), device="cuda")
    ops.seanet_tail(x, packed, out[:, :T])
    torch.cuda.synchronize()
    assert torch.isnan(out[:, T:]).all()
    ref = _tail_ref(x, sd)
    bound = 1e-4 * (1 + ref.abs())
    assert_close(out[:, :T], ref, bound, TAIL_REL, f"tail T={T}")
    if T == 7:
        assert_rejects(out[:, :T], _tail_ref(x, sd, zero_pad=True), bound, TAIL_REL, "zero instead of reflect")
