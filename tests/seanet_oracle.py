"""Torch restatement of Encodec's 24 kHz SEANet decoder, from its layer description (not from any implementation):
runs in any dtype on any device, on a state_dict with transformers' `EncodecDecoder` key names.

    0      causal Conv1d k7 128 -> 512
    1      2-layer LSTM(512), lstm(x)[0] + x
    2-13   per ratio s in (8, 5, 4, 2): ELU, causal ConvTranspose1d k 2s stride s (C -> C/2, trim s on the right),
           ResnetBlock(C/2): shortcut(x) + conv1x1(ELU(conv3(ELU(x)))), hidden C/4, 1x1 conv shortcut
    14-15  ELU, causal Conv1d k7 32 -> 1
Causal convs pad (k - 1) on the left by reflection; an input no longer than the pad is zero-extended to pad + 1
samples first.  Weight norm: w = g v / ||v|| over every dim but 0.

`emulate_bf16=True` rounds every convolution / projection operand (activation and weight) and the LSTM's recurrent
h_{t-1} and W_hh to bf16, the operand rounding of the CUDA path; sums, biases, cell state and activations between
layers keep the working dtype.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

RATIOS = (8, 5, 4, 2)


def _r(t: torch.Tensor, emulate: bool) -> torch.Tensor:
    return t.to(torch.bfloat16).to(t.dtype) if emulate else t


def reflect_pad_left(x: torch.Tensor, p: int) -> torch.Tensor:
    """(B, C, T) -> (B, C, p + T): xpad[i] = x_ext[p - i] for i < p, x_ext = x zero-extended to >= p + 1 samples."""
    if p == 0:
        return x
    T = x.shape[-1]
    xe = F.pad(x, (0, max(0, p + 1 - T)))
    idx = torch.arange(p, 0, -1, device=x.device)
    return torch.cat([xe[..., idx], x], dim=-1)


def _wn(sd, prefix, dtype):
    g = sd[prefix + ".parametrizations.weight.original0"].to(dtype)
    v = sd[prefix + ".parametrizations.weight.original1"].to(dtype)
    return g * v / v.norm(dim=tuple(range(1, v.dim())), keepdim=True), sd[prefix + ".bias"].to(dtype)


def _conv(x, sd, prefix, emulate):
    w, b = _wn(sd, prefix, x.dtype)
    return F.conv1d(reflect_pad_left(_r(x, emulate), w.shape[-1] - 1), _r(w, emulate), b)


def _conv_t(x, sd, prefix, s, emulate):
    w, b = _wn(sd, prefix, x.dtype)
    y = F.conv_transpose1d(_r(x, emulate), _r(w, emulate), b, stride=s)
    return y[..., :s * x.shape[-1]]


def lstm_layer(x, w_ih, w_hh, b_ih, b_hh, emulate=False):
    """x (B, T, C) -> (B, T, H): nn.LSTM semantics (gates i, f, g, o; zero initial state)."""
    B, T, _ = x.shape
    H = w_hh.shape[1]
    xp = _r(x, emulate) @ _r(w_ih, emulate).t() + b_ih + b_hh
    whh = _r(w_hh, emulate)
    h = x.new_zeros(B, H)
    c = x.new_zeros(B, H)
    out = []
    for t in range(T):
        g = xp[:, t] + _r(h, emulate) @ whh.t()
        i, f, gg, o = g.chunk(4, dim=-1)
        c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(gg)
        h = torch.sigmoid(o) * torch.tanh(c)
        out.append(h)
    return torch.stack(out, dim=1)


def resnet_block(x, sd, prefix, emulate=False):
    h = _conv(F.elu(x), sd, prefix + ".block.1.conv", emulate)
    y = _conv(F.elu(h), sd, prefix + ".block.3.conv", emulate)
    return _conv(x, sd, prefix + ".shortcut.conv", emulate) + y


@torch.no_grad()
def decode(sd, emb: torch.Tensor, dtype=torch.float64, emulate_bf16: bool = False) -> torch.Tensor:
    """emb (B, N, 128) token-major -> audio (B, 1, 320 N) in `dtype`."""
    e = emulate_bf16
    x = emb.to(dtype).transpose(1, 2)
    x = _conv(x, sd, "layers.0.conv", e)
    xt = x.transpose(1, 2)
    y = xt
    for l in range(2):
        y = lstm_layer(y, *(sd[f"layers.1.lstm.{n}_l{l}"].to(dtype) for n in ("weight_ih", "weight_hh", "bias_ih",
                                                                             "bias_hh")), emulate=e)
    x = (y + xt).transpose(1, 2)
    for si, s in enumerate(RATIOS):
        i = 2 + 3 * si
        x = _conv_t(F.elu(x), sd, f"layers.{i + 1}.conv", s, e)
        x = resnet_block(x, sd, f"layers.{i + 2}", e)
    return _conv(F.elu(x), sd, "layers.15.conv", e)
