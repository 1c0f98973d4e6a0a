"""Torch restatement of Encodec's 24 kHz SEANet decoder and encoder, from their layer descriptions (not from any
implementation): runs in any dtype on any device, on a state_dict with transformers' `EncodecDecoder` /
`EncodecEncoder` key names.

`decode`:
    0      causal Conv1d k7 128 -> 512
    1      2-layer LSTM(512), lstm(x)[0] + x
    2-13   per ratio s in (8, 5, 4, 2): ELU, causal ConvTranspose1d k 2s stride s (C -> C/2, trim s on the right),
           ResnetBlock(C/2): shortcut(x) + conv1x1(ELU(conv3(ELU(x)))), hidden C/4, 1x1 conv shortcut
    14-15  ELU, causal Conv1d k7 32 -> 1
`encode`:
    0      causal Conv1d k7 1 -> 32
    1-12   per ratio s in (2, 4, 5, 8): ResnetBlock(C), ELU, causal Conv1d k 2s stride s (C -> 2C)
    13     2-layer LSTM(512), lstm(x)[0] + x
    14-15  ELU, causal Conv1d k7 512 -> 128
Causal convs pad (k - stride) on the left by reflection; an input no longer than the pad is zero-extended to pad + 1
samples first (Encodec's rule).  Every length the encoder sees is a multiple of the stride, so no right padding
arises.  Weight norm: w = g v / ||v|| over every dim but 0.

`emulate_bf16=True` rounds every convolution / projection operand (activation and weight) and the LSTM's recurrent
h_{t-1} and W_hh to bf16, the operand rounding of the CUDA path; sums, biases, cell state and activations between
layers keep the working dtype.  So does the encoder's full-rate head (layers 0-2), which the CUDA head kernel computes
in fp32: only its output, the first strided conv's operand, is rounded.
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


def conv(x, sd, prefix, emulate, stride=1):
    """Causal Conv1d with reflect left padding k - stride."""
    w, b = _wn(sd, prefix, x.dtype)
    return F.conv1d(reflect_pad_left(_r(x, emulate), w.shape[-1] - stride), _r(w, emulate), b, stride=stride)


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


def lstm_skip(x, sd, prefix, emulate=False):
    """x (B, C, T) -> lstm(x)[0] + x for the 2-layer LSTM at `prefix`."""
    xt = x.transpose(1, 2)
    y = xt
    for l in range(2):
        y = lstm_layer(y, *(sd[f"{prefix}.{n}_l{l}"].to(x.dtype) for n in ("weight_ih", "weight_hh", "bias_ih",
                                                                          "bias_hh")), emulate=emulate)
    return (y + xt).transpose(1, 2)


def resnet_block(x, sd, prefix, emulate=False):
    h = conv(F.elu(x), sd, prefix + ".block.1.conv", emulate)
    y = conv(F.elu(h), sd, prefix + ".block.3.conv", emulate)
    return conv(x, sd, prefix + ".shortcut.conv", emulate) + y


@torch.no_grad()
def decode(sd, emb: torch.Tensor, dtype=torch.float64, emulate_bf16: bool = False) -> torch.Tensor:
    """emb (B, N, 128) token-major -> audio (B, 1, 320 N) in `dtype`."""
    e = emulate_bf16
    x = emb.to(dtype).transpose(1, 2)
    x = lstm_skip(conv(x, sd, "layers.0.conv", e), sd, "layers.1.lstm", e)
    for si, s in enumerate(RATIOS):
        i = 2 + 3 * si
        x = _conv_t(F.elu(x), sd, f"layers.{i + 1}.conv", s, e)
        x = resnet_block(x, sd, f"layers.{i + 2}", e)
    return conv(F.elu(x), sd, "layers.15.conv", e)


@torch.no_grad()
def encode(sd, audio: torch.Tensor, dtype=torch.float64, emulate_bf16: bool = False) -> torch.Tensor:
    """audio (B, T), T % 320 == 0 -> frames (B, T / 320, 128) token-major in `dtype`."""
    e = emulate_bf16
    x = conv(audio.to(dtype)[:, None], sd, "layers.0.conv", False)
    for si, s in enumerate(reversed(RATIOS)):
        i = 1 + 3 * si
        x = resnet_block(x, sd, f"layers.{i}", e and si > 0)
        x = conv(F.elu(x), sd, f"layers.{i + 2}.conv", e, stride=s)
    x = lstm_skip(x, sd, "layers.13.lstm", e)
    return conv(F.elu(x), sd, "layers.15.conv", e).transpose(1, 2)
