"""Torch restatement of Encodec's 24 kHz SEANet encoder, from its layer description (not from any implementation):
runs in any dtype on any device, on a state_dict with transformers' `EncodecEncoder` key names.  It shares the
decoder restatement's building blocks (`seanet_oracle`: reflect padding, weight norm, ResnetBlock, LSTM) and adds
the strided convolution.

    0      causal Conv1d k7 1 -> 32
    1-12   per ratio s in (2, 4, 5, 8): ResnetBlock(C), ELU, causal Conv1d k 2s stride s (C -> 2C)
    13     2-layer LSTM(512), lstm(x)[0] + x
    14-15  ELU, causal Conv1d k7 512 -> 128
Causal convs pad (k - stride) on the left by reflection (Encodec's rule for inputs no longer than the pad: zero-extend
first); every length here is a multiple of the stride, so no right padding arises.

`emulate_bf16=True` rounds the operands the CUDA path rounds (see `seanet_oracle`).  The full-rate head (layers 0-2)
keeps the working dtype throughout, as the CUDA head kernel computes it in fp32; only its output, the first strided
conv's operand, is rounded.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

import seanet_oracle
from seanet_oracle import RATIOS, _r, _wn, lstm_layer


def conv(x, sd, prefix, emulate, stride=1):
    """Causal Conv1d with reflect left padding k - stride (k - 1 at stride 1, the same as `seanet_oracle._conv`)."""
    w, b = _wn(sd, prefix, x.dtype)
    xp = seanet_oracle.reflect_pad_left(_r(x, emulate), w.shape[-1] - stride)
    return F.conv1d(xp, _r(w, emulate), b, stride=stride)


@torch.no_grad()
def encode(sd, audio: torch.Tensor, dtype=torch.float64, emulate_bf16: bool = False) -> torch.Tensor:
    """audio (B, T), T % 320 == 0 -> frames (B, T / 320, 128) token-major in `dtype`."""
    e = emulate_bf16
    x = conv(audio.to(dtype)[:, None], sd, "layers.0.conv", False)
    for si, s in enumerate(reversed(RATIOS)):
        i = 1 + 3 * si
        x = seanet_oracle.resnet_block(x, sd, f"layers.{i}", e and si > 0)
        x = conv(F.elu(x), sd, f"layers.{i + 2}.conv", e, stride=s)
    xt = x.transpose(1, 2)
    y = xt
    for l in range(2):
        y = lstm_layer(y, *(sd[f"layers.13.lstm.{n}_l{l}"].to(dtype) for n in ("weight_ih", "weight_hh", "bias_ih",
                                                                              "bias_hh")), emulate=e)
    x = (y + xt).transpose(1, 2)
    return conv(F.elu(x), sd, "layers.15.conv", e).transpose(1, 2)
