"""Torch-CPU port of the denoiser oracle — TEST / BASELINE INFRASTRUCTURE, NOT PRODUCT CODE.

Same restatement of `Model.forward` (ns2.py:929-1000) as `denoiser_oracle.py`, expressed with the PyTorch CPU ops
the reference itself calls (F.linear, F.conv1d, F.scaled_dot_product_attention, F.gelu ...), so that it runs on
all host cores through MKL/oneDNN exactly like the reference's own CPU path.  It exists for `bench.py`'s
`cpu_baseline` / `--impl reference` legs (the numpy oracle is the parity checker; numpy's BLAS use leaves most cores
idle and would understate the reference).  `tests/test_oracle_cpu.py` pins it to the same goldens, its autograd
(`model_forward_autograd` in float64) to the reference's fp64 gradients; run on the GPU in float64 it is the reference
of the hand-written backward at the benchmarked dims (tests/test_denoiser_backward_fp64_gpu.py).
Only tests/ and bench.py's CPU legs may import this module.
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch
import torch.nn.functional as F

from .denoiser_oracle import ModelConfig  # noqa: F401  (same config object)

Params = Dict[str, torch.Tensor]


def causal_conv1d(x, w, b, dilation=1):
    """CausalConv1d.forward, ns2.py:593-595 (x channel-first)."""
    pad = dilation * (w.shape[-1] - 1)
    return F.conv1d(F.pad(x, (pad, 0)), w, b, dilation=dilation)


def rmsnorm(x, gamma=None, film=None):
    """RMSNorm.forward, ns2.py:736-746."""
    dim = x.shape[-1]
    out = F.normalize(x, dim=-1) * (dim ** 0.5)
    if gamma is not None:
        out = out * gamma
    if film is None:
        return out
    return out * film[:, None, :dim] + film[:, None, dim:]


def attention(P, prefix, x, heads, context=None, include_queries=False):
    """Attention.forward ns2.py:1055-1069 + Attend (attend.py:102-108: SDPA, no mask, non-causal)."""
    ctx = x if context is None else context
    if context is not None and include_queries:
        ctx = torch.cat((x, ctx), dim=-2)
    q = F.linear(x, P[prefix + "to_q.weight"])
    k, v = F.linear(ctx, P[prefix + "to_kv.weight"]).chunk(2, dim=-1)
    sp = lambda t: t.reshape(t.shape[0], t.shape[1], heads, -1).transpose(1, 2)
    o = F.scaled_dot_product_attention(sp(q), sp(k), sp(v))
    o = o.transpose(1, 2).reshape(x.shape[0], x.shape[1], -1)
    return F.linear(o, P[prefix + "to_out.weight"])


def feedforward(P, prefix, x, causal_conv):
    """FeedForward, ns2.py:1009-1025."""
    h = F.linear(x, P[prefix + "0.weight"], P[prefix + "0.bias"])
    val, gate = h.chunk(2, dim=-1)
    h = F.gelu(gate) * val
    if causal_conv:
        h = causal_conv1d(h.transpose(1, 2), P[prefix + "2.1.weight"], P[prefix + "2.1.bias"]).transpose(1, 2)
        last = "3."
    else:
        last = "2."
    return F.linear(h, P[prefix + last + "weight"], P[prefix + last + "bias"])


def wavenet(P, cfg, x, t, dilations=None):
    """Wavenet / WavenetStack / WavenetResBlock, ns2.py:597-725.  `dilations`: optional (stacks, layers) table that
    replaces the reference's 2**i."""
    x = causal_conv1d(x, P["wavenet.init_conv.weight"], P["wavenet.init_conv.bias"])
    inputs = [x] * cfg.wavenet_layers
    skips = None
    dim = x.shape[1]
    for s in range(cfg.wavenet_stacks):
        has_skip = s == cfg.wavenet_stacks - 1
        residuals, skips = [], []
        for i in range(cfg.wavenet_layers):
            pre = f"wavenet.stacks.{s}.blocks.{i}."
            tt = F.linear(t, P[pre + "to_time_cond.weight"], P[pre + "to_time_cond.bias"])
            g, b = tt[:, :dim, None], tt[:, dim:, None]
            xi = inputs[i]
            res = causal_conv1d(xi, P[pre + "res_conv.weight"], P[pre + "res_conv.bias"])
            y = causal_conv1d(xi, P[pre + "conv.weight"], P[pre + "conv.bias"],
                              2 ** i if dilations is None else dilations[s][i])
            y = y * g + b
            y = y.tanh() * y.sigmoid() + res
            residuals.append(y)
            skips.append(causal_conv1d(y, P[pre + "skip_conv.weight"], P[pre + "skip_conv.bias"]) if has_skip else None)
        inputs = residuals
    return causal_conv1d(torch.stack(skips).sum(dim=0), P["wavenet.final_conv.weight"], P["wavenet.final_conv.bias"])


def perceiver_resampler(P, cfg, prompt):
    """PerceiverResampler.forward, ns2.py:568-579."""
    pre = "perceiver_resampler."
    x = prompt
    if pre + "proj_context.weight" in P:
        x = F.linear(x, P[pre + "proj_context.weight"], P[pre + "proj_context.bias"])
    lat = P[pre + "latents"][None].expand(x.shape[0], -1, -1)
    for i in range(cfg.resampler_depth):
        lat = attention(P, f"{pre}layers.{i}.0.", lat, cfg.heads, context=x, include_queries=True) + lat
        lat = feedforward(P, f"{pre}layers.{i}.1.", lat, causal_conv=False) + lat
    return rmsnorm(lat, gamma=P[pre + "norm.gamma"])


def transformer(P, cfg, x, t, context=None):
    """ConditionableTransformer.forward, ns2.py:786-809."""
    for l in range(cfg.depth):
        pre = f"transformer.layers.{l}."
        film = F.linear(t, P[pre + "0.to_gamma_beta.weight"], P[pre + "0.to_gamma_beta.bias"])
        x = attention(P, pre + "1.", rmsnorm(x, film=film), cfg.heads) + x
        if cfg.condition_on_prompt:
            film = F.linear(t, P[pre + "2.to_gamma_beta.weight"], P[pre + "2.to_gamma_beta.bias"])
            x = attention(P, pre + "3.", rmsnorm(x, film=film), cfg.heads, context=context) + x
        film = F.linear(t, P[pre + "4.to_gamma_beta.weight"], P[pre + "4.to_gamma_beta.bias"])
        x = feedforward(P, pre + "5.", rmsnorm(x, film=film), causal_conv=True) + x
    return F.linear(rmsnorm(x, gamma=P["transformer.to_pred.0.gamma"]), P["transformer.to_pred.1.weight"])


@torch.no_grad()
def model_forward(P: Params, cfg, x, times, prompt=None, cond=None, drop_prompt=None, drop_cond=None):
    """Model.forward, ns2.py:929-1000 (explicit CFG drop masks, None = keep everything), without autograd."""
    return model_forward_autograd(P, cfg, x, times, prompt, cond, drop_prompt, drop_cond)


def model_forward_autograd(P: Params, cfg, x, times, prompt=None, cond=None, drop_prompt=None, drop_cond=None,
                           dilations=None):
    """`model_forward` with autograd left as the caller has it: gradients reach every tensor of P, prompt and cond
    that requires them, so that the port in float64 is a reference for the denoiser's backward.  Runs on the device
    of `x`.  `dilations`: optional (stacks, layers) table of Wavenet dilations instead of the reference's 2**i, for
    building a deliberately wrong reference."""
    B, N, D = x.shape
    xt = times[:, None]
    freqs = xt * P["to_time_cond.0.weights"][None] * 2 * math.pi
    t = torch.cat((xt, freqs.sin(), freqs.cos()), dim=-1)
    t = F.silu(F.linear(t, P["to_time_cond.1.weight"], P["to_time_cond.1.bias"]))
    c = None
    if cfg.condition_on_prompt:
        dp = torch.zeros(B, dtype=torch.bool, device=x.device) if drop_prompt is None else drop_prompt
        dc = torch.zeros(B, dtype=torch.bool, device=x.device) if drop_cond is None else drop_cond
        pc = F.silu(F.linear(prompt.mean(dim=1), P["to_prompt_cond.1.weight"], P["to_prompt_cond.1.bias"]))
        pc = torch.where(dp[:, None], P["null_prompt_cond"][None], pc)
        t = torch.cat((t, pc), dim=-1)
        c = torch.where(dp[:, None, None], P["null_prompt_tokens"][None], perceiver_resampler(P, cfg, prompt))
    xc = x.transpose(1, 2)
    if cfg.condition_on_prompt:
        cp = F.conv1d(cond, P["cond_to_model_dim.weight"], P["cond_to_model_dim.bias"])
        cp = torch.where(dc[:, None, None], P["null_cond"][None], cp)
        L = cp.shape[-1]
        cp = cp[..., :N] if L >= N else F.pad(cp, (0, N - L))
        xc = xc + cp
    xc = wavenet(P, cfg, xc, t, dilations)
    return transformer(P, cfg, xc.transpose(1, 2), t, context=c)
