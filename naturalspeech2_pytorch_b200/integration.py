"""Switching an existing reference object over to the sm_90a path (INTEGRATION.md).

`accelerate(ref_model)` reads the constructor arguments back out of a `naturalspeech2_pytorch.Model` instance
(ns2.py:811-905 stores them as attributes / module shapes), builds the H100 `Model` with the same configuration,
loads the reference's state_dict (the parameter names and shapes are identical, SURVEY Appendix B) and returns it.
`patch_reference(ref_model)` additionally rebinds `forward` / `forward_with_cond_scale` of the reference object, so
that code holding the reference instance (e.g. a reference `NaturalSpeech2` wrapper) runs the CUDA kernels unchanged.
"""
from __future__ import annotations

import types

import torch
from torch import nn

from .model import Model


def infer_model_kwargs(ref: nn.Module) -> dict:
    """Constructor arguments of a reference `Model` instance, recovered from its attributes and parameter shapes."""
    sd = ref.state_dict()
    dim = int(ref.dim)
    layers = ref.transformer.layers
    depth = len(layers)
    attn = layers[0][1]
    heads = int(attn.heads)
    dim_head = sd["transformer.layers.0.1.to_q.weight"].shape[0] // heads
    ff_inner = sd["transformer.layers.0.5.0.weight"].shape[0] // 2
    # inner = int(dim * mult * 2 / 3)  =>  smallest mult reproducing the stored width
    ff_mult = next(m for m in range(1, 65) if int(dim * m * 2 / 3) == ff_inner)
    stacks = ref.wavenet.stacks
    condition_on_prompt = bool(ref.condition_on_prompt)
    dim_time = sd["to_time_cond.1.weight"].shape[0]
    kwargs = dict(dim=dim, depth=depth, dim_head=dim_head, heads=heads, ff_mult=ff_mult,
                  wavenet_layers=len(stacks[0].blocks), wavenet_stacks=len(stacks),
                  dim_cond_mult=dim_time // dim, cond_drop_prob=float(ref.cond_drop_prob),
                  condition_on_prompt=condition_on_prompt)
    if condition_on_prompt:
        kwargs["dim_prompt"] = sd["to_prompt_cond.1.weight"].shape[1]
        kwargs["num_latents_m"] = sd["perceiver_resampler.latents"].shape[0]
        kwargs["resampler_depth"] = len(ref.perceiver_resampler.layers)
    return kwargs


def accelerate(ref: nn.Module, device=None) -> Model:
    """H100 `Model` with the configuration and the weights of the reference `Model` instance `ref`."""
    fast = Model(**infer_model_kwargs(ref))
    fast.load_state_dict(ref.state_dict())
    if device is None:
        device = next(ref.parameters()).device
    return fast.to(device).eval()


def patch_reference(ref: nn.Module, device="cuda") -> Model:
    """Rebind `ref.forward` / `ref.forward_with_cond_scale` to the H100 model built from `ref` (returned).  The
    reference object keeps its parameters; call `fast.load_state_dict(ref.state_dict())` again after updating them."""
    fast = accelerate(ref, device=device)

    def forward(self, x, times, prompt=None, prompt_mask=None, cond=None, cond_drop_prob=None):
        return fast.forward(x, times, prompt=prompt, prompt_mask=prompt_mask, cond=cond, cond_drop_prob=cond_drop_prob)

    def forward_with_cond_scale(self, *args, cond_scale=1., **kwargs):
        return fast.forward_with_cond_scale(*args, cond_scale=cond_scale, **kwargs)

    ref.forward = types.MethodType(forward, ref)
    ref.forward_with_cond_scale = types.MethodType(forward_with_cond_scale, ref)
    return fast
