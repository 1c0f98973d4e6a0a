#!/usr/bin/env python
"""Generate encoder_configs.npz from the REFERENCE implementation: float64 outputs of its SpeechPromptEncoder,
PhonemeEncoder and DurationPitchPredictor at the constructor knobs the default-dims fixtures (encoders.npz) never
reach: conv kernel sizes 1, 3, 5, 7, 11 and 12, GroupNorm groups of 16, 48, 80 and 128 channels, attention widths
heads x 64 != dim, 64- and 192-channel convs, ResnetBlocks of 1 and 3 Blocks, and a token table at width 256.  The
configurations are those of tests/test_encoder_configs_fp64_gpu.py at small sequence lengths.

Runs only where the reference source is readable (make_golden.py's import stubs and param_fill weights, seed 1234);
inputs are regenerated from seeds by `encoder_config_inputs`, and only the outputs are stored.

    python tests/golden/make_golden_encoder_configs.py

The reference annotates SpeechPromptEncoder's `dims` as Tuple[int], which beartype reads as a 1-tuple although the
default is an 8-tuple; multi-conv stacks are built through the undecorated __init__.  Both predictor heads get the
bias HEAD_BIAS, so that every row is on the linear side of the ReLU and the outputs pin the trunks.
"""
from __future__ import annotations

import sys
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent.parent))
sys.path.insert(0, str(HERE.parent))

from param_fill import fill_module, seeded  # noqa: E402

HEAD_BIAS = 10.0
HEADS = ("to_duration_pred", "to_pitch_pred")
ENCODER_CONFIG_CASES = {
    # name: (class name, ctor kwargs, input spec: (B, N) or (B, T, Np) for the predictor)
    "spe_k3_narrow": ("SpeechPromptEncoder",
                      dict(dim_codebook=64, dims=(64, 192, 128), kernel_size=3, padding=1, depth=2, heads=3), (1, 9)),
    "spe_k1_wide": ("SpeechPromptEncoder",
                    dict(dim_codebook=128, dims=(1024,), kernel_size=1, padding=0, depth=1, heads=16), (1, 3)),
    "spe_k11": ("SpeechPromptEncoder",
                dict(dim_codebook=128, dims=(256, 384), kernel_size=11, padding=5, depth=1, heads=4), (1, 7)),
    "phon_d64": ("PhonemeEncoder", dict(num_tokens=30, dim=64, dim_hidden=384, kernel_size=3, depth=2, heads=5), (1, 8)),
    "phon_k12": ("PhonemeEncoder", dict(num_tokens=30, dim=256, dim_hidden=256, kernel_size=12, depth=1, heads=2),
                 (1, 14)),
    "phon_k1": ("PhonemeEncoder", dict(num_tokens=30, dim=512, dim_hidden=1024, kernel_size=1, depth=1, heads=8), (1, 3)),
    "dpp_128": ("DurationPitchPredictor", dict(dim=128, dim_hidden=128, kernel_size=5, depth=2, heads=2,
                                               num_convs_per_resnet_block=1, num_convolutions_per_block=2), (2, 6, 3)),
    "dpp_384": ("DurationPitchPredictor", dict(dim=384, dim_hidden=384, kernel_size=7, depth=1, heads=3,
                                               num_convs_per_resnet_block=3, num_convolutions_per_block=1), (1, 5, 4)),
    "dpp_640": ("DurationPitchPredictor", dict(dim=640, dim_hidden=640, kernel_size=1, depth=1, heads=10), (1, 4, 3)),
    "dpp_1024": ("DurationPitchPredictor", dict(dim=1024, dim_hidden=1024, kernel_size=3, depth=1, heads=16), (1, 3, 2)),
    "dpp_table": ("DurationPitchPredictor", dict(num_phoneme_tokens=60, dim=256, dim_hidden=256, kernel_size=3, depth=2),
                  (1, 6, 3)),
}


def encoder_config_inputs(name):
    """The case's inputs: prompt frames (B, N, dim_codebook); ids (B, T) with a -1 tail; or (phoneme encodings (B, T, D)
    or ids, encoded prompts (B, Np, D)) for the predictor."""
    cls, kwargs, spec = ENCODER_CONFIG_CASES[name]
    g = torch.Generator().manual_seed(41)
    if cls == "DurationPitchPredictor":
        B, T, Np = spec
        D = kwargs["dim_hidden"]
        if "num_phoneme_tokens" in kwargs:
            x = torch.randint(0, kwargs["num_phoneme_tokens"], (B, T), generator=g)
        else:
            x = seeded((B, T, D), 42)
        return x, seeded((B, Np, D), 43)
    B, N = spec
    if cls == "PhonemeEncoder":
        ids = torch.randint(0, kwargs["num_tokens"], (B, N), generator=g)
        ids[:, N - 2:] = -1                                  # padding (ns2.py:279-280)
        return ids
    return seeded((B, N, kwargs["dim_codebook"]), 44)


def build(ns2, cls, kwargs):
    """The reference module in float64 with the param_fill weights (and HEAD_BIAS on the predictor's heads)."""
    c = getattr(ns2, cls)
    torch.manual_seed(0)
    if cls == "SpeechPromptEncoder":   # past the Tuple[int] annotation (see the module docstring)
        m = c.__new__(c)
        c.__init__.__wrapped__(m, kwargs["dim_codebook"], **{k: v for k, v in kwargs.items() if k != "dim_codebook"})
    else:
        m = c(**kwargs)
    fill_module(m, seed=1234)
    m = m.double().eval()
    if cls == "DurationPitchPredictor":
        with torch.no_grad():
            for h in HEADS:
                getattr(m, h).to_pred[0].bias.fill_(HEAD_BIAS)
    return m


def main():
    from golden.make_golden import import_reference
    ns2 = import_reference()
    out = {"head_bias": np.array(HEAD_BIAS)}
    for name, (cls, kwargs, _) in ENCODER_CONFIG_CASES.items():
        m = build(ns2, cls, kwargs)
        x = encoder_config_inputs(name)
        with torch.no_grad():
            if cls == "DurationPitchPredictor":
                x, prompts = x
                y = torch.stack(m(x if x.dtype == torch.int64 else x.double(), prompts.double()))
            else:
                y = m(x if x.dtype == torch.int64 else x.double())
        out[f"{name}_fp64"] = y.numpy()
        out[f"{name}_keys"] = np.array(repr([(k, tuple(v.shape)) for k, v in m.state_dict().items()]))
        print(f"{name}: out {tuple(y.shape)} mean={float(y.mean()):.3f} std={float(y.std()):.3f} "
              f"min={float(y.min()):.3f}")
    np.savez_compressed(HERE / "encoder_configs.npz", **out)


if __name__ == "__main__":
    main()
