"""Shared test helpers: golden loading, model construction with deterministic weights."""
from __future__ import annotations

import ast
from pathlib import Path

import numpy as np
import torch

from param_fill import fill_module

GOLDEN = Path(__file__).resolve().parent / "golden"
MODEL_CASES = ["uncond_small", "cond_small", "cond_samedim", "readme_uncond", "cond_ff2"]
# slices of the benchmarked configurations (dim 512, heads 8, seq 1024, depth 2): inputs are regenerated from seeds,
# outputs are stored on a row subsample (see tests/golden/make_golden.py BIG_CASES)
BIG_MODEL_CASES = ["cfg2_slice", "cfg3_slice"]


def load_model_golden(name: str):
    z = np.load(GOLDEN / f"model_{name}.npz")
    kwargs = dict(ast.literal_eval(str(z["config"])))
    return z, kwargs, int(z["fill_seed"])


def golden_inputs(z, kwargs) -> dict:
    """{x, times[, prompt, cond]} as float32 CPU tensors: stored arrays, or regenerated from the generator's seeds."""
    from param_fill import seeded, seeded_uniform
    if "in_seeded" in z.files:
        shp = tuple(int(v) for v in z["in_shape_x"])
        out = {"x": seeded(shp, 11), "times": seeded_uniform((shp[0],), 12)}
        if kwargs.get("condition_on_prompt"):
            out["prompt"] = seeded(tuple(int(v) for v in z["in_shape_prompt"]), 13)
            out["cond"] = seeded(tuple(int(v) for v in z["in_shape_cond"]), 14)
        return out
    out = {"x": torch.from_numpy(z["in_x"]), "times": torch.from_numpy(z["in_times"])}
    if kwargs.get("condition_on_prompt"):
        out["prompt"] = torch.from_numpy(z["in_prompt"])
        out["cond"] = torch.from_numpy(z["in_cond"])
    return out


def golden_rows(z, out: np.ndarray) -> np.ndarray:
    """Restrict a full (B, N, D) output to the positions the fixture stores."""
    return out[:, z["rows"]] if "rows" in z.files else out


def build_model(kwargs: dict, seed: int, device="cpu"):
    """naturalspeech2_pytorch_b200.Model with the deterministic weights the goldens were generated with."""
    from naturalspeech2_pytorch_b200 import Model
    m = Model(**kwargs)
    fill_module(m, seed)
    return m.to(device).eval()


def numpy_params(model: torch.nn.Module):
    return {k: v.detach().cpu().numpy() for k, v in model.state_dict().items()}


def oracle_config(kwargs: dict):
    from oracle.denoiser_oracle import ModelConfig
    allowed = ModelConfig.__init__.__code__.co_varnames
    return ModelConfig(**{k: v for k, v in kwargs.items() if k in allowed})


def err_stats(got: np.ndarray, ref: np.ndarray):
    d = np.abs(np.asarray(got, dtype=np.float64) - np.asarray(ref, dtype=np.float64))
    return float(d.max()), float(np.sqrt((d ** 2).mean()))


def aligner_golden_cases():
    """(name, value, mask, reference path) of tests/golden/aligner_mas.npz; masks are rebuilt from the stored lengths
    exactly as Aligner.forward does (aligner.py:208-211)."""
    z = np.load(GOLDEN / "aligner_mas.npz")
    for name in sorted(k[:-6] for k in z.files if k.endswith("_value")):
        value = z[f"{name}_value"]
        b, t_x, t_y = value.shape
        xm = (np.arange(t_x)[None, :] < z[f"{name}_xlens"][:, None]).astype(np.float32)
        ym = (np.arange(t_y)[None, :] < z[f"{name}_ylens"][:, None]).astype(np.float32)
        yield name, value, xm[:, :, None] * ym[:, None, :], z[f"{name}_path"]


ENCODER_CASES = ["spe_small", "spe_long", "spe_full", "phon_small"]
DPP_CASES = ["dpp_small", "dpp_512"]


def encoder_case(name: str):
    """(class name, ctor kwargs, input tensor, fp64 reference output, reference autocast-bf16 output, key list)."""
    from golden.make_golden import ENCODER_CASES as SPEC
    z = np.load(GOLDEN / "encoders.npz")
    cls, kwargs, _ = SPEC[name]
    keys = ast.literal_eval(str(z[f"{name}_keys"]))
    return cls, dict(kwargs), torch.from_numpy(z[f"{name}_in"]), z[f"{name}_fp64"], z[f"{name}_bf16_autocast"], keys


def build_encoder(cls: str, kwargs: dict, seed: int = 1234, device="cpu"):
    from naturalspeech2_pytorch_b200 import encoders
    m = getattr(encoders, cls)(**kwargs)
    fill_module(m, seed)
    return m.to(device).eval()


def dpp_case(name: str):
    """(ctor kwargs, phoneme encodings, encoded prompts, fp64 reference (2, B, T), reference autocast-bf16, key list)."""
    from golden.make_golden import ENCODER_CASES as SPEC
    z = np.load(GOLDEN / "encoders.npz")
    _, kwargs, _ = SPEC[name]
    keys = ast.literal_eval(str(z[f"{name}_keys"]))
    return (dict(kwargs), torch.from_numpy(z[f"{name}_in"]), torch.from_numpy(z[f"{name}_prompts"]), z[f"{name}_fp64"],
            z[f"{name}_bf16_autocast"], keys)
