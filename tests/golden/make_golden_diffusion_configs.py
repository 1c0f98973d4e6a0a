#!/usr/bin/env python
"""Generate diffusion_configs.npz from the REFERENCE implementation: its own `NaturalSpeech2` (ns2.py:1160-1684) on
CPU at the constructor configurations of tests/test_diffusion_configs_fp64_gpu.py that it can run, i.e. the linear and
sigmoid schedules (its cosine schedule raises on tensors, SURVEY T12).

Per configuration:
  <name>::loss               the training loss on seeded latents with the two draws of ns2.py:1621,1625 injected by
                             seeding torch's CPU generator (as make_golden.diffusion_goldens does)
  <name>::pred               the model output inside that loss, captured by a forward hook
  <name>::coef<T>            (T, 4) per-step (alpha, sigma, alpha_next, sigma_next) that ddim_sample builds
                             (ns2.py:1396-1402), for T in COEF_STEPS; every sample of the batch gets the same values
  <name>::x<T>, ::v<T>       a DDIM run at T in SAMPLE_STEPS: x (T+1, B, N, D) = every latent from the initial noise to
                             the final sample, v (T, B, N, D) = every model output, captured by wrapping
                             `forward_with_cond_scale`

The model is make_golden.CASES["uncond_small"] with the param_fill weights (seed 1234), in fp32 as the reference trains
and samples.  Latents and draws are regenerated from seeds by `loss_inputs`; only the outputs are stored.

    python tests/golden/make_golden_diffusion_configs.py
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

DIFFUSION_CONFIGS = {
    # name: NaturalSpeech2 keyword arguments
    "sig_v": dict(),
    "sig_kw_eps": dict(schedule_kwargs=dict(start=-2, end=4, tau=0.7), objective="eps"),
    "sig_x0_off": dict(objective="x0", min_snr_loss_weight=False),
    "lin_v_half": dict(noise_schedule="linear", scale=0.5),
    "lin_eps_off": dict(noise_schedule="linear", schedule_kwargs=dict(clip_min=1e-5), objective="eps",
                        min_snr_loss_weight=False, rvq_cross_entropy_loss_weight=0.5),
    "lin_x0_g1": dict(noise_schedule="linear", objective="x0", scale=0.8, min_snr_gamma=1),
    "cos_v": dict(noise_schedule="cosine"),
    "cos_tau075": dict(noise_schedule="cosine", schedule_kwargs=dict(tau=0.75), objective="eps", scale=0.7,
                       min_snr_gamma=3, rvq_cross_entropy_loss_weight=0.5),
    "cos_kw_x0": dict(noise_schedule="cosine", schedule_kwargs=dict(start=0.2, end=0.9), objective="x0",
                      min_snr_loss_weight=False),
}
GOLDEN_CONFIGS = [n for n, kw in DIFFUSION_CONFIGS.items() if kw.get("noise_schedule") != "cosine"]
SAMPLE_STEPS = (1, 2, 7)
COEF_STEPS = (1, 2, 7, 1000)
LOSS_SHAPE = (3, 4, 128)      # (B, N, D) of the loss
SAMPLE_SHAPE = (2, 1, 128)    # of the DDIM runs
LATENT_SEED, DRAW_SEED, SAMPLE_SEED = 61, 62, 63


def loss_inputs():
    """(latents (B, N, D), times (B,), noise (B, N, D)) of the loss, all f32: the draws are those of ns2.py:1621,1625
    after torch.manual_seed(DRAW_SEED)."""
    latents = seeded(LOSS_SHAPE, LATENT_SEED)
    torch.manual_seed(DRAW_SEED)
    times = torch.zeros((LOSS_SHAPE[0],)).float().uniform_(0, 1.)
    noise = torch.randn_like(latents)
    return latents, times, noise


def main():
    from golden.make_golden import CASES, import_reference
    ns2 = import_reference()
    kwargs = CASES["uncond_small"][0]
    model = ns2.Model(**kwargs).eval()
    fill_module(model, seed=1234)
    latents, times, noise = loss_inputs()
    out = {}
    for name in GOLDEN_CONFIGS:
        kw = DIFFUSION_CONFIGS[name]
        # ---- the loss, with the draws injected by seeding ----
        diff = ns2.NaturalSpeech2(model=model, target_sample_hz=24000, timesteps=4, **kw)
        preds = []
        hook = model.register_forward_hook(lambda m, a, o: preds.append(o.detach().clone()))
        torch.manual_seed(DRAW_SEED)
        with torch.no_grad():
            loss = diff(latents)
        hook.remove()
        out[f"{name}::loss"] = np.array(loss.item(), dtype=np.float32)
        out[f"{name}::pred"] = preds[0].numpy()
        # ---- the per-step coefficients ddim_sample builds, recorded from gamma_to_alpha_sigma's two calls ----
        for T in COEF_STEPS:
            diff = ns2.NaturalSpeech2(model=model, target_sample_hz=24000, timesteps=T, **kw)
            recorded, xs, vs = [], [], []
            real = ns2.gamma_to_alpha_sigma

            def record(gamma, scale=1):
                a, s = real(gamma, scale)
                recorded.append((a.reshape(-1).clone(), s.reshape(-1).clone()))
                return a, s

            def model_output(audio, times, **k):
                xs.append(audio.clone())
                v = type(model).forward_with_cond_scale(model, audio, times, **k) if T in SAMPLE_STEPS \
                    else torch.zeros_like(audio)
                vs.append(v.clone())
                return v

            model.forward_with_cond_scale = model_output
            ns2.gamma_to_alpha_sigma = record
            torch.manual_seed(SAMPLE_SEED)
            try:
                with torch.no_grad():
                    final = diff.ddim_sample(SAMPLE_SHAPE)
            finally:
                ns2.gamma_to_alpha_sigma = real
                del model.forward_with_cond_scale
            assert len(recorded) == 2 * T
            coef = torch.stack([torch.stack((*recorded[2 * i], *recorded[2 * i + 1])) for i in range(T)])  # (T, 4, B)
            assert bool((coef == coef[:, :, :1]).all())
            out[f"{name}::coef{T}"] = coef[:, :, 0].numpy()
            if T in SAMPLE_STEPS:
                out[f"{name}::x{T}"] = torch.stack(xs + [final]).numpy()
                out[f"{name}::v{T}"] = torch.stack(vs).numpy()
        print(f"{name}: loss={loss.item():.6f} final |x| max T=7 {float(np.abs(out[f'{name}::x7'][-1]).max()):.3g}")
    np.savez_compressed(HERE / "diffusion_configs.npz", **out)


if __name__ == "__main__":
    main()
