#!/usr/bin/env python
"""Generate grads_cond_train.npz from the REFERENCE implementation: its fp64 autograd through the conditioning front
end of conditional training (ns2.py:1538-1583, 1627-1666, 1886).

Runs only where the reference source is readable (see make_golden.py, whose import stubs and model cases it reuses);
the GPU tests read the committed fixture and regenerate every seeded input with the functions below.

    python tests/golden/make_golden_cond_train.py

Cases (all modules in eval mode: dropout off; cond_drop_prob = 0):
  den_<case>   d loss / d prompt and d loss / d cond of the denoiser alone, for make_golden's cond_small
               (dim_prompt != dim) and cond_samedim (dim_prompt == dim, Lc > N: cond is curtailed)
  e2e_small    SpeechPromptEncoder -> Model(prompt=...); PhonemeEncoder + nn.Embedding pitch table ->
               average_over_durations -> expand_encodings(generate_mask_from_repeats) -> Model(cond=...)
  e2e_wide     the same with the reference's default prompt-encoder widths (eight k=9 convs up to 2048 channels)
  avg_*        utils.average_over_durations on fp32 values (the CPU restatement test)
Stored: losses, every parameter's gradient norm, a few small whole gradients, d prompt in full and d cond on a frame
subsample (fp32), plus the norms of both.
"""
from __future__ import annotations

import sys
import types
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent.parent))
sys.path.insert(0, str(HERE.parent))

from param_fill import fill_module, seeded, seeded_uniform  # noqa: E402

COND_TRAIN_CASES = {
    # (denoiser kwargs, prompt-encoder kwargs, phoneme-encoder kwargs, pitch-table shape, B, N latent frames,
    #  Np prompt frames, T phonemes, L cond frames).  dim_prompt = prompt-encoder output = phoneme dim_hidden =
    # pitch-embedding width (ns2.py:1231-1236); L > N, so the denoiser curtails cond.
    "e2e_small": (dict(dim=128, depth=1, heads=2, wavenet_layers=2, wavenet_stacks=1, dim_prompt=256,
                       condition_on_prompt=True, resampler_depth=1, num_latents_m=16),
                  dict(dim_codebook=128, dims=(256,), depth=1, heads=2),
                  dict(num_tokens=30, dim=128, dim_hidden=256, depth=1, heads=2), (256, 256), 2, 96, 40, 12, 110),
    "e2e_wide": (dict(dim=128, depth=1, heads=2, wavenet_layers=2, wavenet_stacks=1, dim_prompt=512,
                      condition_on_prompt=True, resampler_depth=1, num_latents_m=16),
                 dict(dim_codebook=128, depth=1),
                 dict(num_tokens=30, dim=128, dim_hidden=512, depth=1, heads=2), (256, 512), 2, 64, 40, 9, 70),
}
COND_TRAIN_KEEP = {   # whole gradients stored per case (small ones; every parameter's norm is stored too)
    "e2e_small": ("prompt_enc.conv.1.bias", "prompt_enc.transformer.layers.0.0.gamma", "phoneme_enc.token_emb.weight",
                  "phoneme_enc.conv.1.bias", "phoneme_enc.transformer.layers.0.2.gamma", "pitch_emb.weight",
                  "model.cond_to_model_dim.bias", "model.perceiver_resampler.proj_context.bias"),
    "e2e_wide": ("prompt_enc.conv.5.bias", "prompt_enc.conv.9.bias", "prompt_enc.transformer.layers.0.2.gamma",
                 "phoneme_enc.token_emb.weight", "pitch_emb.weight"),
}
DEN_SEEDS = (61, 62, 63)   # latents, times, noise of the den_* cases


def cond_frames(Lc: int) -> np.ndarray:
    """Frames of d cond stored for the den_* cases: every 4th frame plus the last 8."""
    return np.array(sorted(set(range(0, Lc, 4)) | set(range(Lc - 8, Lc))), dtype=np.int64)


def den_inputs(B, N, dim):
    return seeded((B, N, dim), DEN_SEEDS[0]), seeded_uniform((B,), DEN_SEEDS[1]), seeded((B, N, dim), DEN_SEEDS[2])


def cond_train_inputs(case):
    """Seeded inputs of one end-to-end case: text padding (-1), zero-duration phonemes, sample 1 shorter than L."""
    mkw, skw, pkw, _, B, N, Np, T, L = COND_TRAIN_CASES[case]
    g = torch.Generator().manual_seed(51)
    text = torch.randint(0, pkw["num_tokens"], (B, T), generator=g)
    text[1, T - 3:] = -1
    dur = torch.randint(1, 2 * L // T, (B, T), generator=g)
    dur[0, 2] = 0
    dur[1, T - 3:] = 0
    dur[1, 4] = 0
    dur[0] = (dur[0].float() * L / dur[0].sum()).floor().long()           # sample 0 fills (almost) all L frames
    dur[1] = (dur[1].float() * (0.7 * L) / dur[1].sum()).floor().long()   # sample 1 ends well before L
    assert int(dur.sum(-1).max()) <= L
    pitch = torch.randint(60, 500, (B, 1, L), generator=g).float()        # integer Hz: exact prefix sums
    pitch[:, :, ::7] = 0.                                                  # unvoiced frames
    return dict(prompt=seeded((B, Np, skw["dim_codebook"]), 52), text=text, duration=dur, pitch=pitch,
                latents=seeded((B, N, mkw["dim"]), 53), times=seeded_uniform((B,), 54), noise=seeded((B, N, mkw["dim"]), 55))


def _diffusion_loss(ns2, model, latents, times, noise, **kw):
    """ns2.py:1621-1666 with the recorded draws (sigmoid schedule, objective v, min-SNR-5 weight)."""
    B = latents.shape[0]
    gamma = ns2.sigmoid_schedule(times)
    alpha, sigma = ns2.gamma_to_alpha_sigma(gamma[:, None, None], 1.)
    pred = model(alpha * latents + sigma * noise, times, **kw)
    loss = ((pred - (alpha * noise - sigma * latents)) ** 2).reshape(B, -1).mean(dim=1)
    snr = (alpha * alpha) / (sigma * sigma)
    return (loss * snr.clamp(max=5) / (snr + 1)).mean()


def main():
    from golden.make_golden import CASES, import_reference
    ns2 = import_reference()
    from naturalspeech2_pytorch.utils.utils import average_over_durations
    out = {}
    for case in ("cond_small", "cond_samedim"):
        kwargs, B, N, _, _ = CASES[case]
        zm = np.load(HERE / f"model_{case}.npz")
        model = ns2.Model(**kwargs)
        fill_module(model, seed=1234)
        model = model.double().eval()
        prompt = torch.from_numpy(zm["in_prompt"]).double().requires_grad_(True)
        cond = torch.from_numpy(zm["in_cond"]).double().requires_grad_(True)
        latents, times, noise = den_inputs(B, N, kwargs["dim"])
        loss = _diffusion_loss(ns2, model, latents.double(), times.double(), noise.double(), prompt=prompt, cond=cond,
                               cond_drop_prob=0.)
        loss.backward()
        frames = cond_frames(cond.shape[-1])
        out.update({f"den_{case}::loss": np.array(loss.item()),
                    f"den_{case}::d_prompt": prompt.grad.numpy().astype(np.float32),
                    f"den_{case}::d_prompt_norm": np.array(prompt.grad.norm().item()),
                    f"den_{case}::d_cond_frames": cond.grad[..., frames].numpy().astype(np.float32),
                    f"den_{case}::d_cond_norm": np.array(cond.grad.norm().item())})
        print(f"cond_train[den_{case}]: loss={loss.item():.6f} |d prompt|={prompt.grad.norm():.4e} "
              f"|d cond|={cond.grad.norm():.4e}")
    for case, (mkw, skw, pkw, tshape, B, N, Np, T, L) in COND_TRAIN_CASES.items():
        torch.manual_seed(0)
        mods = {"model": ns2.Model(**mkw), "prompt_enc": ns2.SpeechPromptEncoder(**skw),
                "phoneme_enc": ns2.PhonemeEncoder(**pkw), "pitch_emb": torch.nn.Embedding(*tshape)}
        for name, m in mods.items():
            fill_module(m, seed=1234)
            mods[name] = m.double().eval()
        inp = cond_train_inputs(case)
        prompt_enc = mods["prompt_enc"](inp["prompt"].double())
        phoneme_enc = mods["phoneme_enc"](inp["text"])
        pitch = average_over_durations(inp["pitch"], inp["duration"])          # fp32 frame pitch, as in training
        aln = ns2.generate_mask_from_repeats(inp["duration"]).double()
        aln = torch.nn.functional.pad(aln, (0, L - aln.shape[-1]))            # aln_mask has L (mel) columns
        fake = types.SimpleNamespace(pitch_emb=mods["pitch_emb"])
        cond = ns2.NaturalSpeech2.expand_encodings(fake, phoneme_enc.transpose(1, 2), aln.unsqueeze(1), pitch)
        loss = _diffusion_loss(ns2, mods["model"], inp["latents"].double(), inp["times"].double(), inp["noise"].double(),
                               prompt=prompt_enc, cond=cond, cond_drop_prob=0.)
        loss.backward()
        names, norms = [], []
        for mname, m in mods.items():
            for n, p in m.named_parameters():
                g = p.grad if p.grad is not None else torch.zeros_like(p)
                names.append(f"{mname}.{n}")
                norms.append(g.norm().item())
                if f"{mname}.{n}" in COND_TRAIN_KEEP[case]:
                    out[f"{case}::grad::{mname}.{n}"] = g.numpy().astype(np.float32)
        out[f"{case}::names"] = np.array(names)
        out[f"{case}::norms"] = np.array(norms)
        out[f"{case}::loss"] = np.array(loss.item())
        out[f"{case}::coarse"] = ns2.f0_to_coarse(pitch)[:, 0].numpy().astype(np.int32)
        out[f"{case}::in_text"] = inp["text"].numpy()          # checks that the seeded inputs regenerate identically
        out[f"{case}::in_duration"] = inp["duration"].numpy()
        print(f"cond_train[{case}]: loss={loss.item():.6f} params={len(names)} "
              f"total grad norm={np.sqrt((np.array(norms) ** 2).sum()):.4f}")
    g = torch.Generator().manual_seed(71)
    vals = torch.rand(3, 2, 50, generator=g) * 400
    vals[vals < 120] = 0.                                   # zeros are skipped by the average
    durs = torch.randint(0, 9, (3, 8), generator=g)
    durs[2, 3:6] = 0
    out.update(avg_values=vals.numpy(), avg_durs=durs.numpy(), avg_out=average_over_durations(vals, durs).numpy(),
               avg_out_float_durs=average_over_durations(vals[:, :1], durs.float()).numpy())
    np.savez_compressed(HERE / "grads_cond_train.npz", **out)


if __name__ == "__main__":
    main()
