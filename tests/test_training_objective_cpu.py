"""CPU: the float64 composition of the whole training objective (test_training_objective_fp64_gpu.objective) against the
reference's own end-to-end goldens (tests/golden/grads_cond_train.npz, make_golden_cond_train.py): the reference's
SpeechPromptEncoder, PhonemeEncoder, pitch table, expand_encodings and Model under its diffusion loss, in fp64.  The
goldens have neither the duration / pitch predictor nor the RVQ cross-entropy, so both are off here (weights 0).  What
is left is the glue: which encoder output reaches which Model input, the alignment over L frames, the coarse pitch of
the per-phoneme pitch, q-sample and the min-SNR loss.  Matching the loss, every parameter's gradient norm and the stored
whole gradients pins that glue to the reference's."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F
from torch import nn

from helpers import GOLDEN
from oracle import encoders_oracle as eo
from param_fill import fill_module
from restatements import objective


@pytest.mark.parametrize("case", ["e2e_small", "e2e_wide"])
def test_composed_objective_reproduces_the_reference_goldens(case):
    from golden.make_golden_cond_train import COND_TRAIN_CASES, cond_train_inputs
    from naturalspeech2_pytorch_b200 import Model
    from naturalspeech2_pytorch_b200.diffusion import gamma_to_alpha_sigma, sigmoid_schedule
    from naturalspeech2_pytorch_b200.encoders import PhonemeEncoder, SpeechPromptEncoder, average_over_durations
    z = np.load(GOLDEN / "grads_cond_train.npz")
    mkw, skw, pkw, tshape, B, N, Np, T, L = COND_TRAIN_CASES[case]
    mods = {"model": Model(**mkw), "prompt_enc": SpeechPromptEncoder(**skw), "phoneme_enc": PhonemeEncoder(**pkw),
            "pitch_emb": nn.Embedding(*tshape)}
    for m in mods.values():
        fill_module(m, seed=1234)
    inp = cond_train_inputs(case)
    assert np.array_equal(inp["duration"].numpy(), z[f"{case}::in_duration"])
    ph_pitch = average_over_durations(inp["pitch"], inp["duration"])[:, 0]
    coarse = eo.f0_to_coarse(ph_pitch).long()
    np.testing.assert_array_equal(coarse.numpy(), z[f"{case}::coarse"])
    mask = eo.generate_mask_from_repeats(inp["duration"])
    # the reference's schedule on the float64 times (make_golden_cond_train._diffusion_loss): its start / end
    # sigmoids are fp32 0-d tensors, as in the wrapper's restatement
    alpha, sigma = gamma_to_alpha_sigma(sigmoid_schedule(inp["times"].double()))
    zeros = torch.zeros(B, dtype=torch.bool)
    c = dict(model_kwargs=mkw, heads=(mods["prompt_enc"].heads, mods["phoneme_enc"].heads, None),
             padding=mods["prompt_enc"].padding, prompt=inp["prompt"], text=inp["text"],
             mask=F.pad(mask, (0, L - mask.shape[-1])), onehot=F.one_hot(coarse, tshape[0]), audio=inp["latents"],
             noise=inp["noise"], times=inp["times"], alpha=alpha, sigma=sigma, drop=(zeros, zeros),
             cfg=dict(objective="v", min_snr_loss_weight=True, min_snr_gamma=5, ce_weight=0., weights=(0., 0.)))
    P = {f"{k}.{n}": p.detach().double().requires_grad_(True) for k, m in mods.items() for n, p in m.named_parameters()}
    out = objective(P, torch.float64, c)
    assert "duration_loss" not in out
    grads = dict(zip(P, torch.autograd.grad(out["loss"], list(P.values()), allow_unused=True)))
    loss, ref_loss = float(out["loss"].detach()), float(z[f"{case}::loss"])
    assert abs(loss - ref_loss) <= 1e-10 * abs(ref_loss), (loss, ref_loss)
    names, norms = list(z[f"{case}::names"]), z[f"{case}::norms"]
    assert set(names) <= set(P), sorted(set(names) - set(P))[:8]
    worst = (0.0, None)
    for n, ref in zip(names, norms):
        got = 0.0 if grads[n] is None else float(grads[n].norm())
        if ref == 0:
            assert got == 0, n
            continue
        worst = max(worst, (abs(got - ref) / ref, n))
    kept = [k for k in z.files if k.startswith(f"{case}::grad::")]
    worst_t = (0.0, None)
    for k in kept:
        n = k.split("::")[2]
        ref = torch.from_numpy(z[k]).double()
        worst_t = max(worst_t, (float((grads[n] - ref).norm() / ref.norm()), n))
    print(f"\n{case}: loss {loss:.12g} (reference {ref_loss:.12g}); {len(names)} gradient norms, worst {worst[0]:.1e} "
          f"({worst[1]}); {len(kept)} whole gradients, worst rel-L2 {worst_t[0]:.1e} ({worst_t[1]})")
    assert worst[0] <= 1e-9, worst
    assert len(kept) >= 5 and worst_t[0] <= 1e-6, worst_t      # the goldens store whole gradients in fp32
