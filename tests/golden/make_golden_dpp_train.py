#!/usr/bin/env python
"""Generate grads_dpp_train.npz from the REFERENCE implementation: its fp64 autograd through the duration / pitch
predictor's L1 losses, weighted as ns2.py:1587-1602 weighs them:

    loss = duration_loss_weight * l1(duration, duration_pred) + pitch_loss_weight * l1(pitch, pitch_pred)

Runs only where the reference source is readable (make_golden.py's import stubs and param_fill weights); the tests
regenerate every seeded input with `dpp_train_inputs` and read the head biases and targets from the fixture.

    python tests/golden/make_golden_dpp_train.py

Cases (eval mode: dropout off): dpp_small (dim 128, depth 2, heads 2), dpp_512 (dim 512, depth 1, the reference's
default heads and blocks) and dpp_table (a 50-token table in front, ids as input).  The fixture is built so that the
fp64 branch of every ReLU and every |.| is decided by at least MARGIN: both head biases are set so that every head
pre-activation is >= MARGIN, and each target is the fp64 prediction moved by MARGIN x (1 + u), u ~ U[0, 1), with a
random sign.  Stored: the biases, targets, predictions, both losses, every parameter's gradient norm, and d x (or the
token table's gradient) and d prompts whole.
"""
from __future__ import annotations

import sys
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent.parent))
sys.path.insert(0, str(HERE.parent))

from param_fill import fill_module, seeded, seeded_uniform  # noqa: E402

MARGIN = 1.0
WEIGHTS = (0.7, 0.3)   # duration_loss_weight, pitch_loss_weight
DPP_TRAIN_CASES = {
    # name: (ctor kwargs, B, T, Np)
    "dpp_small": (dict(dim=128, dim_hidden=128, depth=2, heads=2), 2, 37, 50),
    "dpp_512": (dict(dim=512, depth=1), 1, 40, 30),
    "dpp_table": (dict(num_phoneme_tokens=50, dim=128, dim_hidden=128, depth=1, heads=2), 2, 30, 20),
}
HEADS = ("to_duration_pred", "to_pitch_pred")


def dpp_train_inputs(name):
    """(x, prompts): x (B, T, D) phoneme encodings, or (B, T) ids in [0, 50) for the token-table case."""
    kwargs, B, T, Np = DPP_TRAIN_CASES[name]
    D = kwargs.get("dim_hidden", 512)
    if "num_phoneme_tokens" in kwargs:
        x = torch.randint(0, kwargs["num_phoneme_tokens"], (B, T), generator=torch.Generator().manual_seed(81))
    else:
        x = seeded((B, T, D), 82)
    return x, seeded((B, Np, D), 83)


def main():
    from golden.make_golden import import_reference
    ns2 = import_reference()
    out = {}
    for name, (kwargs, B, T, Np) in DPP_TRAIN_CASES.items():
        torch.manual_seed(0)
        m = ns2.DurationPitchPredictor(**kwargs)
        fill_module(m, seed=1234)
        m = m.double().eval()
        x, prompts = dpp_train_inputs(name)
        x = x if x.dtype == torch.int64 else x.double()
        prompts = prompts.double()
        # head pre-activations without the bias: bias 1e3 keeps every row on the linear side of the ReLU
        with torch.no_grad():
            for h in HEADS:
                getattr(m, h).to_pred[0].bias.fill_(1e3)
            pre = [p - 1e3 for p in m(x, prompts)]
            biases = [float(MARGIN - p.min()) for p in pre]            # every pre-activation >= MARGIN
            for h, b in zip(HEADS, biases):
                getattr(m, h).to_pred[0].bias.fill_(b)
            preds = m(x, prompts)
        targets = []
        for i, p in enumerate(preds):
            u = seeded_uniform(p.shape, 90 + i).double()
            sign = torch.where(seeded_uniform(p.shape, 92 + i) < 0.5, -1.0, 1.0).double()
            targets.append(p + sign * MARGIN * (1 + u))
        x_leaf = x if x.dtype == torch.int64 else x.clone().requires_grad_(True)
        pr_leaf = prompts.clone().requires_grad_(True)
        dur, pitch = m(x_leaf, pr_leaf)
        l_dur = torch.nn.functional.l1_loss(targets[0], dur)               # ns2.py:1587
        l_pitch = torch.nn.functional.l1_loss(targets[1], pitch)           # ns2.py:1589-1590
        loss = WEIGHTS[0] * l_dur + WEIGHTS[1] * l_pitch                   # ns2.py:1600-1601
        loss.backward()
        names = [n for n, _ in m.named_parameters()]
        out[f"{name}::names"] = np.array(names)
        out[f"{name}::norms"] = np.array([p.grad.norm().item() if p.grad is not None else 0.0
                                          for _, p in m.named_parameters()])
        out[f"{name}::biases"] = np.array(biases)
        out[f"{name}::targets"] = torch.stack(targets).numpy()
        out[f"{name}::preds"] = torch.stack(preds).numpy()
        out[f"{name}::losses"] = np.array([l_dur.item(), l_pitch.item(), loss.item()])
        if x.dtype == torch.int64:
            out[f"{name}::d_table"] = m.phoneme_token_emb.weight.grad.numpy().astype(np.float32)
        else:
            out[f"{name}::d_x"] = x_leaf.grad.numpy().astype(np.float32)
        out[f"{name}::d_prompts"] = pr_leaf.grad.numpy().astype(np.float32)
        print(f"dpp_train[{name}]: loss={loss.item():.6f} (duration {l_dur.item():.4f}, pitch {l_pitch.item():.4f}) "
              f"biases={biases} params={len(names)} min|pre|={min(float((p + b).min()) for p, b in zip(pre, biases)):.3f}")
    out["weights"] = np.array(WEIGHTS)
    out["margin"] = np.array(MARGIN)
    np.savez_compressed(HERE / "grads_dpp_train.npz", **out)


if __name__ == "__main__":
    main()
