#!/usr/bin/env python
"""Generate grads_rvq_ce.npz from the REFERENCE implementation: its fp64 autograd through the RVQ cross-entropy term of
the training loss (ns2.py:1670-1684, `codec.rq(x_start, codes)`).

Runs only where the reference source is readable (it reuses make_golden.py's import stubs, model cases and
param_fill weights); the GPU tests read the committed fixture and regenerate every seeded input with the functions
below.

    python tests/golden/make_golden_rvq_ce.py

The codec is a stub whose `rq` is tests/rvq_ce_restatement.residual_vq_ce, the fp64 restatement of vector-quantize-pytorch's
ResidualVQ.forward(x, indices=codes).  Its codebooks are seeded (Q=4, K=256); the latents are the stub codec's own
quantized embedding of seeded frames and `codes` its codes, as the reference gets both from `codec(raw audio)`
(ns2.py:1608-1611), with some targets set to -1.

Cases (weight 0.5, recorded times and noise):
  uncond_<objective>  make_golden's uncond_small denoiser for objectives v, eps and x0.  The reference's own
                      NaturalSpeech2.forward runs in fp64, so x_start and safe_div (ns2.py:1673-1680) are its code.
  cond_v              cond_small with precomputed prompt / cond requiring grad (cond_drop_prob = 0).  The reference's
                      conditional forward needs text and an aligner, so ns2.py:1621-1684 are replicated here, as
                      make_golden.gradient_goldens does.
Stored per case: the loss and the CE loss; every parameter's gradient norm of the full loss and of the CE term alone
(w * ce_loss); a few small whole gradients of both; d pred of the CE term on a frame subsample and its norm; for cond_v
the CE term's d prompt in full and d cond on a frame subsample.  times and noise are not stored: rvq_ce_draws
regenerates them.
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

RVQ_Q, RVQ_K = 4, 256
CB_SEED, FRAMES_SEED, DRAW_SEED = 81, 82, 91
CE_WEIGHT = 0.5
CE_KEEP = ("transformer.to_pred.0.gamma", "transformer.layers.1.5.3.bias", "wavenet.final_conv.bias",
           "wavenet.stacks.1.blocks.1.to_time_cond.bias", "to_time_cond.0.weights")


def ce_frames(N):
    """Frames of d pred / d cond stored: every 4th plus the last 3."""
    return np.array(sorted(set(range(0, N, 4)) | set(range(N - 3, N))), dtype=np.int64)


def rvq_ce_inputs(B, N, dim=128):
    """(codebooks (Q, K, dim) f32, latents (B, N, dim) f32 = the codec's quantized frames, codes (B, N, Q) int64)."""
    from oracle import rvq_oracle
    cb = seeded((RVQ_Q, RVQ_K, dim), CB_SEED)
    frames = seeded((B * N, dim), FRAMES_SEED)
    codes = rvq_oracle.encode(frames.numpy(), cb.numpy())
    latents = torch.from_numpy(rvq_oracle.decode(codes, cb.numpy())).view(B, N, dim)
    codes = torch.from_numpy(codes).view(B, N, RVQ_Q)
    codes[0, :9, 1] = -1               # ignored targets: a run at the start of one sample
    codes[1, 3::7, 3] = -1             # and scattered ones in the last stage
    return cb, latents, codes


def rvq_ce_draws(B, N, dim=128):
    """The two draws of ns2.py:1621 and 1625 under DRAW_SEED: times (B,) f32 and noise (B, N, dim) f64."""
    torch.manual_seed(DRAW_SEED)
    times = torch.zeros((B,)).float().uniform_(0, 1.)
    noise = torch.randn((B, N, dim), dtype=torch.float64)
    return times, noise


class _StubCodecMixin:
    """What NaturalSpeech2 reads from a codec (ns2.py:1212-1214, 1244-1246, 1682); `rq` is the fp64 restatement."""

    def __init__(self, codebooks):
        super().__init__()
        self.register_buffer("codebooks", codebooks.double())
        self.target_sample_hz, self.seq_len_multiple_of, self.codebook_dim = 24000, 320, codebooks.shape[-1]
        self.last_ce = None

    def rq(self, x, codes):
        from rvq_ce_restatement import residual_vq_ce
        quantized, ce, _ = residual_vq_ce(x, self.codebooks, codes)
        self.last_ce = ce
        return quantized, ce


def StubCodec(codebooks):
    """A _StubCodecMixin that passes the reference's type check (an audiolm_pytorch.EncodecWrapper, stubbed)."""
    base = sys.modules["audiolm_pytorch"].EncodecWrapper
    return type("StubCodec", (_StubCodecMixin, base), {})(codebooks)


def _store(out, prefix, model, loss, ce, pred, extra_inputs=()):
    """Full-loss and CE-term gradients of every parameter (norms + CE_KEEP tensors), d pred of the CE term."""
    params = [p for _, p in model.named_parameters()]
    ce_term = CE_WEIGHT * ce
    ce_grads = torch.autograd.grad(ce_term, params + [pred] + list(extra_inputs), retain_graph=True, allow_unused=True)
    loss.backward()
    names, norms, ce_norms = [], [], []
    for (n, p), g in zip(model.named_parameters(), ce_grads):
        g = torch.zeros_like(p) if g is None else g
        full = p.grad if p.grad is not None else torch.zeros_like(p)
        names.append(n)
        norms.append(full.norm().item())
        ce_norms.append(g.norm().item())
        if n in CE_KEEP:
            out[f"{prefix}::grad::{n}"] = full.numpy().astype(np.float32)
            out[f"{prefix}::cegrad::{n}"] = g.detach().numpy().astype(np.float32)
    out[f"{prefix}::names"] = np.array(names)
    out[f"{prefix}::norms"] = np.array(norms)
    out[f"{prefix}::ce_norms"] = np.array(ce_norms)
    out[f"{prefix}::loss"] = np.array(loss.item())
    out[f"{prefix}::ce_loss"] = np.array(ce.item())
    d_pred = ce_grads[len(params)].detach()
    out[f"{prefix}::d_pred_ce_frames"] = d_pred[:, ce_frames(d_pred.shape[1])].numpy().astype(np.float32)
    out[f"{prefix}::d_pred_ce_norm"] = np.array(d_pred.norm().item())
    print(f"rvq_ce[{prefix}]: loss={loss.item():.6f} ce={ce.item():.6f} |d pred ce|={ce_grads[len(params)].norm():.4e} "
          f"|ce grads|={np.sqrt((np.array(ce_norms) ** 2).sum()):.4e}")
    return ce_grads[len(params) + 1:]


def main():
    from golden.make_golden import CASES, import_reference
    ns2 = import_reference()
    out = {}
    kwargs, B, N, _, _ = CASES["uncond_small"]
    cb, latents, codes = rvq_ce_inputs(B, N, kwargs["dim"])
    for objective in ("v", "eps", "x0"):
        model = ns2.Model(**kwargs)
        fill_module(model, seed=1234)
        model = model.double()
        codec = StubCodec(cb)
        diff = ns2.NaturalSpeech2(model=model, codec=codec, timesteps=4, objective=objective,
                                  rvq_cross_entropy_loss_weight=CE_WEIGHT)
        preds = []
        hook = model.register_forward_hook(lambda m, i, o: preds.append(o))
        times, noise = rvq_ce_draws(B, N, kwargs["dim"])
        torch.manual_seed(DRAW_SEED)        # the reference's forward makes the same two draws
        loss = diff(latents.double(), codes=codes)
        hook.remove()
        _store(out, f"uncond_{objective}", model, loss, codec.last_ce, preds[0])
        out[f"uncond_{objective}::times"] = times.numpy()

    # conditional: ns2.py:1621-1684 replicated with precomputed prompt / cond (objective v, sigmoid schedule, min-SNR 5)
    kwargs, B, N, _, _ = CASES["cond_small"]
    zm = np.load(HERE / "model_cond_small.npz")
    model = ns2.Model(**kwargs)
    fill_module(model, seed=1234)
    model = model.double()
    cb, latents, codes = rvq_ce_inputs(B, N, kwargs["dim"])
    codec = StubCodec(cb)
    times, noise = rvq_ce_draws(B, N, kwargs["dim"])
    prompt = torch.from_numpy(zm["in_prompt"]).double().requires_grad_(True)
    cond = torch.from_numpy(zm["in_cond"]).double().requires_grad_(True)
    audio = latents.double()
    gamma = ns2.sigmoid_schedule(times)
    alpha, sigma = ns2.gamma_to_alpha_sigma(ns2.right_pad_dims_to(audio, gamma), 1.)
    pred = model(alpha * audio + sigma * noise, times, prompt=prompt, cond=cond, cond_drop_prob=0.)
    target = alpha * noise - sigma * audio
    loss = torch.nn.functional.mse_loss(pred, target, reduction="none").reshape(B, -1).mean(-1)
    snr = (alpha * alpha) / (sigma * sigma)
    loss = (loss * snr.clone().clamp_(max=5) / (snr + 1)).mean()
    x_start = alpha * audio - sigma * pred
    _, ce = codec.rq(x_start, codes)
    loss = loss + CE_WEIGHT * ce
    d_prompt, d_cond = _store(out, "cond_v", model, loss, ce, pred, (prompt, cond))
    out["cond_v::times"] = times.numpy()
    out["cond_v::d_prompt_ce"] = d_prompt.numpy().astype(np.float32)
    out["cond_v::d_cond_ce_frames"] = d_cond[..., ce_frames(d_cond.shape[-1])].numpy().astype(np.float32)
    out["cond_v::d_cond_ce_norm"] = np.array(d_cond.norm().item())
    np.savez_compressed(HERE / "grads_rvq_ce.npz", **out)


if __name__ == "__main__":
    main()
