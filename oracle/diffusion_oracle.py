"""CPU oracle of the diffusion wrapper arithmetic around the denoiser — TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Restatement of the element-wise maths of `NaturalSpeech2.forward` (ns2.py:1613-1684) and
`NaturalSpeech2.ddim_sample` (ns2.py:1379-1431) of lucidrains/naturalspeech2-pytorch @ 659bec7, with the
denoiser passed in as a callable: the three noise schedules with their keyword arguments (ns2.py:1133-1148), `scale`,
the min-SNR weight on or off with any gamma, and the v / eps / x0 objectives in the loss and in the DDIM step.  Every
function takes numpy arrays or torch tensors, so float64 torch autograd through `diffusion_loss` is a reference for
the hand-written backward.  Pinned by tests/golden/diffusion_*.npz (generated from the reference by
tests/golden/make_golden.py and make_golden_diffusion_configs.py).  Only tests/, __graft_entry__.smoke() and
bench.py's CPU legs may import this.
"""
from __future__ import annotations

import math
from functools import partial

import numpy as np


def _torch(x):
    return type(x).__module__.startswith("torch")


def _lib(x):
    if _torch(x):
        import torch
        return torch
    return np


def _scalar_like(v, t):
    """A 0-d array / tensor of value `v` in `t`'s dtype (and device)."""
    if _torch(t):
        import torch
        return torch.tensor(v, dtype=t.dtype, device=t.device)
    return np.asarray(v, dtype=t.dtype)


def _clip(x, lo=None, hi=None):
    if _torch(x):
        return x.clamp(min=lo, max=hi)
    return np.clip(x, lo, hi)


def _sigmoid(x):
    return 1.0 / (1.0 + _lib(x).exp(-x))


# ---- noise schedules, ns2.py:1133-1148 ----
def linear_schedule(t, clip_min=1e-9):
    """simple_linear_schedule, ns2.py:1133-1134."""
    return _clip(1 - t, clip_min)


def cosine_schedule(t, start=0, end=1, tau=1, clip_min=1e-9):
    """ns2.py:1136-1142 with the cosine of t clamped at 0 before the power (SURVEY T12): the formula's value at
    end = 1, where a rounded cos(pi/2) < 0 and a fractional power would give NaN."""
    power = 2 * tau
    v_start = math.cos(start * math.pi / 2) ** power
    v_end = math.cos(end * math.pi / 2) ** power
    output = _clip(_lib(t).cos((t * (end - start) + start) * math.pi / 2), 0) ** power
    output = (v_end - output) / (v_end - v_start)
    return _clip(output, clip_min)


def sigmoid_schedule(t, start=-3, end=3, tau=1, clamp_min=1e-9):
    """ns2.py:1144-1148."""
    v_start = _sigmoid(_scalar_like(start / tau, t))
    v_end = _sigmoid(_scalar_like(end / tau, t))
    gamma = (-_sigmoid((t * (end - start) + start) / tau) + v_end) / (v_end - v_start)
    return _clip(gamma, clamp_min, 1.0)


SCHEDULES = {"linear": linear_schedule, "cosine": cosine_schedule, "sigmoid": sigmoid_schedule}


def gamma_schedule(name="sigmoid", schedule_kwargs=None):
    """The constructor's `partial(schedule, **schedule_kwargs)`, ns2.py:1251-1267."""
    return partial(SCHEDULES[name], **(schedule_kwargs or {}))


def gamma_to_alpha_sigma(gamma, scale=1.0):
    """ns2.py:1152-1153."""
    sqrt = _lib(gamma).sqrt
    return sqrt(gamma) * scale, sqrt(1 - gamma)


def sampling_time_pairs(timesteps, dtype=np.float32):
    """get_sampling_timesteps, ns2.py:1303-1308: consecutive pairs of linspace(1, 0, timesteps + 1)."""
    times = np.linspace(1.0, 0.0, timesteps + 1, dtype=dtype)
    return list(zip(times[:-1], times[1:]))


# ---- training loss, ns2.py:1627-1684 ----
def loss_weight(alpha, sigma, objective="v", min_snr_loss_weight=True, min_snr_gamma=5.0):
    """Per-sample min-SNR loss weight of ns2.py:1651-1664; alpha, sigma (B,) -> (B,).  sigma = 0 gives snr = inf and,
    as in the reference, an infinite or NaN weight where the formula does."""
    snr = (alpha * alpha) / (sigma * sigma)
    clipped = _clip(snr, hi=min_snr_gamma) if min_snr_loss_weight else snr
    if objective == "eps":
        return clipped / snr
    if objective == "x0":
        return clipped
    return clipped / (snr + 1)


def diffusion_target(x_start, noise, alpha, sigma, objective="v"):
    """ns2.py:1637-1644; alpha, sigma (B,)."""
    if objective == "eps":
        return noise
    if objective == "x0":
        return x_start
    return alpha[:, None, None] * noise - sigma[:, None, None] * x_start


def diffusion_loss(pred, x_start, noise, alpha, sigma, objective="v", min_snr_loss_weight=True, min_snr_gamma=5.0):
    """The loss of ns2.py:1637-1666 from the model output `pred` (B, N, D) and alpha, sigma (B,).  The reference
    multiplies the (B,) per-sample MSE by the (B,1,1) weight, which broadcasts to (B,1,B): its mean is
    mean(per-sample MSE) x mean(weight), not the mean of per-sample products.  -> (loss, dict of intermediates)."""
    target = diffusion_target(x_start, noise, alpha, sigma, objective)
    per_sample = ((pred - target) ** 2).reshape(pred.shape[0], -1).mean(1)
    w = loss_weight(alpha, sigma, objective, min_snr_loss_weight, min_snr_gamma)
    loss = (per_sample * w.reshape(-1, 1, 1)).mean()
    return loss, {"target": target, "per_sample": per_sample, "weight": w}


def x_start_from_pred(x, pred, alpha, sigma, objective="v"):
    """x_start from a model output, ns2.py:1412-1421 and 1673-1680 (safe_div clamps alpha at 1e-10, ns2.py:1122)."""
    a, s = alpha[:, None, None], sigma[:, None, None]
    if objective == "v":
        return a * x - s * pred
    if objective == "eps":
        return (x - s * pred) / _clip(a, 1e-10)
    return pred


def training_loss(model_fn, x_start, times, noise, objective="v", min_snr_gamma=5.0, scale=1.0, schedule="sigmoid",
                  schedule_kwargs=None, min_snr_loss_weight=True):
    """ns2.py:1621-1666 with `times` and `noise` given (the reference draws them at 1621 and 1625).
    model_fn(noised, times) -> prediction.  Returns (loss scalar, dict of intermediates)."""
    gamma = gamma_schedule(schedule, schedule_kwargs)(times.astype(x_start.dtype))
    alpha, sigma = gamma_to_alpha_sigma(gamma, scale)
    noised = alpha[:, None, None] * x_start + sigma[:, None, None] * noise
    pred = model_fn(noised, times)
    loss, parts = diffusion_loss(pred, x_start, noise, alpha, sigma, objective, min_snr_loss_weight, min_snr_gamma)
    parts["noised"] = noised
    return loss, parts


# ---- DDIM, ns2.py:1379-1431 ----
def ddim_step_coef(x, v, alpha, sigma, alpha_next, sigma_next, objective="v"):
    """One iteration of ddim_sample (ns2.py:1414-1429) with the step's coefficients given, each (B,)."""
    x0 = x_start_from_pred(x, v, alpha, sigma, objective)
    eps = (x - alpha[:, None, None] * x0) / _clip(sigma[:, None, None], 1e-10)
    return x0 * alpha_next[:, None, None] + eps * sigma_next[:, None, None]


def step_coefficients(t, t_next, scale=1.0, schedule="sigmoid", schedule_kwargs=None):
    """(alpha, sigma, alpha_next, sigma_next) of one step, ns2.py:1396-1402.  The reference shifts times_next by
    `time_difference` only after it has computed these (ns2.py:1406), so the shift never reaches the update."""
    f = gamma_schedule(schedule, schedule_kwargs)
    a, s = gamma_to_alpha_sigma(f(t), scale)
    an, sn = gamma_to_alpha_sigma(f(t_next), scale)
    return a, s, an, sn


def ddim_step(x, v, t, t_next, scale=1.0, objective="v", schedule="sigmoid", schedule_kwargs=None):
    """One iteration of ddim_sample from the step's times (B,); `v` is the model output."""
    dtype = x.dtype
    coef = step_coefficients(np.asarray(t, dtype=dtype), np.asarray(t_next, dtype=dtype), scale, schedule,
                             schedule_kwargs)
    return ddim_step_coef(x, v, *coef, objective=objective)


def ddim_sample(model_fn, x_init, timesteps, scale=1.0, objective="v", schedule="sigmoid", schedule_kwargs=None):
    """ddim_sample, ns2.py:1379-1431, from a given initial noise."""
    x = x_init
    B = x.shape[0]
    for t, tn in sampling_time_pairs(timesteps, dtype=x.dtype):
        tb = np.full((B,), t, dtype=x.dtype)
        tnb = np.full((B,), tn, dtype=x.dtype)
        v = model_fn(x, tb)
        x = ddim_step(x, v, tb, tnb, scale, objective, schedule, schedule_kwargs)
    return x
