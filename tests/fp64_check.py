"""The numerics protocol of the float64 suites (tests/test_*_fp64_gpu.py): our CUDA result against a float64
restatement of the same computation and against that restatement's "twin", the same code in fp32 under
torch.autocast("cuda", bfloat16) (the reference's own reduced-precision mode), on the same bf16-rounded operands.

A tensor passes when
  (i)   rel-L2 <= C x the twin's rel-L2 + floor,
  (ii)  rel-L2 <= ceiling,
  (iii) it is exactly zero wherever the float64 value is exactly zero, and nothing is non-finite.
C, floor and ceiling are per family of modules (FAMILIES below, measured in the suites named there).  A tensor whose
float64 value is all zeros is checked by (iii) alone.

to_q: the attention backward forms D = rowsum(dO * O) from the bf16 output, so where self-attention is nearly flat
to_q's exact gradient falls below that rounding and its twin comparison says nothing (see
test_conditioning_backward_fp64_gpu.py).  Its error is then measured as a share of the gradient of the fused q / kv
projection (`rel_qkv`), bounded by TO_Q_BOUND.  A suite picks one of two rules for the tensors it gives a share:
  SHARE_ONLY  the share alone decides;
  EITHER      the tensor passes under (i)-(ii) or under the share bound.
Without a rule the share is only printed.

`assert_rejected` is the sensitivity half: a deliberately wrong reference must fail the same bounds.
"""
from __future__ import annotations

import contextlib
import math
from dataclasses import dataclass, replace
from typing import NamedTuple

import torch


@dataclass(frozen=True)
class Family:
    c: float          # ours may be C x the twin's rel-L2 ...
    floor: float      # ... + floor (keeps the bound above zero where the twin is exact) ...
    ceiling: float    # ... and at most this

    def without_ceiling(self, c: float | None = None) -> "Family":
        """C x twin + floor alone, optionally with another C: named exceptions and the deep benchmark step."""
        return replace(self, c=self.c if c is None else c, ceiling=math.inf)


# test_denoiser_backward_fp64_gpu.py / test_denoiser_configs_fp64_gpu.py: ours / twin <= 0.81, worst 1.1e-2
DENOISER = Family(c=1.0, floor=2e-3, ceiling=1.5e-2)
# test_conditioning_backward_fp64_gpu.py / test_encoder_configs_fp64_gpu.py: ours / twin <= 1.27, worst 1.50e-2
ENCODERS = Family(c=1.5, floor=2e-3, ceiling=2e-2)
# test_duration_pitch_backward_fp64_gpu.py: ours / twin <= 1.28
PREDICTOR = Family(c=1.5, floor=2e-3, ceiling=2e-2)
FAMILIES = {"denoiser": DENOISER, "encoders": ENCODERS, "predictor": PREDICTOR}
TO_Q_BOUND = 3e-3     # the encoders' to_q: |ours - fp64| / |fp64 to_q ; to_kv|, measured worst 2.39e-3
MARGIN = 20.0         # the predictor's ReLU heads: every |pre-activation| >= MARGIN x our forward's max-abs error

SHARE_ONLY, EITHER = "share only", "either"


def rel_l2(got, ref) -> float:
    ref = torch.as_tensor(ref).double()
    return float((got.detach().double() - ref).norm() / ref.norm())


def rel_qkv(got, ref, ref_kv) -> float:
    """to_q's error relative to the gradient of the whole fused q / kv projection (one wgrad computes both)."""
    return float((got.double() - ref).norm() / torch.cat((ref, ref_kv)).norm())


def bf(g, *shape, scale=1.0):
    """bf16-representable randn on the GPU."""
    return (torch.randn(*shape, generator=g) * scale).bfloat16().float().cuda()


def round_params(module):
    with torch.no_grad():
        for p in module.parameters():
            p.copy_(p.bfloat16().float())        # the packs hold exactly these values


class Stat(NamedTuple):
    rel: float                      # rel-L2 ours
    rel_ac: float                   # rel-L2 of the twin
    share: float | None = None      # to_q: ours as a share of the q / kv gradient
    zeros: int = 0                  # exact zeros of the float64 value
    max_abs: float | None = None    # with max_abs=True: max |ours - fp64|, max |twin - fp64|, max |fp64|
    max_abs_ac: float | None = None
    max_ref: float | None = None


def compare(o, r, ac, kv=None, max_abs=False):
    """Ours `o` against the float64 `r` and the twin `ac` of one tensor: a failure string (non-finite, or non-zero where
    `r` is exactly zero), None when `r` is all zeros (nothing left to compare), else a Stat.  `kv`: the float64 to_kv
    gradient next to a to_q, for its share."""
    o = o.reshape(r.shape)
    if not bool(torch.isfinite(o).all()):
        return "non-finite"
    zero = r == 0
    if bool(zero.any()) and bool((o[zero] != 0).any()):
        return f"{int((o[zero] != 0).sum())} of {int(zero.sum())} exact zeros are not zero"
    if bool(zero.all()):
        return None
    extra = {}
    if max_abs:
        extra = dict(max_abs=float((o.double() - r).abs().max()), max_abs_ac=float((ac.double() - r).abs().max()),
                     max_ref=float(r.abs().max()))
    return Stat(rel_l2(o, r), rel_l2(ac, r), None if kv is None else rel_qkv(o, r, kv), int(zero.sum()), **extra)


def bound(fam: Family, rel_ac: float) -> float:
    return min(fam.c * rel_ac + fam.floor, fam.ceiling)


def use(fam: Family, s, to_q=None) -> float:
    """Share of its bound that s = (rel, rel_ac, share, ...) uses; above 1 is over."""
    rel, rel_ac, share = s[:3]
    u = rel / bound(fam, rel_ac)
    if to_q is None or share is None:
        return u
    return share / TO_Q_BOUND if to_q == SHARE_ONLY else min(u, share / TO_Q_BOUND)


def over(fam: Family, s, to_q=None) -> bool:
    rel, rel_ac, share = s[:3]
    if to_q is None or share is None:
        return rel > bound(fam, rel_ac)
    if to_q == SHARE_ONLY:
        return share > TO_Q_BOUND
    return rel > bound(fam, rel_ac) and share > TO_Q_BOUND


def assert_rejected(ours, wrong, stats, names, fam, to_q=None, at_least=None):
    """The bounds of the real comparison (its twin rel-L2, stats[n].rel_ac) must reject the wrong reference `wrong`
    against our kept gradients `ours` for every name, or for `at_least` of them.  `fam` is a Family or a function of
    the name.  Returns the smallest margin (rel-L2 / bound, name)."""
    fam_of = fam if callable(fam) else (lambda n: fam)
    rejected, margins = [], []
    for n in names:
        s = stats[n]
        o = ours[n].reshape(wrong[n].shape)
        rel = rel_l2(o, wrong[n])
        share = rel_qkv(o, wrong[n], wrong[n.replace("to_q", "to_kv")]) if to_q and s[2] is not None else None
        b = bound(fam_of(n), s[1])
        print(f"  {n}: rel-L2 vs the wrong reference {rel:.3e} (bound {b:.3e}, {rel / b:.1f}x)" +
              (f", {share:.3e} of the q / kv gradient (bound {TO_Q_BOUND:.1e})" if share is not None else ""))
        margins.append((rel / b, n))
        if over(fam_of(n), (rel, s[1], share), to_q):
            rejected.append(n)
    if at_least is None:
        assert rejected == list(names), f"the bound accepts a wrong reference for {sorted(set(names) - set(rejected))}"
    else:
        assert len(rejected) >= at_least, rejected
    return min(margins)


def autograd(fwd, params, d_outs, autocast=False, inputs=None, only=None, cudnn=None, out_prefix=None):
    """{name: gradient} of the restatement fwd(P, dtype) -> {output name: tensor}, in float64, or in fp32 under bf16
    autocast for the twin.  P holds `params` (the modules' rounded fp32 values) and the floating-point `inputs` as
    leaves; outputs whose upstream gradient in `d_outs` is None or absent are left out.  A leaf that no output reaches
    gets zeros.  cudnn: None leaves torch's setting, False turns cuDNN off for both runs, "twin" turns it on only for
    the autocast run (the float64 one without: conv taps that only read the zero padding then get exact zeros).
    With out_prefix, and only=None, the outputs too, under out_prefix + their name."""
    dtype = torch.float32 if autocast else torch.float64
    P = {n: p.detach().to(dtype).requires_grad_(True) for n, p in params.items()}
    P.update({n: t.detach().to(dtype).requires_grad_(True) for n, t in (inputs or {}).items() if t.is_floating_point()})
    names = list(P) if only is None else list(only)
    flags = (contextlib.nullcontext() if cudnn is None else
             torch.backends.cudnn.flags(enabled=autocast if cudnn == "twin" else bool(cudnn)))
    with flags:
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
            outs = fwd(P, dtype)
        used = [(o, d_outs[k]) for k, o in outs.items() if d_outs.get(k) is not None]
        g = torch.autograd.grad([o for o, _ in used], [P[n] for n in names], [d.to(o.dtype) for o, d in used],
                                allow_unused=True)
    res = {n: torch.zeros_like(P[n]) if gi is None else gi.detach() for n, gi in zip(names, g)}
    if out_prefix is not None and only is None:
        res.update({out_prefix + k: o.detach() for k, o in outs.items()})
    return res
