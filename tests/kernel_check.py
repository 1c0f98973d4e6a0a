"""Tolerance checks shared by the kernel edge tests (tests/test_*_edges_gpu.py): a CUDA result against a float64
reference of the same operation computed from the same rounded operands.

Every check has two parts:
  1. an element-wise max-abs bound `err <= bound`, where the caller derives `bound` from the output dtype's rounding
     plus an fp32-accumulation term that grows with sqrt(K) (see `acc_eps`);
  2. a relative-L2 bound on the whole tensor.
`assert_rejects` is the sensitivity half: a deliberately wrong reference must fail both parts, so a tolerance cannot
be widened until it passes everything.
"""
from __future__ import annotations

import math
from contextlib import contextmanager

import torch

U_BF16 = 2.0 ** -8   # 2x the half-ulp rounding of a bf16 output (8 significand bits)
U_F32 = 2.0 ** -23   # 2x the half-ulp rounding of an fp32 output


def acc_eps(k: int) -> float:
    """Relative error of an fp32 sum of k products, in units of sum |a_i b_i|: a random walk of k roundings grows like
    sqrt(k) * 2^-24; 16x allowance for the tensor core's truncating adds -> 2^-20 sqrt(k)."""
    return 2.0 ** -20 * math.sqrt(max(k, 1))


def mismatches(got: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor, rel_l2: float) -> list:
    """Failed criteria (empty list = pass): 'non-finite', 'max-abs ...', 'rel-L2 ...'.  The relative-L2 criterion is
    skipped when the reference is itself inside the rounding noise (||ref|| <= ||bound||): the difference of two
    nearly equal terms, e.g. dK with a single key, has no meaningful relative error and is covered by max-abs alone."""
    got, ref = got.double(), ref.double()
    bound = torch.as_tensor(bound, dtype=torch.float64, device=ref.device).expand_as(ref)
    fails = []
    if not bool(torch.isfinite(got).all()):
        fails.append(f"non-finite: {int((~torch.isfinite(got)).sum())} elements")
        got = torch.nan_to_num(got, nan=1e30, posinf=1e30, neginf=-1e30)
    err = (got - ref).abs()
    over = err > bound
    if bool(over.any()):
        ratio = torch.where(over, err / bound.clamp_min(1e-300), torch.zeros_like(err))
        worst = int(ratio.argmax())
        at = tuple(int(v) for v in torch.unravel_index(torch.tensor(worst), ref.shape))
        fails.append(f"max-abs: {int(over.sum())}/{ref.numel()} elements over the bound; worst at {at}: "
                     f"got {float(got.flatten()[worst]):.6g} ref {float(ref.flatten()[worst]):.6g} "
                     f"bound {float(bound.flatten()[worst]):.3g}")
    nref = float(ref.norm())
    if nref > float(bound.norm()):
        r = float((got - ref).norm()) / nref
        if r > rel_l2:
            fails.append(f"rel-L2: {r:.3e} > {rel_l2:.3e}")
    return fails


def assert_close(got, ref, bound, rel_l2, what: str = "") -> None:
    fails = mismatches(got, ref, bound, rel_l2)
    assert not fails, f"{what}: " + "; ".join(fails)


def assert_rejects(got, wrong_ref, bound, rel_l2, what: str = "") -> None:
    """The tolerance must reject a reference that is subtly wrong: both the max-abs and the rel-L2 criterion fail."""
    fails = mismatches(got, wrong_ref, bound, rel_l2)
    assert any(f.startswith("max-abs") for f in fails), f"{what}: max-abs bound accepts the wrong reference"
    assert any(f.startswith("rel-L2") for f in fails), f"{what}: rel-L2 bound accepts the wrong reference"


def assert_nan(t: torch.Tensor, what: str = "") -> None:
    """Elements that must stay untouched were filled with NaN before the call."""
    assert bool(torch.isnan(t.float()).all()), f"{what}: {int((~torch.isnan(t.float())).sum())} elements were written"


def shifted(x: torch.Tensor, s: int) -> torch.Tensor:
    """y[:, n] = x[:, n - s] for (B, N, C) x, zero where n - s is outside [0, N): a causal (s > 0) or anti-causal
    (s < 0) conv tap with its zero padding."""
    N = x.shape[1]
    y = torch.zeros_like(x)
    if 0 <= s < N:
        y[:, s:] = x[:, :N - s]
    elif -N < s < 0:
        y[:, :N + s] = x[:, -s:]
    return y


def gen(seed: int, device: str = "cuda") -> torch.Generator:
    return torch.Generator(device=device).manual_seed(seed)


def nan_buf(shape, dtype=torch.float32, pad: int = 40, device: str = "cuda"):
    """(buffer, contiguous window): the window is the buffer's first prod(shape) elements, the rest stays NaN."""
    n = math.prod(shape)
    buf = torch.full((n + pad,), float("nan"), device=device, dtype=dtype)
    return buf, buf[:n].view(shape)


@contextmanager
def sm_limit(sms: int):
    """Every kernel's persistent grid sized for at most `sms` SMs (0 = all) inside the block; yields the previous
    limit and restores it on exit."""
    from naturalspeech2_pytorch_b200 import ops
    prev = ops.set_sm_limit(sms)
    try:
        yield prev
    finally:
        ops.set_sm_limit(prev)
