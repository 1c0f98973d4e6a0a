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


# ---- the flash attention reference (tests/test_attention_edges_gpu.py and the ragged attention suites) ----
LOG2E = 1.4426950408889634
ATTN_RL2 = 2.0 ** -6   # relative L2 of every attention output: a few bf16 roundings of P, dS and the stored result


def _attn_heads(t, B, H):
    return t.double().reshape(B, t.shape[1], H, 64).transpose(1, 2)   # (B, H, N, 64)


def _attn_merge(t):
    B, H, N, _ = t.shape
    return t.transpose(1, 2).reshape(B, N, H * 64)


def attention_reference(q, k, v, d_o, H, scale, drop_key_tile=None):
    """The attention edge suites' reference of softmax(q k^T scale) v on (B, N, H x 64) bf16 operands: float64 o, lse
    (log2 domain), dq, dk, dv and their element-wise error bounds for the kernel's arithmetic.
    drop_key_tile: leave keys [128 t, 128 t + 128) out (sensitivity check)."""
    B = q.shape[0]
    qh, kh, vh, doh = (_attn_heads(t, B, H) for t in (q, k, v, d_o))
    if drop_key_tile is not None:
        keep = torch.ones(kh.shape[2], dtype=torch.bool, device=qh.device)
        keep[128 * drop_key_tile:128 * (drop_key_tile + 1)] = False
        kh, vh = kh[:, :, keep], vh[:, :, keep]
    s = qh @ kh.transpose(-1, -2) * scale
    p = torch.softmax(s, dim=-1)
    o = p @ vh
    lse = torch.logsumexp(s, dim=-1) * LOG2E
    nq, nk = qh.shape[2], kh.shape[2]
    # score error: fp32 sum of 64 bf16 products, in log2 units after the scale
    ds = acc_eps(64) * (qh.abs() @ kh.abs().transpose(-1, -2)).amax(-1) * abs(scale) * LOG2E        # (B, H, Nq)
    # lse = m + log2(l): score error, fp32 sum of nk exponentials in l, fp32 rounding of m + log2(l)
    dlse = ds + acc_eps(nk) * LOG2E + 2.0 ** -18 * (1.0 + lse.abs())
    # relative error of each P element as the kernels form it: bf16 rounding of P + score and lse errors through exp2
    ep = 2.0 ** -9 + math.log(2.0) * (ds + dlse)                                                      # (B, H, Nq)
    pv = p @ vh.abs()
    # o: P's error on both the numerator (P V, an fp32 sum of nk terms) and the normaliser, + bf16 rounding of o
    b_o = 2 * (ep[..., None] + acc_eps(nk)) * (pv + o.abs()) + U_BF16 * o.abs()
    dp = doh @ vh.transpose(-1, -2)
    D = (doh * o).sum(-1, keepdim=True)
    dS = p * (dp - D)
    dv = p.transpose(-1, -2) @ doh
    dk = dS.transpose(-1, -2) @ qh * scale
    dq = dS @ kh * scale
    # dS error: P's relative error on |dP - D|; D from the bf16-rounded o (2^-8 of sum |dO||o|); dP's fp32 sum of 64
    # products; bf16 rounding of dS itself
    dD = U_BF16 * (doh.abs() * o.abs()).sum(-1, keepdim=True) + acc_eps(64) * (doh.abs() * o.abs()).sum(-1, keepdim=True)
    e_p = ep[..., None] * p
    e_dS = (e_p * (dp - D).abs() + p * (acc_eps(64) * (doh.abs() @ vh.abs().transpose(-1, -2)) + dD)
            + 2.0 ** -9 * dS.abs()) * abs(scale)
    b_dv = 2 * (e_p.transpose(-1, -2) @ doh.abs() + acc_eps(nq) * (p.transpose(-1, -2) @ doh.abs())) + U_BF16 * dv.abs()
    b_dk = 2 * (e_dS.transpose(-1, -2) @ qh.abs() + acc_eps(nq) * (dS.abs().transpose(-1, -2) @ qh.abs()) * abs(scale)) \
        + U_BF16 * dk.abs()
    b_dq = 2 * (e_dS @ kh.abs() + acc_eps(nk) * (dS.abs() @ kh.abs()) * abs(scale))
    return dict(o=_attn_merge(o), lse=lse, dq=_attn_merge(dq), dk=_attn_merge(dk), dv=_attn_merge(dv),
                b_o=_attn_merge(b_o), b_lse=dlse, b_dq=_attn_merge(b_dq), b_dk=_attn_merge(b_dk), b_dv=_attn_merge(b_dv))


def attention_inputs(B, H, Nq, Nk, seed, growing_max=False):
    """q / k / v as column windows of one fused (B, N, 3 inner) projection, d_o as a window of a wider buffer."""
    inner = H * 64
    g = torch.Generator(device="cuda").manual_seed(seed)
    qkv = torch.randn(B, max(Nq, Nk), 3 * inner, device="cuda", generator=g)
    if growing_max:
        # scores grow along the key axis (the row maximum moves by far more than 2^8 between key tiles), alternating
        # signs, and 64 queries of sample 1 with all-equal (zero) scores
        qkv[:, :Nk, inner:2 * inner] *= torch.linspace(0.2, 12.0, Nk, device="cuda")[None, :, None]
        qkv[:, :Nk:7, inner:2 * inner] *= -1.0
        qkv[1, :64, :inner] = 0.0
    qkv = qkv.to(torch.bfloat16)
    do_full = torch.randn(B, Nq, inner + 64, device="cuda", generator=g).to(torch.bfloat16)
    return qkv[:, :Nq, :inner], qkv[:, :Nk, inner:2 * inner], qkv[:, :Nk, 2 * inner:], do_full[..., :inner]


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
