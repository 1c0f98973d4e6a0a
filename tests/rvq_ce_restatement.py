"""fp64, autograd-capable restatement of the RVQ cross-entropy head — TEST INFRASTRUCTURE, NOT PRODUCT CODE.

`codec.rq(x_start, codes)` (ns2.py:1682) is vector-quantize-pytorch's `ResidualVQ.forward(x, indices=codes)`, third-party
code with no pinned version (see oracle/rvq_oracle.py for the codec's provenance).  This module restates it with torch
ops so that autograd differentiates it; the CE-gradient tests (tests/test_rvq_ce_*.py) and the fixture generator
tests/golden/make_golden_rvq_ce.py use it as the reference.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F


def residual_vq_ce(x, codebooks, codes, own=None):
    """ResidualVQ.forward(x, indices=codes) as NaturalSpeech2 calls it (ns2.py:1682) -> (quantized, ce_loss, own codes).
    Use float64 tensors for a reference.

    Per stage q: d_k = ||r_q - c_k|| (expanded formula, clamped at 0), logits = -d, CE_q = cross_entropy(logits,
    codes[:, q], ignore_index=-1) (NaN when every target is -1), ce_loss = sum_q CE_q; own_q = argmin_k d_k (first on
    ties) unless `own` (F, Q) is given; r_{q+1} = r_q - C_q[own_q] with the codeword a constant (the reference subtracts
    `quantized.detach()`).  A zero distance gets a zero derivative, torch.cdist's backward convention."""
    Q, K, D = codebooks.shape
    r = x.reshape(-1, D)
    tgt = torch.as_tensor(codes).reshape(-1, Q).long().to(r.device)
    cb = codebooks.detach().to(r.device, r.dtype)
    own_out = torch.empty(r.shape[0], Q, dtype=torch.int64, device=r.device)
    quantized = torch.zeros_like(r.detach())
    loss = 0.
    for q in range(Q):
        E = cb[q]
        d2 = ((r * r).sum(-1, keepdim=True) - 2.0 * (r @ E.t()) + (E * E).sum(-1)[None]).clamp_min(0.)
        pos = d2 > 0
        dist = torch.where(pos, d2.clamp_min(torch.finfo(d2.dtype).tiny).sqrt(), torch.zeros_like(d2))
        loss = loss + F.cross_entropy(-dist, tgt[:, q], ignore_index=-1)
        idx = dist.detach().argmin(-1) if own is None else torch.as_tensor(own).reshape(-1, Q)[:, q].long().to(r.device)
        own_out[:, q] = idx
        quantized = quantized + E[idx]
        r = r - E[idx]
    return quantized.view(*x.shape), loss, own_out
