"""numpy restatement of the library's dropout random numbers (include/ns2_b200.h section 2b, csrc/philox.cuh), and fp64
torch restatements of the conditioning encoders with given dropout masks — TEST INFRASTRUCTURE, NOT PRODUCT CODE.

  philox4x32_10        Philox4x32-10 on uint32 arrays (Salmon et al., SC 2011), vectorised
  keep_threshold       t = min(floor(p 2^32 + 0.5), 2^32 - 1) of the float32 p; keep iff word >= t
  keep_scale           float32(1 / (1 - p))
  attention_mask       keep mask (B, H, Nq, Nk) of one attention dropout site
  elementwise_mask     keep mask of n consecutive elements of one element-wise site
  speech_prompt_encoder / phoneme_encoder: oracle.encoders_oracle's restatements with attention masks applied after
                       the softmax and before `@ v`, and the phoneme encoder's conv mask after the SiLU
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle import encoders_oracle as eo

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = 0x9E3779B9, 0xBB67AE85
U32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Four uint32 arrays (broadcast of the counter words) for the 64-bit key (k0, k1)."""
    c = [np.asarray(v, dtype=np.uint64) & U32 for v in (c0, c1, c2, c3)]
    c = list(np.broadcast_arrays(*c))
    k0, k1 = int(k0) & 0xFFFFFFFF, int(k1) & 0xFFFFFFFF
    for _ in range(10):
        p0, p1 = M0 * c[0], M1 * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ np.uint64(k0), p1 & U32, (p0 >> np.uint64(32)) ^ c[3] ^ np.uint64(k1), p0 & U32]
        k0, k1 = (k0 + W0) & 0xFFFFFFFF, (k1 + W1) & 0xFFFFFFFF
    return [v.astype(np.uint32) for v in c]


def _p32(p: float) -> float:
    p = float(np.float32(p))
    if not 0.0 <= p < 1.0:
        raise ValueError(f"dropout p must be in [0, 1), got {p}")
    return p


def keep_threshold(p: float) -> int:
    return min(math.floor(_p32(p) * 2.0 ** 32 + 0.5), 2 ** 32 - 1)


def keep_scale(p: float) -> np.float32:
    return np.float32(1.0 / (1.0 - _p32(p)))


def _attn_index(x):
    return ((x >> 4) << 3) | (x & 7)


def attention_mask(seed: int, site: int, p: float, batches: int, heads: int, q_len: int, kv_len: int) -> np.ndarray:
    """bool (B, H, Nq, Nk): element (b, h, q, k) is word 2 q[3] + k[3] of the Philox block of
    (idx(k & ~8), idx(q & ~8), b heads + h, site), idx(x) = (x >> 4) 8 + (x & 7)."""
    t = keep_threshold(p)
    q, k = np.arange(q_len), np.arange(kv_len)
    uq, uk = np.unique(q & ~8), np.unique(k & ~8)
    bh = (np.arange(batches)[:, None] * heads + np.arange(heads)[None, :])[:, :, None, None]
    words = philox4x32_10(_attn_index(uk)[None, None, None, :], _attn_index(uq)[None, None, :, None], bh, site,
                          seed & 0xFFFFFFFF, seed >> 32)
    w = np.stack(words, axis=-1)                                        # (B, H, |uq|, |uk|, 4)
    iq, ik = np.searchsorted(uq, q & ~8), np.searchsorted(uk, k & ~8)
    sel = ((q >> 3) & 1)[:, None] * 2 + ((k >> 3) & 1)[None, :]
    return w[:, :, iq[:, None], ik[None, :], sel] >= t


def elementwise_mask(seed: int, site: int, p: float, n: int) -> np.ndarray:
    """bool (n,): element i is word i & 3 of the Philox block of ((i >> 2) mod 2^32, i >> 34, 0xffffffff, site)."""
    t = keep_threshold(p)
    g = np.arange((n + 3) // 4, dtype=np.uint64)
    w = np.stack(philox4x32_10(g & U32, g >> np.uint64(32), 0xFFFFFFFF, site, seed & 0xFFFFFFFF, seed >> 32), axis=-1)
    return w.reshape(-1)[:n] >= t


def mask_tensor(mask: np.ndarray, p: float) -> torch.Tensor:
    """keep * scale as an fp64 tensor (what multiplies the dropped values)."""
    return torch.from_numpy(mask).double() * float(keep_scale(p))


# ---- encoders with dropout masks (fp64 torch, any device) ----
def _attention(x, P, pre, heads, mask):
    q = x @ P[pre + "to_q.weight"].T
    k, v = (x @ P[pre + "to_kv.weight"].T).chunk(2, dim=-1)
    b, n, _ = q.shape
    q, k, v = (t.view(b, n, heads, -1).transpose(1, 2) for t in (q, k, v))
    attn = (torch.einsum("bhid,bhjd->bhij", q, k) * (q.shape[-1] ** -0.5)).softmax(dim=-1)
    if mask is not None:
        attn = attn * mask                                                      # attend.py:149
    out = torch.einsum("bhij,bhjd->bhid", attn, v)
    return out.transpose(1, 2).reshape(b, n, -1) @ P[pre + "to_out.weight"].T


def transformer(x, P, prefix, heads, attn_masks=None):
    depth = 1 + max(int(k[len(prefix):].split(".")[1]) for k in P if k.startswith(prefix + "layers."))
    for l in range(depth):
        pre = f"{prefix}layers.{l}."
        m = None if attn_masks is None else attn_masks[l]
        x = _attention(eo._rmsnorm(x, P[pre + "0.gamma"]), P, pre + "1.", heads, m) + x
        x = eo._feedforward(eo._rmsnorm(x, P[pre + "2.gamma"]), P, pre + "3.") + x
    return x


def speech_prompt_encoder(P, x, heads=8, padding=4, attn_masks=None):
    h = x.transpose(1, 2)
    i = 1
    while f"conv.{i}.weight" in P:
        h = F.silu(F.conv1d(h, P[f"conv.{i}.weight"], P[f"conv.{i}.bias"], padding=padding))
        i += 2
    return transformer(h.transpose(1, 2), P, "transformer.", heads, attn_masks)


def phoneme_encoder(P, ids, heads=8, conv_mask=None, attn_masks=None):
    """conv_mask: (B, T, dim_hidden) keep * scale of the conv output (token-major, the library's element order)."""
    pad_id = P["token_emb.weight"].shape[0] - 1
    ids = ids.masked_fill(ids < 0, pad_id)
    h = P["token_emb.weight"][ids].transpose(1, 2)
    w = P["conv.1.weight"]
    h = F.silu(F.conv1d(F.pad(h, (w.shape[-1] - 1, 0)), w, P["conv.1.bias"])).transpose(1, 2)
    if conv_mask is not None:
        h = h * conv_mask                                                       # ns2.py:258
    return transformer(h, P, "transformer.", heads, attn_masks)
