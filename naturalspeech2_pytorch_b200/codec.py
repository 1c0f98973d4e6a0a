"""`EncodecRVQ`: the residual-VQ step of the Encodec codec on sm_90a, behind the duck-type that
`NaturalSpeech2` expects from `audiolm_pytorch.EncodecWrapper` (ns2.py:1213-1214, 1244-1246, 1445, 1496, 1611).

In scope (SURVEY a16): nearest-codeword search over Q sequential residual stages (`ops.rvq_encode`, wgmma
distance filter + exact fp64 re-score => bit-exact indices) and the sum-of-codewords decode (`ops.rvq_decode`).
Encodec's SEANet encoder and decoder plug in as callables:
    encoder(raw_audio (B, T)) -> frames (B, N, 128)        decoder(emb (B, N, 128)) -> audio (B, 1, T)
`seanet.SEANetEncoder` and `seanet.SEANetDecoder` are the 24 kHz encoder and decoder on this library's kernels;
`EncodecRVQ.from_state_dict` builds the whole codec from one transformers `EncodecModel` state_dict.  Without an
encoder the codec accepts encoder-output frames (B, N, 128) directly; without a decoder `decode` returns the latents.
"""
from __future__ import annotations

from typing import Callable, Dict, Optional

import torch
from torch import nn

from . import ops


class EncodecRVQ(nn.Module):
    def __init__(self, codebooks: torch.Tensor, *, target_sample_hz: int = 24000, strides=(2, 4, 5, 8),
                 encoder: Optional[Callable] = None, decoder: Optional[Callable] = None):
        """codebooks: (Q, K, 128) fp32 — `model.quantizer.vq.layers[q]._codebook.embed` of an Encodec model."""
        super().__init__()
        if codebooks.dim() != 3 or codebooks.shape[-1] != 128:
            raise ValueError("codebooks must be (num_quantizers, codebook_size, 128)")
        self.register_buffer("codebooks", codebooks.detach().float().contiguous())
        self.target_sample_hz = target_sample_hz
        self.seq_len_multiple_of = 1
        for s in strides:
            self.seq_len_multiple_of *= s  # 320 for the 24 kHz model
        self.codebook_dim = codebooks.shape[-1]
        self.num_quantizers = codebooks.shape[0]
        self.encoder = encoder
        self.decoder = decoder
        self._prepared = None
        self._prepared_key = None

    @classmethod
    def from_state_dict(cls, sd: Dict[str, torch.Tensor], *, num_quantizers: int = 8) -> "EncodecRVQ":
        """The 24 kHz codec from a transformers `EncodecModel` state_dict: `SEANetEncoder` from `encoder.*`,
        `SEANetDecoder` from `decoder.*`, and the first `num_quantizers` codebooks
        `quantizer.layers.{q}.codebook.embed` (8 = the 6 kbps bandwidth).  Move the result with `.cuda()`."""
        from .seanet import SEANetDecoder, SEANetEncoder
        parts = {}
        for name, module in (("encoder", SEANetEncoder()), ("decoder", SEANetDecoder())):
            module.load_state_dict({k[len(name) + 1:]: v.float() for k, v in sd.items() if k.startswith(name + ".")})
            parts[name] = module.eval()
        cb = torch.stack([sd[f"quantizer.layers.{q}.codebook.embed"] for q in range(num_quantizers)])
        return cls(cb, **parts)

    def _prep(self):
        key = (self.codebooks.data_ptr(), self.codebooks._version, str(self.codebooks.device))
        if self._prepared is None or key != self._prepared_key:
            self._prepared = ops.rvq_prepare(self.codebooks)
            self._prepared_key = key
        return self._prepared

    @torch.no_grad()
    def quantize(self, frames: torch.Tensor, stats: Optional[torch.Tensor] = None):
        """frames (..., 128) fp32 -> (codes (..., Q) int64, emb (..., 128) fp32 = sum of the chosen codewords)."""
        shp = frames.shape[:-1]
        if frames.numel() == 0:  # empty batch: nothing to launch (the reference returns empty tensors too)
            return (torch.empty(*shp, self.num_quantizers, dtype=torch.int64, device=frames.device),
                    torch.empty(*shp, 128, dtype=torch.float32, device=frames.device))
        flat = frames.reshape(-1, 128).float().contiguous()
        codes = ops.rvq_encode(flat, self.codebooks, self._prep(), stats=stats)
        emb = ops.rvq_decode(codes, self.codebooks)
        return codes.view(*shp, self.num_quantizers), emb.view(*shp, 128)

    @torch.no_grad()
    def forward(self, x, return_encoded: bool = False, curtail_from_left: bool = False, **kwargs):
        """Mirror of EncodecWrapper.forward's return convention: (emb (B,N,128), codes (B,N,Q), None)."""
        if x.ndim == 2:
            if self.encoder is None:
                raise NotImplementedError(
                    "raw audio needs an `encoder` callable (e.g. seanet.SEANetEncoder, or build the codec with "
                    "EncodecRVQ.from_state_dict); pass encoder-output frames (B, N, 128) instead")
            m = self.seq_len_multiple_of
            T = x.shape[-1] // m * m
            x = x[..., -T:] if curtail_from_left else x[..., :T]
            x = self.encoder(x)
        codes, emb = self.quantize(x)
        if not return_encoded:
            return codes
        return emb, codes, None

    @torch.no_grad()
    def get_emb_from_indices(self, codes: torch.Tensor) -> torch.Tensor:
        """codes (..., Q) integer -> emb (..., 128) fp32, the sum of the indexed codewords."""
        if codes.is_floating_point() or codes.dim() == 0 or codes.shape[-1] != self.num_quantizers:
            raise ValueError(f"codes must be integer (..., {self.num_quantizers}), got {codes.dtype} "
                             f"{tuple(codes.shape)}")
        shp = codes.shape[:-1]
        if codes.numel() == 0:  # nothing to launch, as in `quantize`
            return torch.empty(*shp, 128, dtype=torch.float32, device=codes.device)
        emb = ops.rvq_decode(codes.reshape(-1, self.num_quantizers).to(torch.int64).contiguous(), self.codebooks)
        return emb.view(*shp, 128)

    @torch.no_grad()
    def decode(self, emb: torch.Tensor) -> torch.Tensor:
        if self.decoder is None:
            return emb
        return self.decoder(emb)

    def rq(self, x: torch.Tensor, codes: torch.Tensor):
        """The call `NaturalSpeech2.forward` makes when rvq_cross_entropy_loss_weight != 0 (ns2.py:1682):
        `_, ce_loss = codec.rq(x_start, codes)` — vector-quantize-pytorch's ResidualVQ.forward(x, indices=codes).
        Per stage: logits = -||r_q - c_k|| (Euclidean), cross-entropy against codes[..., q] (ignore_index -1),
        residual chain through the codec's own nearest codewords; returns (quantized, summed CE loss).
        The loss is differentiable in `x` when gradients are enabled and `x` requires them (one autograd node whose
        backward is `ops.rvq_ce_bwd`); `quantized` and the codebooks are constants, as in the reference (its subtracted
        codewords are detached and the codebooks are buffers)."""
        shp = x.shape[:-1]
        tgt = codes.reshape(-1, self.num_quantizers).to(torch.int64).contiguous()
        if torch.is_grad_enabled() and x.requires_grad:
            loss, own = RqCrossEntropyFunction.apply(x.reshape(-1, 128).float().contiguous(), self, tgt)
        else:
            with torch.no_grad():
                flat = x.reshape(-1, 128).float().contiguous()
                prep = self._prep()
                own = ops.rvq_encode(flat, self.codebooks, prep)
                loss = ops.rvq_ce(flat, self.codebooks, prep[1], own, tgt)
        with torch.no_grad():
            emb = ops.rvq_decode(own, self.codebooks)
        return emb.view(*shp, 128), loss


class RqCrossEntropyFunction(torch.autograd.Function):
    """`EncodecRVQ.rq`'s cross-entropy loss as one autograd node: the forward runs the same kernels as the no-grad path
    (own codes, then the CE head), the backward is one `ops.rvq_ce_bwd` call.  Returns (loss, own codes)."""

    @staticmethod
    def forward(ctx, flat, codec, tgt):
        prep = codec._prep()
        own = ops.rvq_encode(flat, codec.codebooks, prep)
        loss = ops.rvq_ce(flat, codec.codebooks, prep[1], own, tgt)
        ctx.save_for_backward(flat, codec.codebooks, prep[1], own, tgt)
        ctx.mark_non_differentiable(own)
        return loss, own

    @staticmethod
    def backward(ctx, d_loss, _d_own):
        flat, codebooks, cn2, own, tgt = ctx.saved_tensors
        d = ops.rvq_ce_bwd(flat, codebooks, cn2, own, tgt, d_loss.float().reshape(1).contiguous())
        return d, None, None
