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
from .seanet import frame_lengths


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
    def quantize(self, frames: torch.Tensor, stats: Optional[torch.Tensor] = None, *, lengths=None):
        """frames (..., 128) fp32 -> (codes (..., Q) int64, emb (..., 128) fp32 = sum of the chosen codewords).
        lengths (B,) (optional, frames (B, N, 128) padded at the end, in [1, N], at most
        NS2_GEMM_ROW_LENS_MAX_BATCHES samples): sample b's codes and emb past lengths[b] are -1 and exact zeros, and
        its frames there are not read into any valid output."""
        shp = frames.shape[:-1]
        host = None
        if lengths is not None:
            if frames.dim() != 3:
                raise ValueError(f"quantize with lengths takes (B, N, 128) frames, got {tuple(frames.shape)}")
            host = frame_lengths(lengths, frames.shape[0], frames.shape[1], device=frames.device, lo=1)
        if frames.numel() == 0:  # empty batch: nothing to launch (the reference returns empty tensors too)
            return (torch.empty(*shp, self.num_quantizers, dtype=torch.int64, device=frames.device),
                    torch.empty(*shp, 128, dtype=torch.float32, device=frames.device))
        flat = frames.reshape(-1, 128).float()
        if host is not None:   # zero (a copy of) the padding first: the search then meets only finite frames
            flat_lens = ops.lengths(host, len(host), None, device=frames.device)
            flat = ops.mask_rows(flat.clone(memory_format=torch.contiguous_format).view(*shp, 128), flat_lens)
        flat = flat.reshape(-1, 128).contiguous()
        codes = ops.rvq_encode(flat, self.codebooks, self._prep(), stats=stats)
        emb = ops.rvq_decode(codes, self.codebooks)
        codes, emb = codes.view(*shp, self.num_quantizers), emb.view(*shp, 128)
        if host is not None:
            ops.mask_rows(emb, flat_lens)
            codes = codes_past_lengths(codes, host)
        return codes, emb

    @torch.no_grad()
    def forward(self, x, return_encoded: bool = False, curtail_from_left: bool = False, *, lengths=None,
                **kwargs):
        """Mirror of EncodecWrapper.forward's return convention: (emb (B,N,128), codes (B,N,Q), None).
        lengths (B,) (optional, frames): a batch padded at the end.  For raw audio (B, T), sample b is
        x[b, :320 lengths[b]], lengths in [seanet.MIN_FRAMES, T // 320]; nothing is curtailed (curtail_from_left is
        ignored) and the result has T // 320 frames.  Sample b's frames, emb and codes are bit-identical to encoding
        that waveform alone, and past lengths[b] emb is zero and codes are -1.  For frames (B, N, 128) see
        `quantize`."""
        if x.ndim == 2:
            if self.encoder is None:
                raise NotImplementedError(
                    "raw audio needs an `encoder` callable (e.g. seanet.SEANetEncoder, or build the codec with "
                    "EncodecRVQ.from_state_dict); pass encoder-output frames (B, N, 128) instead")
            m = self.seq_len_multiple_of
            T = x.shape[-1] // m * m
            if lengths is not None:
                frame_lengths(lengths, x.shape[0], T // m, device=x.device)   # refuse before the encoder runs
                x = self.encoder(x[..., :T], lengths=lengths)
            else:
                x = x[..., -T:] if curtail_from_left else x[..., :T]
                x = self.encoder(x)
        codes, emb = self.quantize(x, lengths=lengths)
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


def codes_past_lengths(codes: torch.Tensor, lengths) -> torch.Tensor:
    """codes (B, N, Q) int64 -> a new contiguous copy whose rows past lengths[b] (host ints in [0, N]) are -1, the
    `ignore_index` of the RVQ cross-entropy: one `ops.pack_rows` of [codes[b, :len] ; -1 rows], which copies 64-bit
    words, into rows [0, 2N) of a buffer whose first N rows are the result."""
    B, N, Q = codes.shape
    dev = codes.device
    words = torch.empty(B, 2 * N, Q, dtype=torch.int64, device=dev)
    fill = torch.full((1, N, Q), -1, dtype=torch.int64, device=dev).view(torch.bfloat16).expand(B, -1, -1)
    ops.pack_rows(codes.contiguous().view(torch.bfloat16), ops.lengths(lengths, B, N, device=dev, lo=0), fill,
                  ops.lengths([N - n for n in lengths], B, N, device=dev, lo=0), words.view(torch.bfloat16))
    return words[:, :N].contiguous()


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
