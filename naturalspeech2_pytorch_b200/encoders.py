"""Per-sample conditioning encoders of NaturalSpeech2 on the sm_90a kernels (SURVEY section 8, row f3).

`SpeechPromptEncoder` (ns2.py:289-341) and `PhonemeEncoder` (ns2.py:228-287) run once per sample BEFORE the denoiser
loop (`NaturalSpeech2.forward` ns2.py:1537-1539, `sample` 1474-1476).  Both are a stack of k=9 convolutions with SiLU
followed by the plain `Transformer` (ns2.py:1073-1117: RMSNorm -> Attention -> +res, RMSNorm -> GEGLU FeedForward ->
+res).  Same constructor arguments, same parameter names and shapes as the reference, so a reference state_dict loads
unchanged; the module tree only HOLDS parameters, the math goes through `ops` (libns2b200.so):

  Conv1d(k=9, padding=4) + SiLU   one segmented wgmma GEMM with nine shifted-row segments (TMA zero fill = the
                                  "same" padding), SiLU in the epilogue (NS2_GEMM_FLAG_SILU)
  CausalConv1d(k=9) + SiLU        the same GEMM with shifts 8..0 (left padding only, ns2.py:583-595)
  nn.Embedding                    ops.embedding_bf16 (gather + padding substitution)
  Transformer layer               RMSNorm kernel -> fused QKV GEMM -> flash attention -> out-proj GEMM (+residual,
                                  fp32 stream) -> RMSNorm -> GEGLU GEMM -> out GEMM (+residual)

Training: in `train()` mode with gradients enabled (and parameters or a float input that require them)
`SpeechPromptEncoder.forward` and `PhonemeEncoder.forward` record ONE autograd node each (`_EncoderFunction`, the
pattern of training.DenoiserFunction).  Its forward is the inference forward (`_forward` and `_transformer`) given a
`saved` dict, which keeps the activations the backward needs (bit-identical output); its backward walks the encoder in
reverse:
  plain Transformer      training.ff_backward and training.attention_backward (shared with the denoiser's backward)
                         on the transposed packs, rmsnorm_film_bwd(gamma=...)
  k=9 conv + SiLU        pre-activation recomputed with a plain-epilogue GEMM, ops.silu_bwd, then training.conv_backward:
                         one ops.wgrad per tap ("same" padding: shifts +4..-4, causal: 8..0), dgrad = one nine-segment
                         GEMM with mirrored shifts (the prompt encoder's first conv only when the prompt requires grad:
                         it usually comes from the codec)
  nn.Embedding           ops.embedding_bwd (scatter-add; the pad row receives gradient, as in the reference)
Dropout: with `train_dropout` set (default False; `Conditioner(train_dropout=True)` sets it on both encoders) a call
in train() mode - with or without autograd, like nn.Dropout - draws the reference's dropout: every transformer layer's
attention drops softmax probabilities with p = `attn_dropout` (SpeechPromptEncoder's `dropout`, PhonemeEncoder's
`attn_dropout`; Attend, attend.py:106 / 149), and the phoneme encoder drops its causal conv's SiLU output with p =
`conv_dropout` (ns2.py:258).  The masks are Philox streams (include/ns2_b200.h section 2b) of one 64-bit seed drawn per
call from torch's default CPU generator (no device sync; torch.manual_seed reproduces it); site 0 is the conv, site
1 + l the attention of layer l.  The backward regenerates them from the seed in the record.  Without train_dropout, in
eval() mode, or with p = 0 nothing is drawn and the kernels are those of inference.
`DurationPitchPredictor.forward` records one node the same way, for both outputs (duration_pred, pitch_pred) and both
inputs (phoneme encodings or token ids, encoded prompts); its backward walks each trunk in reverse:
  Linear(dim, 1) + ReLU  ops.rowdot_bwd (d x into the trunk's fp32 residual-stream gradient)
  cross attention        training.attention_backward with the keys [RMSNorm(x) ; prompts]: d ctx = d kv Wkv is split
                         into the queries' rows (joining d RMSNorm(x) before rmsnorm_film_bwd) and the prompts' rows
                         (accumulated in fp32 over both trunks and all layers)
  ResnetBlock            per Block in reverse ops.groupnorm_silu_bwd on the saved conv output, then training.
                         conv_backward ("same" k=3: shifts +1..-1); the first Block's d x is added to the identity path
A prediction that gets no gradient skips its trunk (its parameters get None); d x of both trunks is summed, or
scattered into the token table.
The predictor's dropout: its constructor's `dropout` (0.2 by default) is what the reference hands to every layer's
cross Attention (ns2.py:438-446): attention dropout on the softmax probabilities (Attend, attend.py:106 / 149), in the
flash kernels.  The trunk builds its ResnetBlocks without a dropout argument (ns2.py:430, 435), so every Block's
nn.Dropout has the default p = 0 (ns2.py:352, 374) and draws nothing.  With `train_dropout` (default False;
`Conditioner(duration_pitch_dropout=True)` sets it) the attention dropout is drawn exactly as in the encoders: one seed
per call in train() mode, none in eval(), without train_dropout or with p = 0.  The cross attention of layer l of trunk
t (0 duration, 1 pitch; forward order) is site t depth + l.  The record keeps the seed, no mask.
Attention masks are not supported (`mask=None` is what NaturalSpeech2.forward / .sample pass, ns2.py:1475-1476,
1538-1539).  A batch of sequences of different lengths, each padded at its end, is run with per-sample lengths
instead (`lengths=` / `prompt_lens=`): the "same" convolutions read zeros past each sample's end, the
attentions take only a sample's own keys (ops.attention kv_lens), the predictor's GroupNorms take only its own rows, and
padded output rows are exact zeros, so every sample's output is bit-identical to running it alone, unpadded.  What the
padded input rows hold is never read into a valid row.
The two encoders also train with lengths (not with train_dropout: the attention has no key-padded dropout kernel).  The
record keeps the lengths and the backward undoes each row mask of the forward on the gradient (ops.mask_rows), runs the
attention backward with the same key counts (ops.attention_bwd kv_lens: d K / d V rows past them are exact zeros), and
so every parameter gradient is the sum of the per-sample-alone gradients (up to the fp32 summation order of the dQ and
weight-gradient reductions), every input gradient is the alone one, and the gradient of a padded prompt row - or of a
token-table row that only padded ids reach - is exactly zero.  The duration / pitch predictor takes lengths for
sampling only.  Numerics follow the denoiser: bf16 tensor-core operands, fp32 accumulation, fp32 residual stream and norm
statistics.
"""
from __future__ import annotations

from typing import Dict, Optional, Sequence, Tuple

import torch
import torch.nn.functional as F
from torch import nn

from . import _lib, ops
from .ops import conv_segs as _conv_segs
from .model import (_AttentionParams, _NoParam, _PackedCache, _RMSNormParams, _bf, _feedforward_params, _pack_conv,
                    _pack_geglu, _records_graph, _transpose_conv)
from .training import attention_backward, conv_backward, ff_backward, linear_backward, param_grads

_SILU = _lib.NS2_GEMM_FLAG_SILU


class _PlainTransformerParams(nn.Module):
    """Parameter holder of `Transformer` (ns2.py:1073-1108): layers.{l} = [RMSNorm, Attention, RMSNorm, FeedForward]."""

    def __init__(self, dim: int, depth: int, dim_head: int, heads: int, ff_mult: int = 4, final_norm: bool = False):
        super().__init__()
        self.layers = nn.ModuleList([
            nn.ModuleList([_RMSNormParams(dim), _AttentionParams(dim, dim_head, heads), _RMSNormParams(dim),
                           _feedforward_params(dim, ff_mult, causal_conv=False)])
            for _ in range(depth)])
        self.norm = _RMSNormParams(dim) if final_norm else nn.Identity()


_INPUT_GRADS = "<inputs>"   # key of `_train_backward`'s result holding the gradients of the node's inputs


class _EncoderFunction(torch.autograd.Function):
    """One autograd node for a whole encoder: forward = the inference kernels keeping activations, backward = the
    hand-written kernels (`_train_backward`).  apply(enc, reducer, *inputs, *enc.parameters()): the arguments before
    the parameters are the module's inputs, handed to `_train_forward`; its output may be one tensor or a tuple.
    `_train_backward(record, *d_outs)` gets None for an output that received no gradient, and returns the parameter
    gradients (None for parameters it did not reach) and, under _INPUT_GRADS, a tuple of the inputs' gradients (absent:
    none).  `reducer` (parallel.GradReducer or None) receives the parameter gradients when the backward ends."""

    @staticmethod
    def forward(ctx, enc, reducer, *args):
        n_in = len(args) - sum(1 for _ in enc.parameters())
        ctx.set_materialize_grads(False)
        with torch.no_grad():
            out, saved = enc._train_forward(*args[:n_in])
        ctx.enc, ctx.reducer, ctx.saved, ctx.n_in = enc, reducer, saved, n_in
        return out

    @staticmethod
    def backward(ctx, *d_outs):
        with torch.no_grad():
            grads = ctx.enc._train_backward(ctx.saved, *d_outs)
        ctx.saved = None
        d_in = tuple(grads.pop(_INPUT_GRADS, None) or ())
        d_in += (None,) * (ctx.n_in - len(d_in))   # inputs without a gradient (ids, lengths) may be left out
        d_in = [d if need else None for d, need in zip(d_in, ctx.needs_input_grad[2:2 + ctx.n_in])]
        return (None, None, *d_in, *param_grads(ctx.enc, grads, ctx.reducer))


class _EncoderBase(_PackedCache):
    """The shared transformer forward / backward of the encoders."""

    def __init__(self):
        super().__init__()
        self.grad_reducer = None   # parallel.GradReducer: all-reduce of this encoder's gradients (data parallel)
        self.train_dropout = False   # draw the reference's dropout in train() mode (see the module docstring)
        self.attn_dropout = self.conv_dropout = 0.0

    def _dropout_seed(self) -> Optional[int]:
        """The call's 64-bit dropout seed, or None when this call draws no dropout (then nothing is drawn from the
        generator, so the random stream of a run without dropout is unchanged)."""
        if not (self.training and self.train_dropout and (self.attn_dropout > 0 or self.conv_dropout > 0)):
            return None
        return int(torch.randint(0, 2 ** 63 - 1, ()))

    def _attn_dropout(self, seed: Optional[int], layer: int):
        return None if seed is None else (seed, 1 + layer, self.attn_dropout)

    def _pack_transposed_transformer(self, P, T, depth: int) -> None:
        for l in range(depth):
            for k in ("qkv", "o", "w1", "w2"):
                T[f"l{l}_{k}"] = P[f"l{l}_{k}"].t().contiguous()

    def _train_forward(self, x: torch.Tensor, lens: Optional[torch.Tensor] = None):
        """`_forward` keeping the activations `_train_backward` reads -> (output, record)."""
        saved = {"lens": lens}
        return self._forward(x, saved, lens), saved

    # ---- transformer ----
    def _pack_transformer(self, P: Dict[str, torch.Tensor], tr: _PlainTransformerParams, dim: int) -> None:
        for l, (n1, attn, n2, ff) in enumerate(tr.layers):
            P[f"l{l}_g1"] = n1.gamma.detach().float().contiguous()
            P[f"l{l}_g2"] = n2.gamma.detach().float().contiguous()
            P[f"l{l}_qkv"] = _bf(torch.cat((attn.to_q.weight, attn.to_kv.weight), dim=0))
            P[f"l{l}_o"] = _bf(attn.to_out.weight)
            for k, v in _pack_geglu(ff[0], ff[-1]).items():
                P[f"l{l}_{k}"] = v
        if isinstance(tr.norm, _RMSNormParams):
            P["final_g"] = tr.norm.gamma.detach().float().contiguous()

    def _transformer(self, x: torch.Tensor, tr: _PlainTransformerParams, P, heads: int,
                     saved: Optional[dict] = None, seed: Optional[int] = None,
                     kv_lens: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Transformer.forward (ns2.py:1110-1115) on the fp32 residual stream x (B, N, D), updated in place.  With `saved`
        every layer's activations go to saved["layers"] in fresh tensors (`_transformer_backward` reads them).
        seed: the call's dropout seed (None = no attention dropout).  kv_lens: per-sample lengths (keys past them are
        not attended to; the rows past them hold finite values the caller ignores)."""
        keep = saved is not None
        if keep and "final_g" in P:
            raise NotImplementedError("training a Transformer with final_norm=True is not supported")
        B, N, D = x.shape
        dev = x.device
        e = lambda *s, dt=torch.bfloat16: torch.empty(*s, device=dev, dtype=dt)  # noqa: E731
        inner = heads * 64
        layers = []
        for l in range(len(tr.layers)):
            if keep or l == 0:   # inference reuses the first layer's buffers
                Dp = P[f"l{l}_w2"].shape[1]
                L = {"h1": e(B, N, D), "qkv": e(B, N, 3 * inner), "ao": e(B, N, inner), "ff_g": e(B, N, Dp),
                     "lse": e(B, heads, N, dt=torch.float32) if keep else None}
                L["h2"] = e(B, N, D) if keep else L["h1"]
                layers.append(L)
            if keep:
                L["x_in"] = x.clone()
            ops.rmsnorm_film(x, L["h1"], gamma=P[f"l{l}_g1"])
            qkv = ops.gemm(L["h1"], P[f"l{l}_qkv"], L["qkv"], n=3 * inner, epilogue=ops.EPI_BF16)
            ops.attention(qkv[:, :, :inner], qkv[:, :, inner:2 * inner], qkv[:, :, 2 * inner:], L["ao"], heads=heads,
                          lse=L["lse"], dropout=self._attn_dropout(seed, l), kv_lens=kv_lens)
            ops.gemm(L["ao"], P[f"l{l}_o"], x, n=D, epilogue=ops.EPI_F32, resid=x)
            if keep:
                L["x_mid"] = x.clone()
            ops.rmsnorm_film(x, L["h2"], gamma=P[f"l{l}_g2"])
            ops.gemm(L["h2"], P[f"l{l}_w1"], L["ff_g"], n=2 * Dp, epilogue=ops.EPI_GEGLU, bias=P[f"l{l}_b1"])
            ops.gemm(L["ff_g"], P[f"l{l}_w2"], x, n=D, epilogue=ops.EPI_F32, bias=P[f"l{l}_b2"], resid=x)
        if keep:
            saved["layers"] = layers
        if "final_g" in P:
            out = torch.empty_like(x)
            ops.rmsnorm_f32(x, out, P["final_g"])
            return out
        return x

    def _transformer_backward(self, layers: list, tr: _PlainTransformerParams, P, T, heads: int, dxr: torch.Tensor,
                              dxr_bf: torch.Tensor, grads: Dict[str, torch.Tensor], seed: Optional[int] = None,
                              kv_lens: Optional[torch.Tensor] = None) -> None:
        """Transformer backward (ns2.py:1110-1115): dxr (fp32 gradient of the output, updated in place) becomes the
        gradient of the input; dxr_bf its bf16 copy.  Parameter gradients go to `grads` under the reference's names.
        seed: the forward's dropout seed (its attention masks are regenerated).  kv_lens: the forward's per-sample
        lengths; rows of dxr past them that come in as zeros stay exact zeros (the layers are row-wise but for the
        attention, whose d K / d V rows past them are zeros, and a padded query with d O = 0 has dS = 0)."""
        _, N, D = dxr.shape

        def norm_backward(x_in, dh, gamma, key):
            grads[key] = dgamma = torch.zeros(D, device=dxr.device)
            ops.rmsnorm_film_bwd(x_in, dh, dxr, dxr_bf, rows_per_batch=N, gamma=gamma, dgamma=dgamma)

        for l in reversed(range(len(tr.layers))):
            L = layers[l]
            pfx = f"transformer.layers.{l}."
            # ---- feed-forward: x += W2 GEGLU(W1 RMSNorm(x) + b1) + b2 ----
            dh2 = ff_backward(dxr_bf, L["h2"], L["ff_g"], P, T, f"l{l}_", tr.layers[l][3][-1].weight.shape[1],
                              grads, pfx + "3.")
            norm_backward(L["x_mid"], dh2, P[f"l{l}_g2"], pfx + "2.gamma")
            # ---- attention: x += Wo attn(Wqkv RMSNorm(x)) ----
            dh1, _ = attention_backward(dxr_bf, L["h1"], L["ao"], L["lse"], L["qkv"], None, T[f"l{l}_o"], T[f"l{l}_qkv"],
                                        heads, grads, pfx + "1.", dropout=self._attn_dropout(seed, l), kv_lens=kv_lens)
            norm_backward(L["x_in"], dh1, P[f"l{l}_g1"], pfx + "0.gamma")

    def _conv_silu_backward(self, x_in: torch.Tensor, w: torch.Tensor, w_t: Optional[torch.Tensor], bias: torch.Tensor,
                            d_out: torch.Tensor, first_shift: int, grads: Dict[str, torch.Tensor], name: str,
                            dtype=torch.bfloat16) -> Optional[torch.Tensor]:
        """Backward of out = silu(conv_k(x_in) + bias) (segmented GEMM): d_out bf16 (B, N, C_out) -> weight / bias
        gradients under `name`, and d x_in ((B, N, C_in) of `dtype`) when the transposed pack w_t is given."""
        B, N, c_in = x_in.shape
        c_out = w.shape[0]
        k = w.shape[1] // c_in
        pre = ops.gemm(x_in, w, torch.empty(B, N, c_out, device=x_in.device, dtype=torch.bfloat16), n=c_out,
                       epilogue=ops.EPI_BF16, segs=_conv_segs(c_in, k, first_shift), bias=bias)   # recompute
        ops.silu_bwd(pre, d_out)                                                                  # pre <- d pre
        return conv_backward(pre, x_in, grads, name, w_t, k, first_shift, dtype=dtype)

    def _records(self, *inputs) -> bool:
        """Whether a call records the `_EncoderFunction` node: train mode with gradients on, and a parameter or an input
        that requires grad (with every parameter frozen the node still carries the inputs' gradients)."""
        return _records_graph(self) or (self.training and torch.is_grad_enabled() and
                                        any(t.requires_grad for t in inputs))

    def _ragged_lengths(self, lengths, batch: int, n: int, device, name: str) -> Optional[torch.Tensor]:
        """Validated int32 device lengths of a call (None stays None).  Not with train_dropout in train mode: the
        attention has no key-padded dropout kernel, and the phoneme conv dropout's counter is the flat element index."""
        if lengths is None:
            return None
        if self.training and self.train_dropout:
            raise NotImplementedError(f"{type(self).__name__}: {name} are not supported together with train_dropout")
        return ops.lengths(lengths, batch, n, device=device, name=name)

    def _start_backward(self, d_out: torch.Tensor, lens: Optional[torch.Tensor] = None):
        dxr = d_out.float().contiguous().clone()        # fp32 residual-stream gradient, updated in place
        if lens is not None:                            # the forward zeroed the output rows past the lengths
            ops.mask_rows(dxr, lens)
        return dxr, ops.cast_bf16(dxr, torch.empty(dxr.shape, device=dxr.device, dtype=torch.bfloat16))


def _check_transformer_dims(dim: int, dim_head: int):
    if dim_head != 64:
        raise NotImplementedError("the sm_90a attention kernel is specialised for dim_head=64")
    if dim % 128 != 0 or dim > 1024:
        raise NotImplementedError("transformer dim must be a multiple of 128 (<= 1024) for the sm_90a kernels")


class SpeechPromptEncoder(_EncoderBase):
    """ns2.py:289-341.  forward(x: (B, Np, dim_codebook)) -> (B, Np, dims[-1]) fp32.
    forward(x, lengths=(B,)): sample b is x[b, :lengths[b]] (see the module docstring); rows past it come out as zeros,
    in training too (then d x rows past it are exact zeros)."""

    def __init__(self, dim_codebook, dims: Tuple[int, ...] = (256, 2048, 2048, 2048, 2048, 512, 512, 512), *,
                 depth=6, heads=8, dim_head=64, dropout=0.2, kernel_size=9, padding=4, use_flash_attn=True):
        super().__init__()
        dims = [dim_codebook, *dims]
        self.dim, self.dim_out = dims[0], dims[-1]
        if kernel_size > _lib.NS2_GEMM_MAX_SEGS:
            raise NotImplementedError(f"kernel_size must be <= {_lib.NS2_GEMM_MAX_SEGS}")
        if 2 * padding != kernel_size - 1:
            raise NotImplementedError("only 'same' padding (2*padding == kernel_size-1) keeps the sequence length")
        if any(d % 64 for d in dims):
            raise NotImplementedError("channel counts must be multiples of 64 (tensor-core K blocks)")
        _check_transformer_dims(dims[-1], dim_head)
        self.kernel_size, self.padding, self.heads = kernel_size, padding, heads
        self.attn_dropout = dropout   # the reference hands `dropout` to every Attention of its Transformer (ns2.py:332)
        mods = [_NoParam()]                                  # Rearrange('b n c -> b c n')
        for d_in, d_out in zip(dims[:-1], dims[1:]):
            mods.extend([nn.Conv1d(d_in, d_out, kernel_size, padding=padding), _NoParam()])   # conv, SiLU
        mods.append(_NoParam())                              # Rearrange back
        self.conv = nn.Sequential(*mods)
        self.transformer = _PlainTransformerParams(dims[-1], depth, dim_head, heads)

    def _convs(self):
        return [m for m in self.conv if isinstance(m, nn.Conv1d)]

    def _pack(self) -> Dict[str, torch.Tensor]:
        P: Dict[str, torch.Tensor] = {}
        for i, c in enumerate(self._convs()):
            P[f"c{i}_w"] = _pack_conv(c.weight)
            P[f"c{i}_b"] = c.bias.detach().float().contiguous()
        self._pack_transformer(P, self.transformer, self.dim_out)
        return P

    def _pack_transposed(self, P) -> Dict[str, torch.Tensor]:
        T = {f"c{i}_w": _transpose_conv(P[f"c{i}_w"], self.kernel_size) for i in range(len(self._convs()))}
        self._pack_transposed_transformer(P, T, len(self.transformer.layers))
        return T

    def forward(self, x: torch.Tensor, *, lengths=None) -> torch.Tensor:
        assert x.shape[-1] == self.dim
        if not x.is_cuda:
            raise ValueError("SpeechPromptEncoder: input must be a CUDA tensor (the ns2_b200 ops have no CPU path)")
        lens = self._ragged_lengths(lengths, x.shape[0], x.shape[1], x.device, "lengths")
        if self._records(x):
            return _EncoderFunction.apply(self, self.grad_reducer, x, lens, *self.parameters())
        with torch.no_grad():
            return self._forward(x, lens=lens)

    def _forward(self, x: torch.Tensor, saved: Optional[dict] = None, lens: Optional[torch.Tensor] = None) -> torch.Tensor:
        """The forward; with `saved` it also records the activations `_train_backward` reads (same kernels, same output).
        lens: per-sample lengths; every conv input is zero past them, as the "same" padding of a sample run alone."""
        P = self.packed()
        B, N, _ = x.shape
        dev, bf = x.device, torch.bfloat16
        h = ops.cast_bf16(x.float().contiguous(), torch.empty(B, N, self.dim, device=dev, dtype=bf))
        if lens is not None:
            ops.mask_rows(h, lens)
        convs = self._convs()
        conv_in = []
        for i, c in enumerate(convs):
            last = i == len(convs) - 1
            out = torch.empty(B, N, c.out_channels, device=dev, dtype=torch.float32 if last else bf)
            ops.gemm(h, P[f"c{i}_w"], out, n=c.out_channels, epilogue=ops.EPI_F32 if last else ops.EPI_BF16,
                     segs=_conv_segs(c.in_channels, self.kernel_size, self.padding), bias=P[f"c{i}_b"], flags=_SILU)
            if lens is not None:
                ops.mask_rows(out, lens)
            if saved is not None:
                conv_in.append(h)
            h = out
        seed = self._dropout_seed()
        if saved is not None:
            saved.update(conv_in=conv_in, dropout_seed=seed)
        out = self._transformer(h, self.transformer, P, self.heads, saved, seed, kv_lens=lens)
        return out if lens is None else ops.mask_rows(out, lens)

    def _train_forward(self, x: torch.Tensor, lens: Optional[torch.Tensor] = None):
        saved = {"x_requires_grad": x.requires_grad, "x_dtype": x.dtype, "lens": lens}
        return self._forward(x, saved, lens), saved

    def _train_backward(self, S, d_out: torch.Tensor) -> Dict[str, torch.Tensor]:
        P, T = self.packed(), self.packed_transposed()
        grads: Dict[str, torch.Tensor] = {}
        lens = S["lens"]
        dxr, dxr_bf = self._start_backward(d_out, lens)
        self._transformer_backward(S["layers"], self.transformer, P, T, self.heads, dxr, dxr_bf, grads,
                                   S["dropout_seed"], kv_lens=lens)
        d_h = dxr_bf                        # gradient of the last conv's (SiLU) output
        need_dx = S["x_requires_grad"]
        for i in reversed(range(len(self._convs()))):
            # conv i is module conv.{2i+1} (Rearrange, then [Conv1d, SiLU] pairs); conv 0's d x (fp32) only when the
            # prompt requires grad (it usually comes from the codec)
            first = i == 0
            w_t = T[f"c{i}_w"] if need_dx or not first else None
            if lens is not None:            # the forward zeroed this conv's output past the lengths
                ops.mask_rows(d_h, lens)
            d_h = self._conv_silu_backward(S["conv_in"][i], P[f"c{i}_w"], w_t, P[f"c{i}_b"], d_h, self.padding, grads,
                                           f"conv.{2 * i + 1}", dtype=torch.float32 if first else torch.bfloat16)
        if need_dx:
            if lens is not None:            # ... and its input (the "same" conv's dgrad spreads into the padding)
                ops.mask_rows(d_h, lens)
            grads[_INPUT_GRADS] = (d_h.to(S["x_dtype"]),)
        return grads


class PhonemeEncoder(_EncoderBase):
    """ns2.py:228-287.  forward(x: (B, T) int64 phoneme ids, negative = padding) -> (B, T, dim_hidden) fp32.
    A tokenizer (List[str] input) is used exactly like the reference when one is given.
    forward(x, lengths=(B,)): sample b is x[b, :lengths[b]] (see the module docstring); rows past it come out as zeros,
    in training too (then the token-table rows that only padded ids reach get exact-zero gradients)."""

    def __init__(self, *, tokenizer=None, num_tokens=None, dim=512, dim_hidden=512, kernel_size=9, depth=6,
                 dim_head=64, heads=8, conv_dropout=0.2, attn_dropout=0., use_flash=False):
        super().__init__()
        self.tokenizer = tokenizer
        if num_tokens is None and tokenizer is not None:
            num_tokens = tokenizer.vocab_size
        if num_tokens is None:
            raise NotImplementedError("PhonemeEncoder without a token table (nn.Identity embedding) is not supported")
        if kernel_size > _lib.NS2_GEMM_MAX_SEGS:
            raise NotImplementedError(f"kernel_size must be <= {_lib.NS2_GEMM_MAX_SEGS}")
        if dim % 64:
            raise NotImplementedError("dim must be a multiple of 64 (tensor-core K blocks)")
        _check_transformer_dims(dim_hidden, dim_head)
        self.dim, self.dim_hidden, self.kernel_size, self.heads = dim, dim_hidden, kernel_size, heads
        self.conv_dropout, self.attn_dropout = conv_dropout, attn_dropout
        self.token_emb = nn.Embedding(num_tokens + 1, dim)
        self.pad_id = num_tokens
        self.conv = nn.Sequential(_NoParam(), nn.Conv1d(dim, dim_hidden, kernel_size), _NoParam(), _NoParam(), _NoParam())
        self.transformer = _PlainTransformerParams(dim_hidden, depth, dim_head, heads)

    def _pack(self) -> Dict[str, torch.Tensor]:
        c = self.conv[1]
        P = {"emb": self.token_emb.weight.detach().float().contiguous(), "c_w": _pack_conv(c.weight),
             "c_b": c.bias.detach().float().contiguous()}
        self._pack_transformer(P, self.transformer, self.dim_hidden)
        return P

    def _pack_transposed(self, P) -> Dict[str, torch.Tensor]:
        T = {"c_w": _transpose_conv(P["c_w"], self.kernel_size)}
        self._pack_transposed_transformer(P, T, len(self.transformer.layers))
        return T

    def forward(self, x, mask=None, *, lengths=None) -> torch.Tensor:
        if mask is not None:
            raise NotImplementedError("PhonemeEncoder: attention masks are not supported by the sm_90a attention kernel")
        if isinstance(x, (list, tuple)):
            assert self.tokenizer is not None
            x = self.tokenizer.texts_to_tensor_ids(x).to(self.token_emb.weight.device)
        if not x.is_cuda:
            raise ValueError("PhonemeEncoder: input must be a CUDA tensor (the ns2_b200 ops have no CPU path)")
        lens = self._ragged_lengths(lengths, x.shape[0], x.shape[1], x.device, "lengths")
        if self._records():   # ids have no gradient
            return _EncoderFunction.apply(self, self.grad_reducer, x, lens, *self.parameters())
        with torch.no_grad():
            return self._forward(x, lens=lens)

    def _forward(self, x: torch.Tensor, saved: Optional[dict] = None, lens: Optional[torch.Tensor] = None) -> torch.Tensor:
        """The forward; with `saved` it also records the activations `_train_backward` reads (same kernels, same output)."""
        P = self.packed()
        B, T = x.shape
        dev, bf = x.device, torch.bfloat16
        ids = x.long().contiguous()
        e = ops.embedding_bf16(ids, P["emb"], torch.empty(B, T, self.dim, device=dev, dtype=bf), self.pad_id)
        h = torch.empty(B, T, self.dim_hidden, device=dev, dtype=torch.float32)
        # CausalConv1d: left padding dilation*(k-1) (ns2.py:592-595) -> tap t reads position n - (k-1-t)
        ops.gemm(e, P["c_w"], h, n=self.dim_hidden, epilogue=ops.EPI_F32,
                 segs=_conv_segs(self.dim, self.kernel_size, self.kernel_size - 1), bias=P["c_b"], flags=_SILU)
        seed = self._dropout_seed()
        if seed is not None:
            ops.dropout_(h, dropout=(seed, 0, self.conv_dropout))                   # nn.Dropout(conv_dropout), ns2.py:258
        if saved is not None:
            saved.update(ids=ids, emb=e, dropout_seed=seed)
        # the conv is causal: a valid row never reads a padded one, only the attention needs the lengths
        out = self._transformer(h, self.transformer, P, self.heads, saved, seed, kv_lens=lens)
        return out if lens is None else ops.mask_rows(out, lens)

    def _train_backward(self, S, d_out: torch.Tensor) -> Dict[str, torch.Tensor]:
        P, T = self.packed(), self.packed_transposed()
        grads: Dict[str, torch.Tensor] = {}
        # with lengths: the output gradient is masked like the output; the causal conv and the zero d K / d V rows keep
        # every padded row's gradient an exact zero from there on, so embedding_bwd adds nothing for padded ids
        dxr, dxr_bf = self._start_backward(d_out, S["lens"])
        seed = S["dropout_seed"]
        self._transformer_backward(S["layers"], self.transformer, P, T, self.heads, dxr, dxr_bf, grads, seed,
                                   kv_lens=S["lens"])
        if seed is not None and self.conv_dropout > 0:   # the conv's dropout mask, on the fp32 gradient
            ops.cast_bf16(ops.dropout_(dxr, dropout=(seed, 0, self.conv_dropout)), dxr_bf)
        d_e = self._conv_silu_backward(S["emb"], P["c_w"], T["c_w"], P["c_b"], dxr_bf, self.kernel_size - 1, grads,
                                       "conv.1", dtype=torch.float32)
        grads["token_emb.weight"] = ops.embedding_bwd(S["ids"], d_e, torch.zeros_like(P["emb"]), self.pad_id)
        return grads


# --------------------------------------------------------------------------------------------------
# duration / pitch predictor (ns2.py:345-527)
# --------------------------------------------------------------------------------------------------
class _BlockParams(nn.Module):
    """Block (ns2.py:345-365): proj = Conv1d(k, padding k//2), norm = GroupNorm(groups, dim_out)."""

    def __init__(self, dim, dim_out, kernel, groups):
        super().__init__()
        self.proj = nn.Conv1d(dim, dim_out, kernel, padding=kernel // 2)
        self.norm = nn.GroupNorm(groups, dim_out)


class _ResnetBlockParams(nn.Module):
    """ResnetBlock (ns2.py:367-401) with dim == dim_out (res_conv = Identity, the only shape the trunk builds)."""

    def __init__(self, dim, kernel, groups=8, num_convs=2):
        super().__init__()
        self.blocks = nn.Sequential(*[_BlockParams(dim, dim, kernel, groups) for _ in range(num_convs)])
        self.res_conv = nn.Identity()


class _TrunkParams(nn.Module):
    """DurationPitchPredictorTrunk (ns2.py:412-456)."""

    def __init__(self, dim, depth, kernel_size, dim_context, heads, dim_head, num_convs_per_resnet_block,
                 num_convolutions_per_block):
        super().__init__()
        self.layers = nn.ModuleList([])
        for _ in range(depth):
            attn = _AttentionParams(dim, dim_head, heads)
            if dim_context is not None and dim_context != dim:
                attn.to_kv = nn.Linear(dim_context, dim_head * heads * 2, bias=False)
            self.layers.append(nn.ModuleList([
                nn.Sequential(*[_ResnetBlockParams(dim, kernel_size, num_convs=num_convs_per_resnet_block)
                                for _ in range(num_convolutions_per_block)]),
                _RMSNormParams(dim),
                attn]))
        self.to_pred = nn.Sequential(nn.Linear(dim, 1), _NoParam(), _NoParam())


class DurationPitchPredictor(_EncoderBase):
    """ns2.py:468-527.  forward(x: (B, T, dim_hidden) phoneme encodings [or (B, T) ids with a token table],
    encoded_prompts: (B, Np, dim_encoded_prompts)) -> (duration_pred (B, T), pitch_pred (B, T)), both fp32 >= 0.
    forward(..., lengths=(B,), prompt_lens=(B,)): sample b is x[b, :lengths[b]] with the prompt encoded_prompts[b,
    :prompt_lens[b]] (see the module docstring); its predictions past lengths[b] are exact zeros."""

    def __init__(self, *, dim, num_phoneme_tokens=None, tokenizer=None, dim_encoded_prompts=None,
                 num_convolutions_per_block=3, use_resnet_block=True, num_convs_per_resnet_block=2, depth=10,
                 kernel_size=3, heads=8, dim_head=64, dim_hidden=512, dropout=0.2, use_flash_attn=False):
        super().__init__()
        self.tokenizer = tokenizer
        if num_phoneme_tokens is None and tokenizer is not None:
            num_phoneme_tokens = tokenizer.vocab_size
        dim_encoded_prompts = dim if dim_encoded_prompts is None else dim_encoded_prompts
        if not use_resnet_block:
            raise NotImplementedError("only the ResnetBlock trunk (the reference default) is built")
        if kernel_size % 2 != 1 or kernel_size > _lib.NS2_GEMM_MAX_SEGS:
            raise NotImplementedError("kernel_size must be odd and <= NS2_GEMM_MAX_SEGS")
        _check_transformer_dims(dim_hidden, dim_head)
        if dim_encoded_prompts != dim_hidden:
            # keys = cat(norm(x), encoded_prompts) along the sequence (cross_attn_include_queries, ns2.py:1060-1061)
            raise NotImplementedError("dim_encoded_prompts must equal dim_hidden (the reference concatenates them)")
        if num_phoneme_tokens is not None and dim != dim_hidden:
            raise NotImplementedError("the token table width must equal dim_hidden")
        self.dim_hidden, self.heads, self.kernel_size = dim_hidden, heads, kernel_size
        # the reference's `dropout` goes to every cross Attention only (ns2.py:438-446); its Blocks keep p = 0
        # (conv_dropout stays 0); drawn only with train_dropout, see the module docstring
        self.attn_dropout, self.depth = float(dropout), depth
        self.phoneme_token_emb = nn.Embedding(num_phoneme_tokens, dim) if num_phoneme_tokens is not None else nn.Identity()
        mk = lambda: _TrunkParams(dim_hidden, depth, kernel_size, dim_encoded_prompts, heads, dim_head,  # noqa: E731
                                  num_convs_per_resnet_block, num_convolutions_per_block)
        self.to_pitch_pred = mk()
        self.to_duration_pred = mk()

    def _pack(self) -> Dict[str, torch.Tensor]:
        P: Dict[str, torch.Tensor] = {}
        for name, trunk in (("p", self.to_pitch_pred), ("d", self.to_duration_pred)):
            for l, (convs, norm, attn) in enumerate(trunk.layers):
                for r, rb in enumerate(convs):
                    for c, blk in enumerate(rb.blocks):
                        k = f"{name}{l}_{r}_{c}"
                        P[k + "_w"] = _pack_conv(blk.proj.weight)
                        P[k + "_b"] = blk.proj.bias.detach().float().contiguous()
                        P[k + "_gw"] = blk.norm.weight.detach().float().contiguous()
                        P[k + "_gb"] = blk.norm.bias.detach().float().contiguous()
                P[f"{name}{l}_g"] = norm.gamma.detach().float().contiguous()
                P[f"{name}{l}_q"] = _bf(attn.to_q.weight)
                P[f"{name}{l}_kv"] = _bf(attn.to_kv.weight)
                P[f"{name}{l}_o"] = _bf(attn.to_out.weight)
            P[f"{name}_pw"] = trunk.to_pred[0].weight.detach().float().reshape(-1).contiguous()
            P[f"{name}_pb"] = trunk.to_pred[0].bias.detach().float().contiguous()
        if isinstance(self.phoneme_token_emb, nn.Embedding):
            P["emb"] = self.phoneme_token_emb.weight.detach().float().contiguous()
        return P

    def _pack_transposed(self, P) -> Dict[str, torch.Tensor]:
        T = {}
        for name, trunk in (("p", self.to_pitch_pred), ("d", self.to_duration_pred)):
            for l, (convs, _, _) in enumerate(trunk.layers):
                for r, rb in enumerate(convs):
                    for c in range(len(rb.blocks)):
                        k = f"{name}{l}_{r}_{c}_w"
                        T[k] = _transpose_conv(P[k], self.kernel_size)
                for w in ("q", "kv", "o"):
                    T[f"{name}{l}_{w}"] = P[f"{name}{l}_{w}"].t().contiguous()
        return T

    @staticmethod
    def _norm_config(trunk: _TrunkParams):
        """(groups, eps) of the trunk's GroupNorms (every Block of a trunk is built alike)."""
        if not len(trunk.layers):
            return 8, 1e-5
        norm = trunk.layers[0][0][0].blocks[0].norm
        return norm.num_groups, norm.eps

    def _cross_attn_dropout(self, seed: Optional[int], name: str, l: int):
        """(seed, site, p) of the cross attention of layer l of trunk `name`: site t depth + l, t = 0 for the duration
        trunk and 1 for the pitch trunk (None without a seed)."""
        t = 0 if name == "d" else 1
        return None if seed is None else (seed, t * self.depth + l, self.attn_dropout)

    def _trunk(self, name: str, trunk: _TrunkParams, P, x0: torch.Tensor, prompts_bf: torch.Tensor,
               saved: Optional[dict] = None, seed: Optional[int] = None, ragged: Optional[tuple] = None) -> torch.Tensor:
        """DurationPitchPredictorTrunk.forward (ns2.py:457-466).  With `saved` the activations `_trunk_backward` reads
        go to saved[name] in fresh tensors (same kernels, same output).  seed: the call's dropout seed (None = none).
        ragged: (lengths, prompt_lens, lengths + prompt_lens) of a batch of different lengths; x0 must be zero past
        the lengths.  Then the stream's bf16 copy that the "same" convs read is kept zero there (the GroupNorms write
        zeros), the keys are the packed prefix [norm(x)[:T_b] ; prompts[:Np_b]], and the predictions past T_b are 0."""
        keep = saved is not None
        B, T, D = x0.shape
        Np = prompts_bf.shape[1]
        dev, bf, H = x0.device, torch.bfloat16, self.heads
        inner = H * 64
        groups, eps = self._norm_config(trunk)
        segs = _conv_segs(D, self.kernel_size, self.kernel_size // 2)
        e = lambda *s, dt=bf: torch.empty(*s, device=dev, dtype=dt)  # noqa: E731
        lens, plens, kv_lens = ragged if ragged is not None else (None, None, None)
        x = x0.clone()                                               # fp32 stream of this trunk
        x_bf = ops.cast_bf16(x, e(B, T, D))
        c = e(B, T, D, dt=torch.float32)
        h_bf = e(B, T, D)
        layers = []
        for l, (convs, _, _) in enumerate(trunk.layers):
            if keep or l == 0:   # inference reuses the first layer's buffers
                ctx = e(B, T + Np, D)                                # [norm(x) ; encoded prompts] (ns2.py:1060-1061)
                if ragged is None:
                    ctx[:, T:].copy_(prompts_bf)
                L = {"nx": e(B, T, D), "q": e(B, T, inner), "kv": e(B, T + Np, 2 * inner), "o": e(B, T, inner),
                     "ctx": ctx, "lse": e(B, H, T, dt=torch.float32) if keep else None, "blocks": []}
            for r, rb in enumerate(convs):
                nb = len(rb.blocks)
                src = x_bf
                for ci in range(nb):
                    k = f"{name}{l}_{r}_{ci}"
                    ops.gemm(src, P[k + "_w"], c, n=D, epilogue=ops.EPI_F32, segs=segs, bias=P[k + "_b"])
                    if keep:
                        L["blocks"].append((src.clone(), c.clone()))   # conv input (bf16), GroupNorm input (fp32)
                    if ci < nb - 1:
                        ops.groupnorm_silu(c, P[k + "_gw"], P[k + "_gb"], groups, eps=eps, out_bf16=h_bf, lens=lens)
                        src = h_bf
                    else:   # out = blocks(x) + res_conv(x), res_conv = Identity (ns2.py:399-401)
                        ops.groupnorm_silu(c, P[k + "_gw"], P[k + "_gb"], groups, eps=eps, resid=x, out_f32=x,
                                           out_bf16=x_bf, lens=lens)
            if keep:
                L["x_mid"] = x.clone()
                layers.append(L)
            nx, q, kv, o, ctx = L["nx"], L["q"], L["kv"], L["o"], L["ctx"]
            ops.rmsnorm_film(x, nx, gamma=P[f"{name}{l}_g"])
            if ragged is None:
                ctx[:, :T].copy_(nx)
            else:
                ops.pack_rows(nx, lens, prompts_bf, plens, ctx)
            ops.gemm(nx, P[f"{name}{l}_q"], q, n=inner, epilogue=ops.EPI_BF16)
            ops.gemm(ctx, P[f"{name}{l}_kv"], kv, n=2 * inner, epilogue=ops.EPI_BF16)
            ops.attention(q, kv[:, :, :inner], kv[:, :, inner:], o, heads=H, lse=L["lse"],
                          dropout=self._cross_attn_dropout(seed, name, l), kv_lens=kv_lens)
            ops.gemm(o, P[f"{name}{l}_o"], x, n=D, epilogue=ops.EPI_F32, resid=x)   # attn(norm(x), prompts) + x
            ops.cast_bf16(x, x_bf)
            if ragged is not None:   # the next ResnetBlock's first conv reads it
                ops.mask_rows(x_bf, lens)
        pred = e(B, T, dt=torch.float32)
        ops.rowdot(x, P[f"{name}_pw"], P[f"{name}_pb"], pred, relu=True)            # Linear(dim, 1) + ReLU
        if ragged is not None:
            ops.mask_rows(pred.view(B, T, 1), lens)
        if keep:
            saved[name] = {"layers": layers, "x": x, "pred": pred.clone()}
        return pred

    def _trunk_backward(self, name: str, trunk: _TrunkParams, P, T, S: dict, d_pred: torch.Tensor,
                        d_prompts: torch.Tensor, grads: Dict[str, torch.Tensor], pfx: str,
                        seed: Optional[int] = None) -> torch.Tensor:
        """Backward of `_trunk` from d pred (B, T): parameter gradients go to `grads` under pfx + the reference's names,
        d prompts (B, Np, D) f32 is accumulated in place; returns d x0 (B, T, D) f32.  seed: the forward's dropout seed
        (its masks are regenerated)."""
        x = S["x"]
        B, Tn, D = x.shape
        Np = d_prompts.shape[1]
        dev, bf, H = x.device, torch.bfloat16, self.heads
        inner = H * 64
        k, half = self.kernel_size, self.kernel_size // 2
        groups, eps = self._norm_config(trunk)
        dgrad_segs = ops.conv_dgrad_segs(D, k, half)
        e = lambda *s, dt=bf: torch.empty(*s, device=dev, dtype=dt)  # noqa: E731
        dxr = torch.zeros_like(x)                     # fp32 gradient of the trunk's residual stream
        dxr_bf, dh, d_c = e(B, Tn, D), e(B, Tn, D), e(B, Tn, D)
        d_kv = e(B, Tn + Np, 2 * inner)
        # ---- to_pred: ReLU(Linear(dim, 1)) (ns2.py:451-455) ----
        grads[pfx + "to_pred.0.weight"], grads[pfx + "to_pred.0.bias"] = ops.rowdot_bwd(
            x, P[f"{name}_pw"], S["pred"], d_pred.float().contiguous(), dxr)
        for l in reversed(range(len(trunk.layers))):
            L = S["layers"][l]
            lp = f"{pfx}layers.{l}."
            # ---- x += Wo attn(Wq nx, Wkv [nx ; prompts]), nx = RMSNorm(x): the keys include the queries ----
            ops.cast_bf16(dxr, dxr_bf)
            d_nx, _ = attention_backward(dxr_bf, L["nx"], L["o"], L["lse"], L["q"], L["kv"], T[f"{name}{l}_o"],
                                         T[f"{name}{l}_q"], H, grads, lp + "2.", d_kv=d_kv,
                                         dropout=self._cross_attn_dropout(seed, name, l))
            linear_backward(d_kv, L["ctx"], grads, lp + "2.to_kv", bias=False)
            # d ctx = d kv Wkv, split: the first Tn rows join the query path's d nx, the rest is d prompts
            d_nx32 = ops.gemm(d_kv[:, :Tn], T[f"{name}{l}_kv"], e(B, Tn, D, dt=torch.float32), n=D, epilogue=ops.EPI_F32)
            ops.gemm(d_kv[:, Tn:], T[f"{name}{l}_kv"], d_prompts, n=D, epilogue=ops.EPI_F32, resid=d_prompts)
            ops.accum_bf16(d_nx32, d_nx, dh)
            grads[lp + "1.gamma"] = dgamma = torch.zeros(D, device=dev)
            ops.rmsnorm_film_bwd(L["x_mid"], dh, dxr, dxr_bf, rows_per_batch=Tn, gamma=P[f"{name}{l}_g"], dgamma=dgamma)
            # ---- ResnetBlocks in reverse: out = blocks(x) + x (ns2.py:397-401) ----
            convs = trunk.layers[l][0]
            i = len(L["blocks"])
            for r in reversed(range(len(convs))):
                dy = dxr                              # d out of the last Block; the identity keeps dxr as it is
                for ci in reversed(range(len(convs[r].blocks))):
                    i -= 1
                    src, c = L["blocks"][i]
                    key, bp = f"{name}{l}_{r}_{ci}", f"{lp}0.{r}.blocks.{ci}."
                    grads[bp + "norm.weight"], grads[bp + "norm.bias"] = ops.groupnorm_silu_bwd(
                        c, P[key + "_gw"], P[key + "_gb"], groups, dy, d_c, eps=eps)
                    conv_backward(d_c, src, grads, bp + "proj", None, k, half)
                    if ci > 0:
                        dy = ops.gemm(d_c, T[key + "_w"], e(B, Tn, D, dt=torch.float32), n=D, epilogue=ops.EPI_F32,
                                      segs=dgrad_segs)
                    else:   # the first conv reads the ResnetBlock's input: its d x joins the identity path's
                        ops.gemm(d_c, T[key + "_w"], dxr, n=D, epilogue=ops.EPI_F32, segs=dgrad_segs, resid=dxr)
        return dxr

    def forward(self, x, encoded_prompts: torch.Tensor, prompt_mask=None, *, lengths=None, prompt_lens=None):
        if prompt_mask is not None:
            raise NotImplementedError("DurationPitchPredictor: prompt masks are not supported by the sm_90a attention kernel")
        if isinstance(x, (list, tuple)):
            assert self.tokenizer is not None
            x = self.tokenizer.texts_to_tensor_ids(x).to(encoded_prompts.device)
        if not (x.is_cuda and encoded_prompts.is_cuda):
            raise ValueError("DurationPitchPredictor: inputs must be CUDA tensors (the ns2_b200 ops have no CPU path)")
        ragged = None
        if lengths is not None or prompt_lens is not None:
            B, T = x.shape[:2]
            Np = encoded_prompts.shape[1]
            if self._records(x, encoded_prompts):
                raise NotImplementedError("DurationPitchPredictor: lengths / prompt_lens are supported for sampling only "
                                          "(no autograd)")
            lens = self._ragged_lengths(lengths if lengths is not None else [T] * B, B, T, x.device, "lengths")
            plens = self._ragged_lengths(prompt_lens if prompt_lens is not None else [Np] * B, B, Np, x.device,
                                         "prompt_lens")
            ragged = (lens, plens, lens + plens)
        if self._records(x, encoded_prompts):
            return _EncoderFunction.apply(self, self.grad_reducer, x, encoded_prompts, *self.parameters())
        with torch.no_grad():
            return self._forward(x, encoded_prompts, ragged=ragged)

    def _train_forward(self, x: torch.Tensor, encoded_prompts: torch.Tensor):
        saved = {"x_dtype": x.dtype, "prompts_dtype": encoded_prompts.dtype}
        return self._forward(x, encoded_prompts, saved), saved

    def _forward(self, x: torch.Tensor, encoded_prompts: torch.Tensor, saved: Optional[dict] = None,
                 ragged: Optional[tuple] = None):
        """The forward; with `saved` it also records what `_train_backward` reads (same kernels, same output).
        ragged: see `_trunk`; the input rows past the lengths are replaced by zeros (a copy, the input is not touched)."""
        P = self.packed()
        dev, bf = x.device, torch.bfloat16
        if "emb" in P:
            B, T = x.shape
            ids = x.long().contiguous()
            e = ops.embedding_bf16(ids, P["emb"], torch.empty(B, T, self.dim_hidden, device=dev, dtype=bf), 0)
            if ragged is not None:
                ops.mask_rows(e, ragged[0])
            x = e.float()
            if saved is not None:
                saved["ids"] = ids
        elif ragged is not None:
            x = ops.mask_rows(x.float().clone(memory_format=torch.contiguous_format), ragged[0])
        x = x.float().contiguous()
        B, Np, Dp = encoded_prompts.shape
        assert x.shape[-1] == self.dim_hidden and Dp == self.dim_hidden
        prompts_bf = ops.cast_bf16(encoded_prompts.float().contiguous(), torch.empty(B, Np, Dp, device=dev, dtype=bf))
        seed = self._dropout_seed()
        if saved is not None:
            saved["dropout_seed"] = seed
        duration = self._trunk("d", self.to_duration_pred, P, x, prompts_bf, saved, seed, ragged)
        pitch = self._trunk("p", self.to_pitch_pred, P, x, prompts_bf, saved, seed, ragged)
        return duration, pitch

    def _train_backward(self, S, d_duration: Optional[torch.Tensor], d_pitch: Optional[torch.Tensor]):
        """Gradients of every parameter and of (x, encoded_prompts) given d duration_pred / d pitch_pred; a trunk whose
        prediction received no gradient is skipped and its parameters get None."""
        P, T = self.packed(), self.packed_transposed()
        grads: Dict[str, Optional[torch.Tensor]] = {}
        x = S["d"]["x"]
        B, Tn, D = x.shape
        Np = S["d"]["layers"][0]["ctx"].shape[1] - Tn if len(self.to_duration_pred.layers) else 0
        d_prompts = torch.zeros(B, Np, D, device=x.device)
        dx = None
        for name, trunk, pfx, d in (("d", self.to_duration_pred, "to_duration_pred.", d_duration),
                                    ("p", self.to_pitch_pred, "to_pitch_pred.", d_pitch)):
            if d is None:
                grads.update({pfx + n: None for n, _ in trunk.named_parameters()})
                continue
            dx_t = self._trunk_backward(name, trunk, P, T, S[name], d, d_prompts, grads, pfx, S["dropout_seed"])
            dx = dx_t if dx is None else dx.add_(dx_t)          # x feeds both trunks
        if "emb" in P:   # the ids get no gradient; the table does (pad id 0, as `_forward` gathers)
            grads["phoneme_token_emb.weight"] = ops.embedding_bwd(S["ids"], dx, torch.zeros_like(P["emb"]), 0)
            d_x = None
        else:
            d_x = dx.to(S["x_dtype"])
        grads[_INPUT_GRADS] = (d_x, d_prompts.to(S["prompts_dtype"]))
        return grads


# --------------------------------------------------------------------------------------------------
# the conditional front end of NaturalSpeech2.sample (ns2.py:1472-1483)
# --------------------------------------------------------------------------------------------------
def f0_to_coarse(f0: torch.Tensor, f0_bin: int = 256, f0_max: float = 1100.0, f0_min: float = 50.0) -> torch.Tensor:
    """ns2.py:164-177 — (B, T)-sized host-side glue kept in torch like the noise schedules."""
    f0_mel_max = 1127 * torch.log(1 + torch.tensor(f0_max) / 700)
    f0_mel_min = 1127 * torch.log(1 + torch.tensor(f0_min) / 700)
    f0_mel = 1127 * (1 + f0 / 700).log()
    pos = f0_mel > 0
    f0_mel = torch.where(pos, (f0_mel - f0_mel_min) * (f0_bin - 2) / (f0_mel_max - f0_mel_min) + 1, f0_mel)
    f0_mel = f0_mel.clamp(min=1, max=f0_bin - 1)
    return (f0_mel + 0.5).int()


def average_over_durations(values: torch.Tensor, durs: torch.Tensor) -> torch.Tensor:
    """Per-phoneme mean of frame-level values (utils/utils.py:4-26): values (B, C, L), durs (B, T) frame counts ->
    (B, C, T).  Only NONZERO frames are averaged (unvoiced pitch is 0); a phoneme without one gets 0.  Prefix sums over
    the frames, differenced at each phoneme's [start, end) — (B, T)-sized host glue like f0_to_coarse."""
    B, C, _ = values.shape
    end = durs.cumsum(dim=1).long()
    start = torch.cat((torch.zeros_like(end[:, :1]), end[:, :-1]), dim=1)
    gather_at = lambda t, at: t.gather(2, at[:, None, :].expand(B, C, at.shape[1]))  # noqa: E731
    zero_col = torch.zeros(B, C, 1, dtype=values.dtype, device=values.device)
    prefix = torch.cat((zero_col, values.cumsum(dim=2)), dim=2)
    voiced = torch.cat((zero_col.long(), (values != 0.0).cumsum(dim=2)), dim=2)
    total = (gather_at(prefix, end) - gather_at(prefix, start)).to(values.dtype)
    count = (gather_at(voiced, end) - gather_at(voiced, start)).to(values.dtype)
    return torch.where(count == 0.0, count, total / count).to(values.dtype)


def frames_to_text_index(duration: torch.Tensor, length: Optional[int] = None) -> torch.Tensor:
    """The hard alignment of generate_mask_from_repeats (ns2.py:87-104) as one text index per frame: (B, L) int32,
    L = `length` or else the max total duration, -1 past a sample's own length.  mask[b, i, n] of the reference ==
    (idx[b, n] == i)."""
    repeats = duration.int()
    cumsum = repeats.cumsum(dim=-1)
    lengths = cumsum[:, -1]
    L = int(lengths.amax().item()) if length is None else int(length)
    seq = torch.arange(L, device=duration.device).unsqueeze(0).expand(duration.shape[0], L).contiguous()
    idx = torch.searchsorted(cumsum, seq, right=True)          # first i with cumsum[i] > n
    idx = torch.where(seq < lengths.unsqueeze(-1), idx, torch.full_like(idx, -1))
    return idx.int().contiguous()


class _ExpandFunction(torch.autograd.Function):
    """Length regulation with a backward: d phoneme_enc and d pitch_table through ops.expand_encodings_bwd."""

    @staticmethod
    def forward(ctx, phoneme_enc, pitch_table, coarse, idx, reducer):
        ctx.save_for_backward(coarse, idx)
        ctx.reducer, ctx.shapes = reducer, (tuple(phoneme_enc.shape), tuple(pitch_table.shape))
        ctx.dtypes = (phoneme_enc.dtype, pitch_table.dtype)
        return ops.expand_encodings(phoneme_enc.detach().float().contiguous(), coarse,
                                    pitch_table.detach().float().contiguous(), idx)

    @staticmethod
    def backward(ctx, d_cond):
        coarse, idx = ctx.saved_tensors
        d_tok = d_cond.float().transpose(1, 2)          # (B, L, D): the denoiser hands over a token-major buffer
        if d_tok.stride(2) != 1:
            d_tok = d_tok.contiguous()
        dev = d_cond.device
        d_phon = torch.zeros(ctx.shapes[0], device=dev) if ctx.needs_input_grad[0] else None
        d_table = torch.zeros(ctx.shapes[1], device=dev) if ctx.needs_input_grad[1] else None
        ops.expand_encodings_bwd(d_tok, coarse, idx, d_phon, d_table)
        if ctx.reducer is not None and d_table is not None:
            ctx.reducer.reduce(d_table)
            ctx.reducer.finish()
        return (d_phon.to(ctx.dtypes[0]) if d_phon is not None else None,
                d_table.to(ctx.dtypes[1]) if d_table is not None else None, None, None, None)


def expand_encodings(phoneme_enc: torch.Tensor, duration: torch.Tensor, pitch: torch.Tensor,
                     pitch_table: torch.Tensor, length: Optional[int] = None, reducer=None) -> torch.Tensor:
    """cond (B, D, L) of ns2.py:1478-1483: phoneme encodings + coarse-pitch embeddings repeated `duration` frames.
    pitch: per-phoneme (B, T) f0.  L = `length` (frames past a sample's total duration are 0) or the max total duration.
    Differentiable with respect to phoneme_enc and pitch_table when autograd tracks them (`reducer`: GradReducer that
    receives the pitch table's gradient)."""
    idx = frames_to_text_index(duration, length)
    coarse = f0_to_coarse(pitch.float()).contiguous()
    if torch.is_grad_enabled() and (phoneme_enc.requires_grad or pitch_table.requires_grad):
        return _ExpandFunction.apply(phoneme_enc, pitch_table, coarse, idx, reducer)
    return ops.expand_encodings(phoneme_enc.float().contiguous(), coarse, pitch_table.detach().float().contiguous(), idx)


class Conditioner(nn.Module):
    """The per-sample conditional front end of NaturalSpeech2 (ns2.py:1472-1483 sampling, 1537-1583 training) as the
    `conditioner` callable of `naturalspeech2_pytorch_b200.NaturalSpeech2`: prompt latents + phoneme ids -> (prompt_enc,
    cond).  Sub-module names follow the reference's NaturalSpeech2 attributes (ns2.py:1231-1236), so the matching slices
    of a reference checkpoint load with `load_state_dict(..., strict=False)`.

    mode="train" takes the durations from the caller: `duration` (B, T) frame counts per phoneme (the reference
    aligner's `aln_hard`, from an external aligner or the reference's Aligner) and frame-level `pitch` (B, L) /
    (B, 1, L).  The aligner network and its losses are not run; the duration / pitch predictor only with
    train_duration_pitch (below): in the reference they only feed `aux_loss`, which is never returned (ns2.py:1600-1602),
    so by default the diffusion loss is the only gradient path into the prompt encoder, the phoneme encoder and
    `pitch_emb`.  `grad_reducer` (parallel.GradReducer) all-reduces
    their gradients in data-parallel training.

    train_dropout=True makes training draw the reference's dropout in both encoders (their `train_dropout`; see the
    module docstring).  The default False keeps them deterministic, as before the option existed.
    duration_pitch_dropout=True does the same for the duration / pitch predictor (its cross attentions' dropout, the
    only dropout of the reference's predictor with p > 0); train_dropout leaves the predictor deterministic.

    train_duration_pitch=True also trains the duration / pitch predictor: mode="train" runs it on the same encoder
    outputs and returns (prompt_enc, cond, duration_loss, pitch_loss), the reference's L1 losses against the given
    durations and the per-phoneme pitch (ns2.py:1579-1590).  Their gradients reach the predictor and, through its
    inputs, both encoders; NaturalSpeech2.forward weights and adds them (duration_loss_weight, pitch_loss_weight).

    mode="train" with prompt_lens / phoneme_lens (a batch padded at its ends): sample b is prompt[b, :prompt_lens[b]]
    and text[b, :phoneme_lens[b]] with its durations, which must be 0 past phoneme_lens[b].  Each sample's prompt_enc
    and cond are those of the sample alone (zero past its prompt length and its total duration), and the gradients
    reaching the encoders are the sums of the per-sample-alone ones (see the module docstring).  Not together with
    train_dropout or train_duration_pitch."""

    train_duration_pitch = False

    def __init__(self, *, dim_codebook=128, num_phoneme_tokens=None, tokenizer=None, duration_pitch_dim=512,
                 pitch_emb_dim=256, pitch_emb_pp_hidden_dim=512, train_dropout=False, train_duration_pitch=False,
                 duration_pitch_dropout=False):
        super().__init__()
        self.phoneme_enc = PhonemeEncoder(tokenizer=tokenizer, num_tokens=num_phoneme_tokens)
        self.prompt_enc = SpeechPromptEncoder(dim_codebook=dim_codebook)
        self.phoneme_enc.train_dropout = self.prompt_enc.train_dropout = bool(train_dropout)
        self.duration_pitch = DurationPitchPredictor(dim=duration_pitch_dim)
        self.duration_pitch.train_dropout = bool(duration_pitch_dropout)
        self.pitch_emb = nn.Embedding(pitch_emb_dim, pitch_emb_pp_hidden_dim)
        self.train_duration_pitch = bool(train_duration_pitch)
        self.grad_reducer = None

    @property
    def grad_reducer(self):
        return self._grad_reducer

    @grad_reducer.setter
    def grad_reducer(self, reducer):
        self._grad_reducer = reducer
        for name in ("prompt_enc", "phoneme_enc", "duration_pitch"):
            if name in self._modules:   # a Conditioner may be assembled around some of them
                self._modules[name].grad_reducer = reducer

    def forward(self, prompt=None, text=None, text_lens=None, mode="sample", pitch=None, duration=None, *,
                prompt_lens=None, phoneme_lens=None, **unused):
        """`text_lens` is accepted and ignored, as in the reference (ns2.py:1462).  mode="sample" with `prompt_lens` /
        `phoneme_lens` (per-sample lengths of a batch padded at the end) returns (prompt_enc, cond, cond_lens): each
        sample's outputs are those of running it alone, zero past its lengths; cond_lens (B,) int32 is each sample's
        total predicted duration in frames (cond is zero past it)."""
        ragged = prompt_lens is not None or phoneme_lens is not None
        if mode == "train":
            return self._forward_train(prompt, text, pitch, duration, prompt_lens, phoneme_lens)
        if mode != "sample":
            raise NotImplementedError(f"Conditioner: unknown mode {mode!r} (sample | train)")
        assert prompt is not None and text is not None
        with torch.no_grad():
            if not ragged:
                prompt_enc = self.prompt_enc(prompt)
                phoneme_enc = self.phoneme_enc(text)
                duration, pitch = self.duration_pitch(phoneme_enc, prompt_enc)
                cond = expand_encodings(phoneme_enc, duration, pitch, self.pitch_emb.weight)
                return prompt_enc, cond
            prompt_enc = self.prompt_enc(prompt, lengths=prompt_lens)
            phoneme_enc = self.phoneme_enc(text, lengths=phoneme_lens)
            duration, pitch = self.duration_pitch(phoneme_enc, prompt_enc, lengths=phoneme_lens, prompt_lens=prompt_lens)
            cond = expand_encodings(phoneme_enc, duration, pitch, self.pitch_emb.weight)
            cond_lens = duration.int().sum(dim=-1, dtype=torch.int32)   # the frames frames_to_text_index fills
        return prompt_enc, cond, cond_lens

    def _forward_train(self, prompt, text, pitch, duration, prompt_lens=None, phoneme_lens=None):
        """ns2.py:1538-1583 with the aligner's hard durations given: prompt_enc = prompt_enc(prompt), cond =
        expand_encodings(phoneme_enc(text), durations, average_over_durations(pitch, durations)) with L = pitch frames.
        prompt_lens / phoneme_lens: per-sample lengths, see the class docstring."""
        if duration is None:
            raise NotImplementedError(
                "Conditioner(mode='train') needs duration=(B, T) frame counts per phoneme (the aligner's aln_hard): the "
                "aligner network is not built, durations come from the caller")
        if prompt is None or text is None or pitch is None:
            raise ValueError("Conditioner(mode='train') needs prompt=, text= and frame-level pitch= (B, L) or (B, 1, L)")
        if isinstance(text, (list, tuple)):
            raise ValueError("Conditioner(mode='train') takes phoneme ids (B, T), not strings")
        if pitch.dim() == 2:
            pitch = pitch.unsqueeze(1)
        if pitch.dim() != 3 or pitch.shape[1] != 1:
            raise ValueError(f"pitch must be (B, L) or (B, 1, L), got {tuple(pitch.shape)}")
        B, T = text.shape
        L = pitch.shape[-1]
        if tuple(duration.shape) != (B, T) or pitch.shape[0] != B:
            raise ValueError(f"duration must be (B, T) = {(B, T)} and pitch (B, 1, L); got {tuple(duration.shape)}, "
                             f"{tuple(pitch.shape)}")
        if duration.is_floating_point() and not bool((duration == duration.round()).all()):
            raise ValueError("duration must hold whole frame counts")
        if bool((duration < 0).any()):
            raise ValueError("duration must be non-negative")
        total = duration.long().sum(dim=-1)
        if bool((total > L).any()):
            raise ValueError(f"durations sum to {int(total.max())} frames, past the {L} frames of pitch")
        if phoneme_lens is not None:   # host-side checks: nothing is launched for a refused call
            lens = ops.lengths(phoneme_lens, B, T, device=duration.device, name="phoneme_lens")
            past = torch.arange(T, device=duration.device)[None, :] >= lens[:, None].long()
            if bool(((duration != 0) & past).any()):
                raise ValueError("duration must be 0 past phoneme_lens (padded phonemes take no frames)")
        if prompt_lens is not None or phoneme_lens is not None:
            if self.train_duration_pitch:
                raise NotImplementedError("Conditioner(train_duration_pitch=True) does not take prompt_lens / "
                                          "phoneme_lens: the duration / pitch predictor trains without lengths")
            if self.training and (self.prompt_enc.train_dropout or self.phoneme_enc.train_dropout):
                raise NotImplementedError("Conditioner(train_dropout=True) does not take prompt_lens / phoneme_lens: "
                                          "the attention has no key-padded dropout")
        prompt_enc = self.prompt_enc(prompt, lengths=prompt_lens)
        phoneme_enc = self.phoneme_enc(text, lengths=phoneme_lens)
        with torch.no_grad():
            ph_pitch = average_over_durations(pitch.float(), duration)[:, 0]      # (B, T), ns2.py:1581
        cond = expand_encodings(phoneme_enc, duration, ph_pitch, self.pitch_emb.weight, length=L,
                                reducer=self._grad_reducer)
        if not self.train_duration_pitch:
            return prompt_enc, cond
        duration_pred, pitch_pred = self.duration_pitch(phoneme_enc, prompt_enc)
        duration_loss = F.l1_loss(duration.float(), duration_pred)                # ns2.py:1587
        pitch_loss = F.l1_loss(ph_pitch, pitch_pred)                              # ns2.py:1589-1590
        return prompt_enc, cond, duration_loss, pitch_loss
