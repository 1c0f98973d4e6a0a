"""Training step of the denoiser: hand-written backward of `Model._forward_impl` (SURVEY rows a18 / f1).

`loss.backward()` is how the reference is used (README.md:60-63, ns2.py:1886).  Here `Model.forward` records ONE autograd
node (`DenoiserFunction`) when gradients are enabled.  Its forward is the inference forward, `Model._forward_impl`, given
a `saved` dict: the same kernels in the same order (bit-identical output) with the activations the backward needs kept in
fresh tensors.  Its backward walks the network in reverse and launches, per layer,
  * dgrad GEMMs     ns2_gemm on transposed weight packs (anti-causal shifts for the causal convs),
  * wgrad GEMMs     ns2_wgrad (wgmma, MN-major operands, fp32 reduce-add into the packed gradient),
  * attention bwd   ns2_attn_bwd (wgmma flash backward from the saved log-sum-exp),
  * the element-wise backward kernels of csrc/backward.cu (RMSNorm+FiLM, GEGLU, Wavenet gate, bias column sums).
Pre-activations that the fused forward epilogues never materialise (GEGLU's value/gate pair, the Wavenet conv output
before FiLM) and the feed-forward's conv output, which the forward folds into the output projection and never
computes, are recomputed with plain-epilogue GEMMs instead of being stored.  Gradients come out in the packed bf16
layouts' fp32 twins, under the state_dict's keys; `param_grads` gives them the parameters' shapes.
Each building block has one implementation, shared by the denoiser, the perceiver and the encoders (encoders.py):
`linear_backward`, `conv_backward`, `ff_backward` (with `geglu_backward`) and `attention_backward`.

Scope: unconditional and conditional denoisers (BASELINE configs[1], configs[2]/[4]): perceiver resampler, cross
attention, prompt FiLM vector, aligned-condition projection and the classifier-free-guidance null parameters included.
The (B,)-sized conditioning vectors — timestep embedding (LearnedSinusoidalPosEmb + Linear + SiLU, ns2.py:108-120,
839-843) and prompt vector (mean-pool + Linear + SiLU, ns2.py:858-862) — are differentiated with torch autograd on a
recomputation: 32 x 2048 values each, host-side glue like the noise schedules.  `prompt_mask` is unsupported (as in
the inference path).
When autograd asks for them (an encoder upstream: encoders.Conditioner in train mode) the backward also returns
d loss / d prompt (perceiver context projection dgrad + the mean-pool's share, spread by ops.add_rows_bcast) and
d loss / d cond (one dgrad GEMM through the aligned-condition projection, token-major, handed over as a channel-first
view); otherwise nothing extra runs.  `x` and `times` stay non-differentiable (latents come from the codec).
With per-sample prompt lengths (`Model.forward(prompt_lens=)`) the perceiver's attention backward takes the forward's
key counts M + prompt_lens (ops.attention_bwd kv_lens) and the mean-pool's share of d prompt is d mean[b] / prompt_lens[b]
over the rows [0, prompt_lens[b]): d prompt rows past a sample's length are exact zeros.  The latent sequence needs no
lengths: the WaveNet and feed-forward convs are causal and the batch shares one latent length.
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch
import torch.nn.functional as F

from . import ops

bf = torch.bfloat16


def _wgrad(dy: torch.Tensor, x: torch.Tensor) -> torch.Tensor:
    """dW = dy^T x (fp32, (dy cols, x cols)) of a projection y = x W^T."""
    n, k = dy.shape[-1], x.shape[-1]
    return ops.wgrad(dy, x, torch.zeros(n, k, device=dy.device), n=n, k=k)


def _colsum(dy: torch.Tensor) -> torch.Tensor:
    """Bias gradient: dy summed over every row (fp32)."""
    return ops.colsum(dy, torch.zeros(dy.shape[-1], device=dy.device))


def _dgrad(dy: torch.Tensor, w_t: torch.Tensor, dtype=bf, out=None, **gemm_args) -> torch.Tensor:
    """d x = dy W on the transposed pack w_t (x cols, dy cols), into `out` or a fresh tensor of `dtype`."""
    if out is None:
        out = torch.empty(*dy.shape[:2], w_t.shape[0], device=dy.device, dtype=dtype)
    return ops.gemm(dy, w_t, out, n=w_t.shape[0], epilogue=ops.EPI_F32 if out.dtype == torch.float32 else ops.EPI_BF16,
                    **gemm_args)


def linear_backward(dy, x, grads: Dict[str, torch.Tensor], name: str, w_t=None, bias: bool = True,
                    width: Optional[int] = None, dtype=bf) -> Optional[torch.Tensor]:
    """Backward of y = x W^T (+ b): grads[name + ".weight"] (its first `width` input columns when the pack is
    zero-padded beyond the layer's width) and grads[name + ".bias"]; returns d x (of `dtype`) when the transposed pack
    w_t is given."""
    dw = _wgrad(dy, x)
    grads[name + ".weight"] = dw if width is None else dw[:, :width]
    if bias:
        grads[name + ".bias"] = _colsum(dy)
    return None if w_t is None else _dgrad(dy, w_t, dtype)


def conv_wgrad(dy, x, dw, n: int, c_in: int, kernel: int, first_shift: int, **wgrad_args) -> torch.Tensor:
    """dw[:, t*c_in:(t+1)*c_in] += the weight gradient of tap t of an `ops.conv_segs` convolution (tap t reads
    x[n - (first_shift - t) * dilation]); returns those columns as the reference's (O, I, k) view.  `wgrad_args`: the
    groups / strides / dilations of a grouped convolution."""
    for t in range(kernel):
        ops.wgrad(dy, x, dw[:, t * c_in:(t + 1) * c_in], n=n, k=c_in, shift_units=first_shift - t, **wgrad_args)
    return dw[:, :kernel * c_in].view(dw.shape[0], kernel, c_in).permute(0, 2, 1)


def conv_backward(dy, x, grads: Dict[str, torch.Tensor], name: str, w_t, kernel: int, first_shift: int,
                  width: Optional[int] = None, dtype=bf) -> Optional[torch.Tensor]:
    """Backward of y = conv(x) + b (stride 1, packed by `model._pack_conv`, tap t reads x[n - (first_shift - t)]):
    grads[name + ".weight" / ".bias"] in the reference's layout (the first `width` channels when the pack is zero-padded
    beyond the layer's width); returns d x (of `dtype`, mirrored shifts on the transposed pack) when w_t is given."""
    c_out, c_in = dy.shape[-1], x.shape[-1]
    dw = conv_wgrad(dy, x, torch.zeros(c_out, kernel * c_in, device=dy.device), c_out, c_in, kernel, first_shift)
    db = _colsum(dy)
    grads[name + ".weight"], grads[name + ".bias"] = (dw, db) if width is None else (dw[:width, :width], db[:width])
    if w_t is None:
        return None
    return _dgrad(dy, w_t, dtype, segs=ops.conv_dgrad_segs(c_out, kernel, first_shift))


def geglu_backward(h, d_g, w1, b1, w1_t, Di: int, grads: Dict[str, torch.Tensor], name: str) -> torch.Tensor:
    """Backward of g = GEGLU(h @ w1^T + b1), w1 / b1 packed by `model._pack_geglu` (inner width Di padded to Dp): the
    pre-activation is recomputed with a plain-epilogue GEMM, lin1's gradients go to grads[name + ".weight" / ".bias"] in
    the reference's layout (value rows, then gate rows), and d h (bf16) is returned."""
    B, N, D = h.shape
    Dp = w1.shape[0] // 2
    pre = ops.gemm(h, w1, torch.empty(B, N, 2 * Dp, device=h.device, dtype=bf), n=2 * Dp, epilogue=ops.EPI_BF16, bias=b1)
    ops.geglu_bwd(pre, d_g)                                                              # pre <- d pre
    dW1 = _wgrad(pre, h).view(Dp // 128, 2, 128, D)
    db1 = _colsum(pre).view(Dp // 128, 2, 128)
    grads[name + ".weight"] = torch.cat((dW1[:, 0].reshape(Dp, D)[:Di], dW1[:, 1].reshape(Dp, D)[:Di]), dim=0)
    grads[name + ".bias"] = torch.cat((db1[:, 0].reshape(Dp)[:Di], db1[:, 1].reshape(Dp)[:Di]), dim=0)
    return _dgrad(pre, w1_t)


def ff_backward(dy, h, g, P, T, pk: str, Di: int, grads: Dict[str, torch.Tensor], name: str,
                causal_conv: bool = False) -> torch.Tensor:
    """Backward of FeedForward (ns2.py:1009-1025) y = W2 [causal conv](GEGLU(W1 h + b1)) + b2 from the saved GEGLU output
    g.  Weights are P / T[pk + "w1" / "b1" / "wc" / "bc" / "w2" / "wo"], the inner width Di padded in the packs;
    gradients go to grads[name + Sequential index + ...].  Returns d h (bf16).
    With the causal k=3 conv the forward ran conv and W2 as one folded conv (pack "wo", `model._fold_conv_linear`) and
    kept no conv output: c = conv(g) + bc is recomputed for W2's gradient alone, d c = dy W2 gives the conv's
    gradients, and d g is the folded conv's dgrad straight from dy (K = 3 D instead of 3 Dp)."""
    if not causal_conv:
        d_g = linear_backward(dy, g, grads, name + "2", T[pk + "w2"], width=Di)
    else:
        Dp = g.shape[-1]
        c = ops.gemm(g, P[pk + "wc"], torch.empty_like(g), n=Dp, epilogue=ops.EPI_BF16, bias=P[pk + "bc"],
                     segs=ops.conv3_segs(Dp))
        d_c = linear_backward(dy, c, grads, name + "3", T[pk + "w2"], width=Di)
        conv_backward(d_c, g, grads, name + "2.1", None, 3, 2, width=Di)
        d_g = _dgrad(dy, T[pk + "wo"], segs=ops.conv_dgrad_segs(dy.shape[-1], 3, 2))
    return geglu_backward(h, d_g, P[pk + "w1"], P[pk + "b1"], T[pk + "w1"], Di, grads, name + "0")


def attention_backward(dy, x, o, lse, q, kv, w_o_t, w_q_t, heads: int, grads: Dict[str, torch.Tensor], name: str,
                       d_kv=None, x_kv=None, w_kv_t=None, dropout=None, kv_lens=None):
    """Backward of y = Wo attn(Wq x, Wkv x_kv) (Attention, ns2.py:1029-1053, bias-free) from the forward's attention
    output o and log-sum-exp.  to_out / to_q / to_kv gradients go to grads[name + ...]; returns (d x, d x_kv), bf16.
      * self-attention: kv is None and q is the fused (B, N, 3*inner) qkv of one GEMM on x (transposed pack w_q_t),
        so one wgrad and one dgrad cover q, k and v;
      * cross-attention: d kv goes to `d_kv` (a fresh buffer when None).  Given the context x_kv and its transposed pack
        w_kv_t, to_kv's gradient and d x_kv are computed too; otherwise d x_kv is None and to_kv is the caller's.
    `dropout`: the forward's attention dropout (seed, site, p), or None (see ops.attention).  `kv_lens`: the forward's
    per-sample key counts, or None (see ops.attention_bwd): d kv rows past them come out as exact zeros."""
    B, N = dy.shape[:2]
    inner = heads * 64
    dev = dy.device
    grads[name + "to_out.weight"] = _wgrad(dy, o)
    d_o = _dgrad(dy, w_o_t)
    fused = kv is None
    if fused:
        d_q = torch.empty(B, N, 3 * inner, device=dev, dtype=bf)
        q, kv, d_kv = q[:, :, :inner], q[:, :, inner:], d_q[:, :, inner:]
    elif d_kv is None:
        d_kv = torch.empty(B, kv.shape[1], 2 * inner, device=dev, dtype=bf)
    dq = torch.zeros(B, N, inner, device=dev)
    ops.attention_bwd(q, kv[:, :, :inner], kv[:, :, inner:], o, d_o, lse, dq, d_kv[:, :, :inner], d_kv[:, :, inner:],
                      heads=heads, dropout=dropout, kv_lens=kv_lens)
    if fused:
        d_q[:, :, :inner].copy_(dq)   # fp32 accumulator -> bf16 slot (layout glue)
        dw = _wgrad(d_q, x)
        grads[name + "to_q.weight"], grads[name + "to_kv.weight"] = dw[:inner], dw[inner:]
    else:
        d_q = ops.cast_bf16(dq, torch.empty(B, N, inner, device=dev, dtype=bf))
        grads[name + "to_q.weight"] = _wgrad(d_q, x)
    d_x_kv = None if x_kv is None else linear_backward(d_kv, x_kv, grads, name + "to_kv", w_kv_t, bias=False)
    return _dgrad(d_q, w_q_t), d_x_kv


def train_backward(model, S: dict, d_out: torch.Tensor, reducer=None, input_grads=None) -> Dict[str, torch.Tensor]:
    """Gradients of every parameter (keys of `model.named_parameters()`), given d(loss)/d(prediction).
    `reducer` (parallel.GradReducer): finished gradient buffers are handed over layer by layer, so that their
    all-reduce overlaps the rest of the backward pass.
    `input_grads`: a dict whose keys "prompt" / "cond" (present = wanted) receive d(loss)/d(prompt) (B, Np, dim_prompt)
    and d(loss)/d(cond) (B, dim_prompt, Lc) — per-sample gradients, kept out of the reducer."""
    want_prompt = input_grads is not None and "prompt" in input_grads
    want_cond = input_grads is not None and "cond" in input_grads
    flush = (lambda: reducer.reduce_all(grads)) if reducer is not None else (lambda: None)
    B, N = S["B"], S["N"]
    D, G, inner, H = model.dim, model.wavenet_layers, model.inner, model.heads
    Di = model.ff_inner
    dev = d_out.device
    P = model.packed()
    T = model.packed_transposed()
    film = S["film"]
    e = lambda *s, dt=bf: torch.empty(*s, device=dev, dtype=dt)
    z = lambda *s: torch.zeros(*s, device=dev, dtype=torch.float32)
    grads: Dict[str, torch.Tensor] = {}
    dfilm = z(B, film.shape[1])
    t_cond = S["t"].contiguous()
    dil = [2 ** i for i in range(G)]

    # ---- to_pred: Linear (no bias) after RMSNorm(gamma) ----
    lens = S.get("lens")
    if lens is not None:   # the forward zeroed the prediction past each latent length: no gradient flows from there
        d_out = ops.mask_rows(d_out.float().clone(memory_format=torch.contiguous_format), lens)
    dout_bf = ops.cast_bf16(d_out.float().contiguous(), e(B, N, D))
    dhf = linear_backward(dout_bf, S["hf"], grads, "transformer.to_pred.1", T["pred_w"], bias=False)
    dxr = z(B, N, D)                       # fp32 gradient of the residual stream
    dxr_bf = e(B, N, D)
    dgam = z(D)
    ops.rmsnorm_film_bwd(S["x_final"], dhf, dxr, dxr_bf, rows_per_batch=N, gamma=P["pred_gamma"], dgamma=dgam)
    grads["transformer.to_pred.0.gamma"] = dgam

    npl = model._norms_per_layer
    conditional = model.condition_on_prompt
    if conditional:
        M = model.num_latents_m
        d_xkv = e(B, M, model.depth * 2 * inner)

    def norm_backward(x_in, dh, fo):   # RMSNorm + FiLM whose (gamma, beta) are film[:, fo:fo + 2D]
        ops.rmsnorm_film_bwd(x_in, dh, dxr, dxr_bf, rows_per_batch=N, film=film[:, fo:fo + 2 * D],
                             dfilm=dfilm[:, fo:fo + 2 * D])

    for l in reversed(range(model.depth)):
        L = S["layers"][l]
        pfx = f"transformer.layers.{l}."
        fo = model._film_tr_off + l * npl * 2 * D
        # ---- feed-forward branch: x += W2 conv(GEGLU(W1 h2)) ----
        dh2 = ff_backward(dxr_bf, L["h2"], L["ff_g"], P, T, f"l{l}_ff_", Di, grads, pfx + "5.", causal_conv=True)
        norm_backward(L["x_mid"], dh2, fo + (npl - 1) * 2 * D)
        # ---- cross-attention branch: x += Wxo attn(Wxq h_x, Wxkv c); Wxkv's gradient is taken for all layers at once ----
        if conditional:
            kv = slice(l * 2 * inner, (l + 1) * 2 * inner)
            dh_x, _ = attention_backward(dxr_bf, L["h_x"], L["ao2"], L["lse2"], L["xq"], S["xkv"][:, :, kv], T[f"l{l}_xo"],
                                         T[f"l{l}_xq"], H, grads, pfx + "3.", d_kv=d_xkv[:, :, kv])
            norm_backward(L["x_c"], dh_x, fo + 2 * D)
        # ---- attention branch: x += Wo attn(Wqkv h1) ----
        dh1, _ = attention_backward(dxr_bf, L["h1"], L["ao"], L["lse"], L["qkv"], None, T[f"l{l}_o"], T[f"l{l}_qkv"], H,
                                    grads, pfx + "1.", kv_lens=lens)
        norm_backward(L["x_in"], dh1, fo)
        # FiLM projections of this layer's norms: their rows of dfilm are final now, so the weight gradient (the largest
        # gradient buffers of the model) joins this layer's all-reduce instead of trailing the whole backward
        dWl = ops.film_wgrad(dfilm[:, fo:fo + npl * 2 * D], t_cond, torch.empty(npl * 2 * D, model.dim_cond, device=dev),
                             accumulate=False)
        for k, idx in enumerate((0, 2, 4) if conditional else (0, 4)):
            grads[pfx + f"{idx}.to_gamma_beta.weight"] = dWl[k * 2 * D:(k + 1) * 2 * D]
        flush()   # this layer's gradients are final: their all-reduce overlaps the layers still to come

    if conditional:
        # d prompt, term (a): through the perceiver's context projection (identity when dim_prompt == dim)
        d_prompt = _conditioning_backward_tokens(model, S, T, d_xkv, grads, want_prompt)
        if want_prompt:
            input_grads["prompt"] = d_prompt
    # ---- wavenet: final 1x1 conv, skip sum, 4 stacks of 8 dilation columns, init conv ----
    # (1x1 conv gradients keep the GEMM's 2-D shape; `param_grads` gives them the parameters' shapes)
    d_skip = linear_backward(dxr_bf, S["skip"], grads, "wavenet.final_conv", T["wn_final_w"])
    # the skip convs are one GEMM over the concatenated stack outputs with the summed bias: split its gradient
    dWskip, dbskip = _wgrad(d_skip, S["stack_out"][-1]), _colsum(d_skip)
    nst = model.wavenet_stacks
    for g in range(G):
        grads[f"wavenet.stacks.{nst - 1}.blocks.{g}.skip_conv.weight"] = dWskip[:, g * D:(g + 1) * D]
        grads[f"wavenet.stacks.{nst - 1}.blocks.{g}.skip_conv.bias"] = dbskip
    # dcy: [dc | dy] halves, so that one grouped dgrad GEMM reads the conv taps from dc and the 1x1 res conv from dy
    dcy = e(B, N, 2 * G * D)
    _dgrad(d_skip, T["wn_skip_w"], out=dcy[:, :, G * D:])     # d y of the last stack
    c_pre = e(B, N, G * D)
    for s in reversed(range(nst)):
        x_in = S["stack_out"][s - 1] if s > 0 else S["h0"]
        gcs = D if s > 0 else 0
        fo_s = s * G * 2 * D
        # recompute the conv output (incl. bias) that FiLM + the gate consumed
        ops.gemm(x_in, P[f"wn{s}_w"], c_pre, n=D, epilogue=ops.EPI_BF16, bias=P[f"wn{s}_b"], segs=ops.conv3_segs(D),
                 groups=G, a_group_col_stride=gcs, b_group_row_stride=D, out_group_col_stride=D, dil=dil)
        dy = dcy[:, :, G * D:]
        dc = dcy[:, :, :G * D]
        ops.wavenet_gate_bwd(c_pre, dy, dc, film[:, fo_s:], dfilm[:, fo_s:], dim=D, groups=G, film_group_stride=2 * D)
        dWs = ops.film_wgrad(dfilm[:, fo_s:fo_s + G * 2 * D], t_cond, torch.empty(G * 2 * D, model.dim_cond, device=dev),
                             accumulate=False)   # this stack's FiLM projections (see the transformer loop)
        for g in range(G):
            grads[f"wavenet.stacks.{s}.blocks.{g}.to_time_cond.weight"] = dWs[g * 2 * D:(g + 1) * 2 * D]
        # [conv taps | res conv] of the G blocks in one (G*D, 4*D) buffer, like the forward pack
        grouped = dict(groups=G, dy_group_col_stride=D, x_group_col_stride=gcs, dw_group_row_stride=D)
        dWp = z(G * D, 4 * D)
        dWc = conv_wgrad(dc, x_in, dWp, D, D, 3, 2, dil=dil, **grouped)
        ops.wgrad(dy, x_in, dWp[:, 3 * D:], n=D, k=D, **grouped)
        dbc, dbr = _colsum(dc), _colsum(dy)
        for g in range(G):
            blk = f"wavenet.stacks.{s}.blocks.{g}."
            grads[blk + "conv.weight"] = dWc[g * D:(g + 1) * D]
            grads[blk + "res_conv.weight"] = dWp[g * D:(g + 1) * D, 3 * D:]
            grads[blk + "conv.bias"] = dbc[g * D:(g + 1) * D]
            grads[blk + "res_conv.bias"] = dbr[g * D:(g + 1) * D]
        # d(input of every column): anti-causal taps on dc + the transposed 1x1 on dy
        segs = ops.conv_dgrad_segs(D, 3, 2) + [(G * D, 3 * D, D, 0, 0)]
        d_in = e(B, N, G * D)
        ops.gemm(dcy, T[f"wn{s}_w"], d_in, n=D, epilogue=ops.EPI_BF16, segs=segs, groups=G, a_group_col_stride=D,
                 b_group_row_stride=D, out_group_col_stride=D, dil=dil)
        flush()
        if s > 0:
            dcy[:, :, G * D:].copy_(d_in)       # becomes d y of the previous stack
        else:
            d_h0 = ops.group_sum(d_in, e(B, N, D), dim=D, groups=G)   # h0 feeds all columns
    # x_in = x + pad_or_curtail(where(cdrop, null_cond, cond_proj)) (ns2.py:978-992): d x_in from the init conv's dgrad
    d_xin = conv_backward(d_h0, S["x_bf"], grads, "wavenet.init_conv", T["wn_init_w"] if conditional else None, 3, 2)
    if conditional:
        Lc = S["Lc"]
        n_used = min(Lc, N)
        keep = (~S["cdrop"])[:, None, None]
        d_cp = torch.zeros(B, Lc, D, device=dev, dtype=bf)
        d_cp[:, :n_used] = torch.where(keep, d_xin[:, :n_used], torch.zeros((), device=dev, dtype=bf))   # masking glue
        grads["null_cond"] = (d_xin[:, :n_used].float() * S["cdrop"][:, None, None]).sum((0, 1)).unsqueeze(-1)
        # d cond = d_cp @ W (1x1 conv dgrad), token-major; curtailed frames (n >= N) stay exact zeros.  Returned as the
        # channel-first view cond has, so nothing is transposed.
        d_cond = linear_backward(d_cp, S["cond_bf"], grads, "cond_to_model_dim", T["cond_w"] if want_cond else None,
                                 dtype=torch.float32)
        if want_cond:
            input_grads["cond"] = d_cond.permute(0, 2, 1)

    # ---- FiLM projections (one stacked matrix) and the timestep embedding ----
    rows = film.shape[1]
    dbf = dfilm.sum(0)
    dfilm_bf = ops.cast_bf16(dfilm, e(1, B, rows))
    dt = _dgrad(dfilm_bf, T["film_w"], torch.float32)[0]
    if conditional:
        # prompt FiLM vector: where(drop, null_prompt_cond, silu(Linear(mean(prompt)))) (ns2.py:952-962); (B,)-sized glue
        d_pc = dt[:, model.dim_time:]
        grads["null_prompt_cond"] = (d_pc * S["drop"][:, None]).sum(0)
        lin = model.to_prompt_cond[1]
        with torch.enable_grad():
            lw = lin.weight.detach().float().requires_grad_(True)
            lb = lin.bias.detach().float().requires_grad_(True)
            mean = S["prompt_mean"].detach().requires_grad_(want_prompt)
            F.silu(F.linear(mean, lw, lb)).backward(d_pc * (~S["drop"])[:, None])
        grads["to_prompt_cond.1.weight"], grads["to_prompt_cond.1.bias"] = lw.grad, lb.grad
        if want_prompt:   # d prompt, term (b): the mean-pool spreads d mean evenly over the prompt rows
            plens = S["prompt_lens"]
            if plens is None:
                ops.add_rows_bcast(input_grads["prompt"], mean.grad.contiguous(), 1.0 / S["pr_Np"])
            else:         # ... over each sample's own rows: d mean[b] / prompt_lens[b] on [0, prompt_lens[b]), zero past
                ops.add_rows_bcast(input_grads["prompt"], (mean.grad * (1.0 / plens.double()).float()[:, None]).contiguous())
                ops.mask_rows(input_grads["prompt"], plens)
        dt = dt[:, :model.dim_time]
    off = 0
    for s in range(nst):
        for g in range(G):
            key = f"wavenet.stacks.{s}.blocks.{g}.to_time_cond."
            grads[key + "bias"] = dbf[off:off + 2 * D]
            off += 2 * D
    for l in range(model.depth):
        for idx in ((0, 2, 4) if conditional else (0, 4)):
            key = f"transformer.layers.{l}.{idx}.to_gamma_beta."
            grads[key + "bias"] = dbf[off:off + 2 * D]
            off += 2 * D
    # (B,)-sized timestep embedding: torch autograd on a recomputation (ns2.py:108-120, 839-843)
    tc = model.to_time_cond
    with torch.enable_grad():
        wts = tc[0].weights.detach().float().requires_grad_(True)
        lw = tc[1].weight.detach().float().requires_grad_(True)
        lb = tc[1].bias.detach().float().requires_grad_(True)
        tt = S["times"][:, None]
        freqs = tt * wts[None] * 2 * math.pi
        emb = torch.cat((tt, freqs.sin(), freqs.cos()), dim=-1)
        F.silu(F.linear(emb, lw, lb)).backward(dt.contiguous())
    grads["to_time_cond.0.weights"], grads["to_time_cond.1.weight"], grads["to_time_cond.1.bias"] = wts.grad, lw.grad, lb.grad
    if reducer is not None:
        flush()
        reducer.finish()
    return grads


def _conditioning_backward_tokens(model, S, T, d_xkv, grads, want_prompt: bool):
    """Backward of everything that produced the cross-attention context: the stacked K/V projection of all layers,
    the null-token substitution and the PerceiverResampler (ns2.py:532-579, 964-968).  Returns d prompt (fp32) when
    `want_prompt`, without its mean-pool term."""
    P = model.packed()
    B, D, M, inner, H = S["B"], model.dim, model.num_latents_m, model.inner, model.heads
    dev = d_xkv.device
    e = lambda *s, dt=bf: torch.empty(*s, device=dev, dtype=dt)
    z = lambda *s: torch.zeros(*s, device=dev, dtype=torch.float32)
    # one GEMM holds the cross-attention K/V projections of every layer: split its weight gradient
    dWkv = _wgrad(d_xkv, S["c_bf"])
    for l in range(model.depth):
        grads[f"transformer.layers.{l}.3.to_kv.weight"] = dWkv[l * 2 * inner:(l + 1) * 2 * inner]
    d_c = _dgrad(d_xkv, T["x_kv_all"]).float()
    drop = S["drop"]
    grads["null_prompt_tokens"] = (d_c * drop[:, None, None]).sum(0)
    d_tok = ops.cast_bf16((d_c * (~drop)[:, None, None]).contiguous(), e(B, M, D))
    # ---- perceiver: final RMSNorm(gamma), then the layers in reverse ----
    pr = model.perceiver_resampler
    dlat, dlat_bf = z(B, M, D), e(B, M, D)
    dgam = z(D)
    ops.rmsnorm_film_bwd(S["pr_lat"], d_tok, dlat, dlat_bf, rows_per_batch=M, gamma=pr.norm.gamma.detach().float().contiguous(),
                         dgamma=dgam)
    grads["perceiver_resampler.norm.gamma"] = dgam
    Np = S["pr_Np"]
    kv_lens = None if S["prompt_lens"] is None else S["prompt_lens"] + M   # keys [latents ; prompt[:prompt_lens]]
    d_proj = z(B, Np, D)
    for i in reversed(range(len(pr.layers))):
        L = S["pr_layers"][i]
        pfx = f"perceiver_resampler.layers.{i}."
        # feed-forward (no conv, no pre-norm): lat += W2 GEGLU(W1 lat)
        ops.accum_bf16(dlat, ff_backward(dlat_bf, L["lat_bf2"], L["g"], P, T, f"pr{i}_ff_", pr.ff_inner, grads,
                                         pfx + "1."), dlat_bf)
        # attention over cat(latents, projected prompt): lat += Wo attn(Wq lat, Wkv cat)
        d_lat, d_cat = attention_backward(dlat_bf, L["lat_bf"], L["o"], L["lse"], L["q"], L["kv"], T[f"pr{i}_o"],
                                          T[f"pr{i}_q"], H, grads, pfx + "0.", x_kv=L["cat"], w_kv_t=T[f"pr{i}_kv"],
                                          kv_lens=kv_lens)
        ops.accum_bf16(dlat, d_lat)
        ops.accum_bf16(dlat, d_cat[:, :M].contiguous(), dlat_bf)
        ops.accum_bf16(d_proj, d_cat[:, M:].contiguous())
    grads["perceiver_resampler.latents"] = dlat.sum(0)
    if "pr_proj_w" not in P:
        return d_proj
    return linear_backward(ops.cast_bf16(d_proj, e(B, Np, D)), S["pr_p_bf"], grads, "perceiver_resampler.proj_context",
                           T["pr_proj_w"] if want_prompt else None, dtype=torch.float32)


def param_grads(module: torch.nn.Module, grads: Dict[str, torch.Tensor], reducer=None) -> list:
    """The gradients of `module.parameters()` from a hand-written backward's `grads` (keys of `named_parameters()`), in
    the parameters' shapes and dtypes; raises when one is missing.  A None entry (a part of the module the loss does
    not reach) stays None, as torch autograd leaves it.  `reducer` (parallel.GradReducer) all-reduces them first."""
    missing = [n for n, _ in module.named_parameters() if n not in grads]
    if missing:
        raise RuntimeError(f"{type(module).__name__} backward produced no gradient for {missing[:4]}...")
    if reducer is not None:
        reducer.reduce_all({n: g for n, g in grads.items() if g is not None})
        reducer.finish()
    return [None if grads[n] is None else grads[n].reshape(p.shape).to(p.dtype) for n, p in module.named_parameters()]


class DenoiserFunction(torch.autograd.Function):
    """One autograd node for the whole denoiser: forward saves activations, backward runs the kernels above."""

    @staticmethod
    def forward(ctx, model, x, times, prompt, cond, cond_drop_prob, prompt_lens, lengths, *params):
        saved = {}
        out = model._forward_impl(x, times, prompt, cond=cond, cond_drop_prob=cond_drop_prob, saved=saved,
                                  prompt_lens=prompt_lens, lengths=lengths)
        ctx.model, ctx.saved = model, saved
        ctx.in_dtypes = (prompt.dtype if prompt is not None else None, cond.dtype if cond is not None else None)
        return out

    @staticmethod
    def backward(ctx, d_out):
        # d prompt / d cond only when autograd asks for them (an encoder upstream): otherwise no extra kernel runs
        inputs = {k: None for k, i in (("prompt", 3), ("cond", 4)) if ctx.needs_input_grad[i]}
        with torch.no_grad():
            grads = train_backward(ctx.model, ctx.saved, d_out, getattr(ctx.model, "grad_reducer", None),
                                   input_grads=inputs or None)
        ctx.saved = None
        d_prompt, d_cond = inputs.get("prompt"), inputs.get("cond")
        if d_prompt is not None:
            d_prompt = d_prompt.to(ctx.in_dtypes[0])
        if d_cond is not None:
            d_cond = d_cond.to(ctx.in_dtypes[1])
        return (None, None, None, d_prompt, d_cond, None, None, None, *param_grads(ctx.model, grads))


class MseRowsFunction(torch.autograd.Function):
    """Per-sample mean squared error (ns2.py:1646-1647) with the hand-written forward / backward kernels.  `lens`
    (validated int32 CUDA (B,), optional): sample b is its first lens[b] rows; its mean and gradient are those of the
    sample alone, and the gradient past them is exact zeros."""

    @staticmethod
    def forward(ctx, pred, target, lens=None):
        pred, target = pred.contiguous(), target.contiguous()
        ctx.save_for_backward(pred, target)
        ctx.lens = lens
        return ops.mse_rows(pred, target, torch.empty(pred.shape[0], device=pred.device), lens=lens)

    @staticmethod
    def backward(ctx, d_rows):
        pred, target = ctx.saved_tensors
        per = pred.numel() // pred.shape[0]
        if ctx.lens is None:
            coef = (d_rows.float() * (2.0 / per)).contiguous()
        else:   # 2 / (lens[b] * row elements), rounded to fp32 as the alone call's 2.0 / per is
            coef = (d_rows.float() * (2.0 / (ctx.lens.double() * (per // pred.shape[1]))).float()).contiguous()
        return ops.mse_bwd(pred, target, coef, out_f32=torch.empty_like(pred), lens=ctx.lens), None, None
