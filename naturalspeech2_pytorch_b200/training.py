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
before FiLM) are recomputed with plain-epilogue GEMMs instead of being stored.  Gradients come out in the packed bf16
layouts' fp32 twins and are scattered back to the reference's parameter shapes (same keys as the state_dict).
`geglu_backward` and `attention_backward` are shared with the encoders' backward (encoders.py).

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
"""
from __future__ import annotations

import math
from typing import Dict

import torch
import torch.nn.functional as F

from . import ops
from .model import _round_up

bf = torch.bfloat16


def _transpose_conv(w: torch.Tensor, kernel: int) -> torch.Tensor:
    """(O, k*I) tap-major conv pack -> (I, k*O) [in][tap][out] pack for the dgrad GEMM."""
    O = w.shape[0]
    return w.view(O, kernel, -1).permute(2, 1, 0).reshape(-1, kernel * O).contiguous()


def pack_transposed(model) -> Dict[str, torch.Tensor]:
    """bf16 transposed twins of `Model.packed()` for the dgrad GEMMs (rebuilt whenever the forward packs are)."""
    P = model.packed()
    D, G = model.dim, model.wavenet_layers
    T: Dict[str, torch.Tensor] = {}
    t = lambda w: w.t().contiguous()
    T["film_w"] = t(P["film_w"])                                        # (dim_cond, rows)
    for s in range(model.wavenet_stacks):
        w = P[f"wn{s}_w"].view(G, D, 4, D)                              # [group][out][tap0,tap1,tap2,res][in]
        T[f"wn{s}_w"] = w.permute(0, 3, 2, 1).reshape(G * D, 4 * D).contiguous()   # [group][in][tap][out]
    T["wn_skip_w"] = t(P["wn_skip_w"])                                  # (G*D, D)
    T["wn_final_w"] = t(P["wn_final_w"])
    for l in range(model.depth):
        T[f"l{l}_qkv"] = t(P[f"l{l}_qkv"])                              # (D, 3*inner)
        T[f"l{l}_o"] = t(P[f"l{l}_o"])                                  # (inner, D)
        T[f"l{l}_ff_w1"] = t(P[f"l{l}_ff_w1"])                          # (D, 2*Dp)
        T[f"l{l}_ff_wc"] = _transpose_conv(P[f"l{l}_ff_wc"], 3)         # (Dp, 3*Dp)
        T[f"l{l}_ff_w2"] = t(P[f"l{l}_ff_w2"])                          # (Dp, D)
    T["pred_w"] = t(P["pred_w"])
    T["wn_init_w"] = _transpose_conv(P["wn_init_w"], 3)
    if model.condition_on_prompt:
        T["cond_w"] = t(P["cond_w"])                                   # (dim_prompt, D): d cond
        if "pr_proj_w" in P:
            T["pr_proj_w"] = t(P["pr_proj_w"])                         # (dim_prompt, D): d prompt
        T["x_kv_all"] = t(P["x_kv_all"])                               # (D, depth*2*inner)
        for l in range(model.depth):
            T[f"l{l}_xq"] = t(P[f"l{l}_xq"])
            T[f"l{l}_xo"] = t(P[f"l{l}_xo"])
        for i in range(len(model.perceiver_resampler.layers)):
            for k in ("q", "kv", "o", "ff_w1", "ff_w2"):
                T[f"pr{i}_{k}"] = t(P[f"pr{i}_{k}"])
    return T


def geglu_backward(h, d_g, w1, b1, w1_t, Di: int, grads: Dict[str, torch.Tensor], name: str) -> torch.Tensor:
    """Backward of g = GEGLU(h @ w1^T + b1), w1 / b1 packed by `model._pack_geglu` (inner width Di padded to Dp): the
    pre-activation is recomputed with a plain-epilogue GEMM, lin1's gradients go to grads[name + ".weight" / ".bias"] in
    the reference's layout (value rows, then gate rows), and d h (bf16) is returned."""
    B, N, D = h.shape
    Dp = w1.shape[0] // 2
    dev = h.device
    pre = ops.gemm(h, w1, torch.empty(B, N, 2 * Dp, device=dev, dtype=bf), n=2 * Dp, epilogue=ops.EPI_BF16, bias=b1)
    ops.geglu_bwd(pre, d_g)                                                              # pre <- d pre
    dW1 = ops.wgrad(pre, h, torch.zeros(2 * Dp, D, device=dev), n=2 * Dp, k=D).view(Dp // 128, 2, 128, D)
    db1 = ops.colsum(pre, torch.zeros(2 * Dp, device=dev)).view(Dp // 128, 2, 128)
    grads[name + ".weight"] = torch.cat((dW1[:, 0].reshape(Dp, D)[:Di], dW1[:, 1].reshape(Dp, D)[:Di]), dim=0)
    grads[name + ".bias"] = torch.cat((db1[:, 0].reshape(Dp)[:Di], db1[:, 1].reshape(Dp)[:Di]), dim=0)
    return ops.gemm(pre, w1_t, torch.empty(B, N, D, device=dev, dtype=bf), n=D, epilogue=ops.EPI_BF16)


def attention_backward(L: dict, dxr, dxr_bf, w_o_t, w_qkv_t, heads: int, grads: Dict[str, torch.Tensor], name: str,
                       **norm) -> None:
    """Backward of x += Wo attn(Wqkv h1), h1 = RMSNorm(x_in), from the layer record L (x_in, h1, qkv, lse, ao):
    to_out / to_q / to_kv gradients go to grads[name + ...]; dxr (fp32, in place) and dxr_bf become the gradient of x_in.
    `norm` is the RMSNorm's part of ops.rmsnorm_film_bwd: film= / dfilm= or gamma= / dgamma=."""
    B, N, D = dxr.shape
    inner = heads * 64
    dev = dxr.device
    grads[name + "to_out.weight"] = ops.wgrad(dxr_bf, L["ao"], torch.zeros(D, inner, device=dev), n=D, k=inner)
    d_ao = ops.gemm(dxr_bf, w_o_t, torch.empty(B, N, inner, device=dev, dtype=bf), n=inner, epilogue=ops.EPI_BF16)
    qkv = L["qkv"]
    d_qkv = torch.empty(B, N, 3 * inner, device=dev, dtype=bf)
    dq = torch.zeros(B, N, inner, device=dev)
    ops.attention_bwd(qkv[:, :, :inner], qkv[:, :, inner:2 * inner], qkv[:, :, 2 * inner:], L["ao"], d_ao, L["lse"],
                      dq, d_qkv[:, :, inner:2 * inner], d_qkv[:, :, 2 * inner:], heads=heads)
    d_qkv[:, :, :inner].copy_(dq)   # fp32 accumulator -> bf16 slot (layout glue)
    dWqkv = ops.wgrad(d_qkv, L["h1"], torch.zeros(3 * inner, D, device=dev), n=3 * inner, k=D)
    grads[name + "to_q.weight"] = dWqkv[:inner]
    grads[name + "to_kv.weight"] = dWqkv[inner:]
    dh1 = ops.gemm(d_qkv, w_qkv_t, torch.empty(B, N, D, device=dev, dtype=bf), n=D, epilogue=ops.EPI_BF16)
    ops.rmsnorm_film_bwd(L["x_in"], dh1, dxr, dxr_bf, rows_per_batch=N, **norm)


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
    Dp = _round_up(Di, 128)
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
    dout_bf = ops.cast_bf16(d_out.float().contiguous(), e(B, N, D))
    grads["transformer.to_pred.1.weight"] = ops.wgrad(dout_bf, S["hf"], z(D, D), n=D, k=D)
    dhf = ops.gemm(dout_bf, T["pred_w"], e(B, N, D), n=D, epilogue=ops.EPI_BF16)
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
    for l in reversed(range(model.depth)):
        L = S["layers"][l]
        pfx = f"transformer.layers.{l}."
        fo = model._film_tr_off + l * npl * 2 * D
        fo3 = fo + (npl - 1) * 2 * D
        # ---- feed-forward branch: x += W2 conv(GEGLU(W1 h2)) ----
        dW2 = ops.wgrad(dxr_bf, L["ff_c"], z(D, Dp), n=D, k=Dp)
        grads[pfx + "5.3.weight"] = dW2[:, :Di]
        grads[pfx + "5.3.bias"] = ops.colsum(dxr_bf, z(D))
        d_c = ops.gemm(dxr_bf, T[f"l{l}_ff_w2"], e(B, N, Dp), n=Dp, epilogue=ops.EPI_BF16)
        dWc = z(Dp, 3 * Dp)
        for tap in range(3):   # tap t multiplies g[n - (2 - t)]
            ops.wgrad(d_c, L["ff_g"], dWc[:, tap * Dp:(tap + 1) * Dp], n=Dp, k=Dp, shift_units=2 - tap)
        grads[pfx + "5.2.1.weight"] = dWc.view(Dp, 3, Dp)[:Di, :, :Di].permute(0, 2, 1)
        grads[pfx + "5.2.1.bias"] = ops.colsum(d_c, z(Dp))[:Di]
        d_g = ops.gemm(d_c, T[f"l{l}_ff_wc"], e(B, N, Dp), n=Dp, epilogue=ops.EPI_BF16, segs=ops.conv_dgrad_segs(Dp, 3, 2))
        dh2 = geglu_backward(L["h2"], d_g, P[f"l{l}_ff_w1"], P[f"l{l}_ff_b1"], T[f"l{l}_ff_w1"], Di, grads, pfx + "5.0")
        ops.rmsnorm_film_bwd(L["x_mid"], dh2, dxr, dxr_bf, rows_per_batch=N, film=film[:, fo3:fo3 + 2 * D],
                             dfilm=dfilm[:, fo3:fo3 + 2 * D])
        # ---- cross-attention branch: x += Wxo attn(Wxq h_x, Wxkv c) ----
        if conditional:
            fo2 = fo + 2 * D
            grads[pfx + "3.to_out.weight"] = ops.wgrad(dxr_bf, L["ao2"], z(D, inner), n=D, k=inner)
            d_ao2 = ops.gemm(dxr_bf, T[f"l{l}_xo"], e(B, N, inner), n=inner, epilogue=ops.EPI_BF16)
            kv = S["xkv"][:, :, l * 2 * inner:(l + 1) * 2 * inner]
            dkv = d_xkv[:, :, l * 2 * inner:(l + 1) * 2 * inner]
            dq2 = z(B, N, inner)
            ops.attention_bwd(L["xq"], kv[:, :, :inner], kv[:, :, inner:], L["ao2"], d_ao2, L["lse2"], dq2,
                              dkv[:, :, :inner], dkv[:, :, inner:], heads=H)
            dq2_bf = ops.cast_bf16(dq2, e(B, N, inner))
            grads[pfx + "3.to_q.weight"] = ops.wgrad(dq2_bf, L["h_x"], z(inner, D), n=inner, k=D)
            dh_x = ops.gemm(dq2_bf, T[f"l{l}_xq"], e(B, N, D), n=D, epilogue=ops.EPI_BF16)
            ops.rmsnorm_film_bwd(L["x_c"], dh_x, dxr, dxr_bf, rows_per_batch=N, film=film[:, fo2:fo2 + 2 * D],
                                 dfilm=dfilm[:, fo2:fo2 + 2 * D])
        # ---- attention branch: x += Wo attn(Wqkv h1) ----
        attention_backward(L, dxr, dxr_bf, T[f"l{l}_o"], T[f"l{l}_qkv"], H, grads, pfx + "1.",
                           film=film[:, fo:fo + 2 * D], dfilm=dfilm[:, fo:fo + 2 * D])
        # FiLM projections of this layer's norms: their rows of dfilm are final now, so the weight gradient (the largest
        # gradient buffers of the model) joins this layer's all-reduce instead of trailing the whole backward
        dWl = ops.film_wgrad(dfilm[:, fo:fo + npl * 2 * D], t_cond, torch.empty(npl * 2 * D, model.dim_cond, device=dev),
                             accumulate=False)
        for k, idx in enumerate((0, 2, 4) if conditional else (0, 4)):
            grads[pfx + f"{idx}.to_gamma_beta.weight"] = dWl[k * 2 * D:(k + 1) * 2 * D]
        flush()   # this layer's gradients are final: their all-reduce overlaps the layers still to come

    if conditional:
        # d of the perceiver context: bf16 d(proj) when it has a projection, else fp32 d(prompt)
        d_ctx = _conditioning_backward_tokens(model, S, T, d_xkv, grads)
        if want_prompt:
            # d prompt, term (a): through the perceiver's context projection (identity when dim_prompt == dim)
            if "pr_proj_w" in P:
                input_grads["prompt"] = ops.gemm(d_ctx, T["pr_proj_w"], e(B, S["pr_Np"], model.dim_prompt, dt=torch.float32),
                                                 n=model.dim_prompt, epilogue=ops.EPI_F32)
            else:
                input_grads["prompt"] = d_ctx
    # ---- wavenet: final 1x1 conv, skip sum, 4 stacks of 8 dilation columns, init conv ----
    grads["wavenet.final_conv.weight"] = ops.wgrad(dxr_bf, S["skip"], z(D, D), n=D, k=D).unsqueeze(-1)
    grads["wavenet.final_conv.bias"] = ops.colsum(dxr_bf, z(D))
    d_skip = ops.gemm(dxr_bf, T["wn_final_w"], e(B, N, D), n=D, epilogue=ops.EPI_BF16)
    last = S["stack_out"][-1]
    dWskip = ops.wgrad(d_skip, last, z(D, G * D), n=D, k=G * D)
    dbskip = ops.colsum(d_skip, z(D))
    nst = model.wavenet_stacks
    for g in range(G):
        grads[f"wavenet.stacks.{nst - 1}.blocks.{g}.skip_conv.weight"] = dWskip[:, g * D:(g + 1) * D].unsqueeze(-1)
        grads[f"wavenet.stacks.{nst - 1}.blocks.{g}.skip_conv.bias"] = dbskip
    # dcy: [dc | dy] halves, so that one grouped dgrad GEMM reads the conv taps from dc and the 1x1 res conv from dy
    dcy = e(B, N, 2 * G * D)
    ops.gemm(d_skip, T["wn_skip_w"], dcy[:, :, G * D:], n=G * D, epilogue=ops.EPI_BF16)     # d y of the last stack
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
        dWp = z(G * D, 4 * D)
        for tap in range(3):
            ops.wgrad(dc, x_in, dWp[:, tap * D:(tap + 1) * D], n=D, k=D, shift_units=2 - tap, groups=G,
                      dy_group_col_stride=D, x_group_col_stride=gcs, dw_group_row_stride=D, dil=dil)
        ops.wgrad(dy, x_in, dWp[:, 3 * D:], n=D, k=D, groups=G, dy_group_col_stride=D, x_group_col_stride=gcs,
                  dw_group_row_stride=D)
        dbc, dbr = ops.colsum(dc, z(G * D)), ops.colsum(dy, z(G * D))
        for g in range(G):
            blk = f"wavenet.stacks.{s}.blocks.{g}."
            w = dWp[g * D:(g + 1) * D]
            grads[blk + "conv.weight"] = w[:, :3 * D].view(D, 3, D).permute(0, 2, 1)
            grads[blk + "res_conv.weight"] = w[:, 3 * D:].unsqueeze(-1)
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
    dWi = z(D, 3 * D)
    for tap in range(3):
        ops.wgrad(d_h0, S["x_bf"], dWi[:, tap * D:(tap + 1) * D], n=D, k=D, shift_units=2 - tap)
    grads["wavenet.init_conv.weight"] = dWi.view(D, 3, D).permute(0, 2, 1)
    grads["wavenet.init_conv.bias"] = ops.colsum(d_h0, z(D))
    if conditional:
        # x_in = x + pad_or_curtail(where(cdrop, null_cond, cond_proj)) (ns2.py:978-992): d x_in from the init conv's dgrad
        d_xin = ops.gemm(d_h0, T["wn_init_w"], e(B, N, D), n=D, epilogue=ops.EPI_BF16, segs=ops.conv_dgrad_segs(D, 3, 2))
        Lc = S["Lc"]
        n_used = min(Lc, N)
        keep = (~S["cdrop"])[:, None, None]
        d_cp = torch.zeros(B, Lc, D, device=dev, dtype=bf)
        d_cp[:, :n_used] = torch.where(keep, d_xin[:, :n_used], torch.zeros((), device=dev, dtype=bf))   # masking glue
        grads["null_cond"] = (d_xin[:, :n_used].float() * S["cdrop"][:, None, None]).sum((0, 1)).unsqueeze(-1)
        grads["cond_to_model_dim.weight"] = ops.wgrad(d_cp, S["cond_bf"], z(D, model.dim_prompt), n=D,
                                                      k=model.dim_prompt).unsqueeze(-1)
        grads["cond_to_model_dim.bias"] = ops.colsum(d_cp, z(D))
        if want_cond:
            # d cond = d_cp @ W (1x1 conv dgrad), token-major; curtailed frames (n >= N) stay exact zeros.  Returned as
            # the channel-first view cond has, so nothing is transposed.
            d_cond = ops.gemm(d_cp, T["cond_w"], e(B, Lc, model.dim_prompt, dt=torch.float32), n=model.dim_prompt,
                              epilogue=ops.EPI_F32)
            input_grads["cond"] = d_cond.permute(0, 2, 1)

    # ---- FiLM projections (one stacked matrix) and the timestep embedding ----
    rows = film.shape[1]
    dbf = dfilm.sum(0)
    dfilm_bf = ops.cast_bf16(dfilm, e(1, B, rows))
    dt = ops.gemm(dfilm_bf, T["film_w"], e(1, B, model.dim_cond, dt=torch.float32), n=model.dim_cond, epilogue=ops.EPI_F32)[0]
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
            ops.add_rows_bcast(input_grads["prompt"], mean.grad.contiguous(), 1.0 / S["pr_Np"])
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


def _conditioning_backward_tokens(model, S, T, d_xkv, grads):
    """Backward of everything that produced the cross-attention context: the stacked K/V projection of all layers,
    the null-token substitution and the PerceiverResampler (ns2.py:532-579, 964-968)."""
    P = model.packed()
    B, D, M, inner, H = S["B"], model.dim, model.num_latents_m, model.inner, model.heads
    Di = model.ff_inner
    Dp = _round_up(Di, 128)
    dev = d_xkv.device
    e = lambda *s, dt=bf: torch.empty(*s, device=dev, dtype=dt)
    z = lambda *s: torch.zeros(*s, device=dev, dtype=torch.float32)
    dWkv = ops.wgrad(d_xkv, S["c_bf"], z(model.depth * 2 * inner, D), n=model.depth * 2 * inner, k=D)
    for l in range(model.depth):
        grads[f"transformer.layers.{l}.3.to_kv.weight"] = dWkv[l * 2 * inner:(l + 1) * 2 * inner]
    d_c = ops.gemm(d_xkv, T["x_kv_all"], e(B, M, D), n=D, epilogue=ops.EPI_BF16).float()
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
    ctx = M + Np
    d_proj = z(B, Np, D)
    for i in reversed(range(len(pr.layers))):
        L = S["pr_layers"][i]
        pfx = f"perceiver_resampler.layers.{i}."
        # feed-forward (no conv, no pre-norm): lat += W2 GEGLU(W1 lat)
        grads[pfx + "1.2.weight"] = ops.wgrad(dlat_bf, L["g"], z(D, Dp), n=D, k=Dp)[:, :Di]
        grads[pfx + "1.2.bias"] = ops.colsum(dlat_bf, z(D))
        d_g = ops.gemm(dlat_bf, T[f"pr{i}_ff_w2"], e(B, M, Dp), n=Dp, epilogue=ops.EPI_BF16)
        ops.accum_bf16(dlat, geglu_backward(L["lat_bf2"], d_g, P[f"pr{i}_ff_w1"], P[f"pr{i}_ff_b1"], T[f"pr{i}_ff_w1"], Di,
                                            grads, pfx + "1.0"), dlat_bf)
        # attention over cat(latents, projected prompt): lat += Wo attn(Wq lat, Wkv cat)
        grads[pfx + "0.to_out.weight"] = ops.wgrad(dlat_bf, L["o"], z(D, inner), n=D, k=inner)
        d_o = ops.gemm(dlat_bf, T[f"pr{i}_o"], e(B, M, inner), n=inner, epilogue=ops.EPI_BF16)
        dq = z(B, M, inner)
        d_kv = e(B, ctx, 2 * inner)
        ops.attention_bwd(L["q"], L["kv"][:, :, :inner], L["kv"][:, :, inner:], L["o"], d_o, L["lse"], dq, d_kv[:, :, :inner],
                          d_kv[:, :, inner:], heads=H)
        dq_bf = ops.cast_bf16(dq, e(B, M, inner))
        grads[pfx + "0.to_q.weight"] = ops.wgrad(dq_bf, L["lat_bf"], z(inner, D), n=inner, k=D)
        grads[pfx + "0.to_kv.weight"] = ops.wgrad(d_kv, L["cat"], z(2 * inner, D), n=2 * inner, k=D)
        d_cat = ops.gemm(d_kv, T[f"pr{i}_kv"], e(B, ctx, D), n=D, epilogue=ops.EPI_BF16)
        ops.accum_bf16(dlat, ops.gemm(dq_bf, T[f"pr{i}_q"], e(B, M, D), n=D, epilogue=ops.EPI_BF16))
        ops.accum_bf16(dlat, d_cat[:, :M].contiguous(), dlat_bf)
        ops.accum_bf16(d_proj, d_cat[:, M:].contiguous())
    grads["perceiver_resampler.latents"] = dlat.sum(0)
    if "pr_proj_w" in P:
        d_proj_bf = ops.cast_bf16(d_proj, e(B, Np, D))
        grads["perceiver_resampler.proj_context.weight"] = ops.wgrad(d_proj_bf, S["pr_p_bf"], z(D, model.dim_prompt), n=D,
                                                                     k=model.dim_prompt)
        grads["perceiver_resampler.proj_context.bias"] = ops.colsum(d_proj_bf, z(D))
        return d_proj_bf
    return d_proj


class DenoiserFunction(torch.autograd.Function):
    """One autograd node for the whole denoiser: forward saves activations, backward runs the kernels above."""

    @staticmethod
    def forward(ctx, model, x, times, prompt, cond, cond_drop_prob, *params):
        saved = {}
        out = model._forward_impl(x, times, prompt, cond=cond, cond_drop_prob=cond_drop_prob, saved=saved)
        ctx.model, ctx.saved = model, saved
        ctx.names = [n for n, _ in model.named_parameters()]
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
        missing = [n for n in ctx.names if n not in grads]
        if missing:
            raise RuntimeError(f"backward produced no gradient for {missing[:4]}...")
        d_prompt, d_cond = inputs.get("prompt"), inputs.get("cond")
        if d_prompt is not None:
            d_prompt = d_prompt.to(ctx.in_dtypes[0])
        if d_cond is not None:
            d_cond = d_cond.to(ctx.in_dtypes[1])
        return (None, None, None, d_prompt, d_cond, None, *[grads[n].reshape(p.shape).to(p.dtype)
                                                          for n, p in ctx.model.named_parameters()])


class MseRowsFunction(torch.autograd.Function):
    """Per-sample mean squared error (ns2.py:1646-1647) with the hand-written forward / backward kernels."""

    @staticmethod
    def forward(ctx, pred, target):
        pred, target = pred.contiguous(), target.contiguous()
        ctx.save_for_backward(pred, target)
        return ops.mse_rows(pred, target, torch.empty(pred.shape[0], device=pred.device))

    @staticmethod
    def backward(ctx, d_rows):
        pred, target = ctx.saved_tensors
        per = pred.numel() // pred.shape[0]
        coef = (d_rows.float() * (2.0 / per)).contiguous()
        return ops.mse_bwd(pred, target, coef, out_f32=torch.empty_like(pred)), None
