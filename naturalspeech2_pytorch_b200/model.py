"""`Model`: the NaturalSpeech2 denoiser (time FiLM -> Wavenet -> conditionable Transformer) on sm_90a kernels.

Drop-in for `naturalspeech2_pytorch.Model` (ns2.py:811-1000): same constructor, same `forward` /
`forward_with_cond_scale` signatures, same parameter names and shapes (SURVEY Appendix B), so a reference
state_dict loads unchanged.  The module tree below only *holds* parameters (nn.Linear / nn.Conv1d instances are
never called); the math runs through `ops` (libns2b200.so):

  time embedding     ops.time_cond                         ns2.py:108-120, 839-843
  all FiLM vectors   one stacked GEMM for the 32 wavenet blocks + every adaptive RMSNorm   ns2.py:613,731
  Wavenet            init conv, 4 launches of 8 dilation columns each (conv + res_conv + FiLM + gate fused),
                     skip sum as one K=8*dim GEMM, final conv                              ns2.py:597-725
  Transformer layer  RMSNorm+FiLM -> fused QKV GEMM -> flash attention -> out-proj(+residual)
                     [-> cross attention over the perceiver latents]
                     -> RMSNorm+FiLM -> GEGLU GEMM -> causal k=3 conv GEMM with the out projection folded
                     into its taps (+residual)                                             ns2.py:786-809
Numerics: bf16 tensor-core operands, fp32 accumulation, fp32 residual stream / norm statistics / softmax,
fp32 output (the protocol of SURVEY section 7, H1).
"""
from __future__ import annotations

import math
import weakref
from collections import OrderedDict
from typing import Dict, Optional

import torch
from torch import nn

from . import ops

_KBLK = 64


def _exists(v):
    return v is not None


def _round_up(v: int, m: int) -> int:
    return (v + m - 1) // m * m


def _bf(t):
    return t.detach().to(torch.bfloat16).contiguous()


def _pack_geglu(lin1: nn.Linear, lin2: nn.Linear) -> Dict[str, torch.Tensor]:
    """GEGLU FeedForward Linear pair (ns2.py:1001-1025) -> {w1, b1, w2, b2}: the inner width zero-padded to Dp, a multiple
    of 128, and lin1's value and gate rows interleaved in 128-row tiles, so that one EPI_GEGLU tile holds a value block
    and its gate block.  `training.geglu_backward` turns the gradient of this layout back into lin1's."""
    D, Di = lin1.weight.shape[1], lin2.weight.shape[1]
    Dp = _round_up(Di, 128)
    dev = lin1.weight.device
    wv = torch.zeros(Dp, D, device=dev)
    wg = torch.zeros(Dp, D, device=dev)
    wv[:Di], wg[:Di] = lin1.weight[:Di], lin1.weight[Di:]  # first half = value, second = gate (ns2.py:1006)
    bv = torch.zeros(Dp, device=dev)
    bg = torch.zeros(Dp, device=dev)
    bv[:Di], bg[:Di] = lin1.bias[:Di], lin1.bias[Di:]
    w1 = torch.stack((wv.view(-1, 128, D), wg.view(-1, 128, D)), dim=1).reshape(2 * Dp, D)
    b1 = torch.stack((bv.view(-1, 128), bg.view(-1, 128)), dim=1).reshape(2 * Dp)
    w2 = torch.zeros(D, Dp, device=dev)
    w2[:, :Di] = lin2.weight
    return {"w1": _bf(w1), "b1": b1.float().contiguous(), "w2": _bf(w2), "b2": lin2.bias.detach().float().contiguous()}


def _pack_conv(w: torch.Tensor, i_pad: Optional[int] = None, o_pad: Optional[int] = None) -> torch.Tensor:
    """Conv1d weight (O, I, k) -> bf16 (o_pad, k*i_pad), tap t at columns [t*i_pad, t*i_pad + I); zero padded."""
    O, I, k = w.shape
    i_pad, o_pad = i_pad or I, o_pad or O
    out = w.new_zeros(o_pad, k, i_pad)
    out[:O, :, :I] = w.detach().permute(0, 2, 1)
    return _bf(out.view(o_pad, k * i_pad))


def _fold_conv_linear(convs, lins, i_pad: int):
    """Each conv followed by a Linear with nothing between them (FeedForward's causal conv and output projection,
    ns2.py:1019-1024) as ONE conv from the conv's input straight to the Linear's output:
    tap t = W2 @ Wc[:, :, t], bias = W2 @ bc + b2.  Returns per pair (the `_pack_conv` layout, input width zero-padded to
    i_pad; the fp32 bias).  On CUDA one `ops.fold_conv_linear` launch folds every pair (fp32 accumulation, no TF32,
    rounded to bf16 once); parameters on the CPU, where no kernel runs, are folded in float64."""
    st = lambda ts: torch.stack([t.detach().float() for t in ts]).contiguous()  # noqa: E731
    if convs[0].weight.is_cuda:
        wo, bo = ops.fold_conv_linear(st(l.weight for l in lins), st(c.weight for c in convs),
                                      st(c.bias for c in convs), st(l.bias for l in lins), i_pad)
        return list(zip(wo.unbind(0), bo.unbind(0)))
    out = []
    for conv, lin in zip(convs, lins):
        w2 = lin.weight.detach().double()
        w = torch.einsum("od,dit->oit", w2, conv.weight.detach().double())    # (D, Di, 3)
        b = w2 @ conv.bias.detach().double() + lin.bias.detach().double()
        out.append((_pack_conv(w, i_pad), b.float().contiguous()))
    return out


def _transpose_conv(w: torch.Tensor, kernel: int) -> torch.Tensor:
    """`_pack_conv` layout (O, k*I) -> (I, k*O) [in][tap][out] pack for the dgrad GEMM."""
    O = w.shape[0]
    return w.view(O, kernel, -1).permute(2, 1, 0).reshape(-1, kernel * O).contiguous()


def _capture(step) -> torch.cuda.CUDAGraph:
    """Warm `step` up on a side stream (workspaces, packing, lazy CUDA init), then capture it into a CUDA graph."""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    # thread_local: other threads (e.g. the NCCL watchdog) may touch CUDA while this thread captures
    with torch.cuda.graph(graph, capture_error_mode="thread_local"):
        step()
    return graph


def _records_graph(m: nn.Module) -> bool:
    """Whether a call of `m` records its hand-written autograd node: train mode, gradients on, a trainable parameter."""
    return m.training and torch.is_grad_enabled() and any(p.requires_grad for p in m.parameters())


class _PackedCache(nn.Module):
    """Packed bf16 weights of a parameter-holding module: `_pack()` builds the forward packs and `_pack_transposed(P)`
    their transposed twins for the dgrad GEMMs of the backward pass.  Both are rebuilt when a parameter changes."""

    def __init__(self):
        super().__init__()
        self._packed: Optional[Dict[str, torch.Tensor]] = None
        self._packed_sig = None
        self._packed_T: Optional[Dict[str, torch.Tensor]] = None
        self.register_load_state_dict_post_hook(lambda module, incompatible: module.invalidate_packed())

    def invalidate_packed(self) -> None:
        """Drop the packed weights.  Called automatically by `load_state_dict`, `.to()` / `.cuda()` / `.float()` and
        whenever a parameter's version counter moves (optimizer steps, in-place ops).  Updates made THROUGH `.data`
        (e.g. the `p.data.lerp_()` of ema_pytorch) do not bump the version counter: call this after them."""
        self._packed = self._packed_sig = self._packed_T = None

    def _apply(self, fn, *args, **kwargs):
        out = super()._apply(fn, *args, **kwargs)
        self.invalidate_packed()
        return out

    def packed(self) -> Dict[str, torch.Tensor]:
        sig = tuple((p.data_ptr(), p._version) for p in self.parameters())
        if self._packed is None or sig != self._packed_sig:
            self.invalidate_packed()   # and whatever a subclass built on the old packs
            with torch.no_grad():
                self._packed = self._pack()
            self._packed_sig = sig
        return self._packed

    def packed_transposed(self) -> Dict[str, torch.Tensor]:
        """Transposed bf16 packs for the dgrad GEMMs of the backward pass (training.py), rebuilt with `packed()`."""
        P = self.packed()
        if self._packed_T is None:
            with torch.no_grad():
                self._packed_T = self._pack_transposed(P)
        return self._packed_T


class _NoParam(nn.Module):
    """Placeholder keeping Sequential indices aligned with the reference (Reduce / Rearrange / GEGLU / SiLU)."""


class _SinusoidalFreqs(nn.Module):
    """Parameter holder of LearnedSinusoidalPosEmb (ns2.py:108-120): `weights` (dim/2,)."""

    def __init__(self, dim: int):
        super().__init__()
        assert dim % 2 == 0
        self.weights = nn.Parameter(torch.randn(dim // 2))


class _AttentionParams(nn.Module):
    """Parameter holder of Attention (ns2.py:1029-1053): to_q, to_kv, to_out, all bias-free."""

    def __init__(self, dim: int, dim_head: int, heads: int):
        super().__init__()
        inner = dim_head * heads
        self.to_q = nn.Linear(dim, inner, bias=False)
        self.to_kv = nn.Linear(dim, inner * 2, bias=False)
        self.to_out = nn.Linear(inner, dim, bias=False)


class _RMSNormParams(nn.Module):
    """Parameter holder of RMSNorm (ns2.py:727-734)."""

    def __init__(self, dim: int, scale: bool = True, dim_cond: Optional[int] = None):
        super().__init__()
        self.to_gamma_beta = nn.Linear(dim_cond, dim * 2) if _exists(dim_cond) else None
        self.gamma = nn.Parameter(torch.ones(dim)) if scale else None


def _feedforward_params(dim: int, mult: int, causal_conv: bool) -> nn.Sequential:
    """Same Sequential indices (and RNG order: conv first) as FeedForward (ns2.py:1009-1025)."""
    inner = int(dim * mult * 2 / 3)
    conv = None
    if causal_conv:
        conv = nn.Sequential(_NoParam(), nn.Conv1d(inner, inner, 3), _NoParam())
    mods = [nn.Linear(dim, inner * 2), _NoParam()]
    if conv is not None:
        mods.append(conv)
    mods.append(nn.Linear(inner, dim))
    return nn.Sequential(*mods)


class _WavenetBlockParams(nn.Module):
    def __init__(self, dim: int, dilation: int, skip_conv: bool, dim_cond_mult: int):
        super().__init__()
        self.to_time_cond = nn.Linear(dim * dim_cond_mult, dim * 2)
        self.conv = nn.Conv1d(dim, dim, 3, dilation=dilation)
        self.res_conv = nn.Conv1d(dim, dim, 1)
        self.skip_conv = nn.Conv1d(dim, dim, 1) if skip_conv else None


class _WavenetStackParams(nn.Module):
    def __init__(self, dim: int, layers: int, has_skip: bool, dim_cond_mult: int):
        super().__init__()
        self.has_skip = has_skip
        self.blocks = nn.ModuleList([
            _WavenetBlockParams(dim, 2 ** i, has_skip, dim_cond_mult) for i in range(layers)])


class _WavenetParams(nn.Module):
    def __init__(self, dim: int, stacks: int, layers: int, dim_cond_mult: int):
        super().__init__()
        self.init_conv = nn.Conv1d(dim, dim, 3)
        self.stacks = nn.ModuleList([
            _WavenetStackParams(dim, layers, s == stacks - 1, dim_cond_mult) for s in range(stacks)])
        self.final_conv = nn.Conv1d(dim, dim, 1)


class _TransformerParams(nn.Module):
    def __init__(self, dim, depth, dim_head, heads, ff_mult, dim_cond_mult, cross_attn):
        super().__init__()
        dim_cond = dim * dim_cond_mult
        self.layers = nn.ModuleList([])
        for _ in range(depth):
            self.layers.append(nn.ModuleList([
                _RMSNormParams(dim, scale=False, dim_cond=dim_cond),
                _AttentionParams(dim, dim_head, heads),
                _RMSNormParams(dim, scale=False, dim_cond=dim_cond) if cross_attn else None,
                _AttentionParams(dim, dim_head, heads) if cross_attn else None,
                _RMSNormParams(dim, scale=False, dim_cond=dim_cond),
                _feedforward_params(dim, ff_mult, causal_conv=True),
            ]))
        self.to_pred = nn.Sequential(_RMSNormParams(dim), nn.Linear(dim, dim, bias=False))


class _PerceiverParams(nn.Module):
    def __init__(self, dim, depth, dim_context, num_latents, dim_head, heads, ff_mult=4):
        super().__init__()
        self.ff_inner = int(dim * ff_mult * 2 / 3)   # its own feed-forward width: the reference keeps ff_mult=4 here
        self.proj_context = nn.Linear(dim_context, dim) if dim_context != dim else nn.Identity()
        self.latents = nn.Parameter(torch.randn(num_latents, dim))
        nn.init.normal_(self.latents, std=0.02)
        self.layers = nn.ModuleList([
            nn.ModuleList([_AttentionParams(dim, dim_head, heads), _feedforward_params(dim, ff_mult, False)])
            for _ in range(depth)])
        self.norm = _RMSNormParams(dim)


class Conditioning(dict):
    """Timestep-invariant conditioning of one (prompt, cond) pair (`Model.precompute_conditioning`): a dict subclass so
    that captured CUDA graphs can remember — through a weak reference — which conditioning their static buffers hold."""


def _prob_mask_like(shape, prob, device):
    # ns2.py:79-85 — kept in torch so the RNG stream matches the reference (SURVEY H7)
    if prob == 1:
        return torch.ones(shape, device=device, dtype=torch.bool)
    if prob == 0:
        return torch.zeros(shape, device=device, dtype=torch.bool)
    return torch.zeros(shape, device=device).float().uniform_(0, 1) < prob


class Model(_PackedCache):
    """H100 denoiser; constructor and call signatures of ns2.py:811-937."""

    def __init__(self, dim, *, depth, dim_head=64, heads=8, ff_mult=4, wavenet_layers=8,
                 wavenet_stacks=4, dim_cond_mult=4, use_flash_attn=True, dim_prompt=None,
                 num_latents_m=32, resampler_depth=2, cond_drop_prob=0., condition_on_prompt=False):
        super().__init__()
        if dim_head != 64:
            raise NotImplementedError("the sm_90a attention kernel is specialised for dim_head=64")
        if dim % 128 != 0 or dim > 1024:
            raise NotImplementedError("dim must be a multiple of 128 (<= 1024) for the sm_90a kernels")
        if not 1 <= wavenet_layers <= 8:
            raise NotImplementedError("wavenet_layers must be in [1, 8] (one launch covers <= 8 dilation columns)")
        self.dim = dim
        self.depth = depth
        self.heads = heads
        self.dim_head = dim_head
        self.inner = heads * dim_head
        self.ff_inner = int(dim * ff_mult * 2 / 3)
        self.wavenet_layers = wavenet_layers
        self.wavenet_stacks = wavenet_stacks
        self.num_latents_m = num_latents_m
        self.dim_prompt = dim_prompt
        self.use_flash_attn = use_flash_attn  # accepted for signature parity; the flash kernel is the only path

        dim_time = dim * dim_cond_mult
        self.dim_time = dim_time
        self.to_time_cond = nn.Sequential(_SinusoidalFreqs(dim), nn.Linear(dim + 1, dim_time), _NoParam())

        self.cond_drop_prob = cond_drop_prob
        self.condition_on_prompt = condition_on_prompt
        self.to_prompt_cond = None
        if condition_on_prompt:
            assert _exists(dim_prompt), "dim_prompt is required when condition_on_prompt=True"
            if dim_prompt % _KBLK != 0:
                raise NotImplementedError("dim_prompt must be a multiple of 64")
            self.null_prompt_cond = nn.Parameter(torch.randn(dim_time))
            self.null_prompt_tokens = nn.Parameter(torch.randn(num_latents_m, dim))
            nn.init.normal_(self.null_prompt_cond, std=0.02)
            nn.init.normal_(self.null_prompt_tokens, std=0.02)
            self.to_prompt_cond = nn.Sequential(_NoParam(), nn.Linear(dim_prompt, dim_time), _NoParam())
            self.perceiver_resampler = _PerceiverParams(dim, resampler_depth, dim_prompt, num_latents_m,
                                                        dim_head, heads)
        self.null_cond = None
        self.cond_to_model_dim = None
        if condition_on_prompt:
            self.cond_to_model_dim = nn.Conv1d(dim_prompt, dim, 1)
            self.null_cond = nn.Parameter(torch.zeros(dim, 1))

        dim_cond_mult = dim_cond_mult * (2 if condition_on_prompt else 1)
        self.dim_cond = dim * dim_cond_mult
        self.wavenet = _WavenetParams(dim, wavenet_stacks, wavenet_layers, dim_cond_mult)
        self.transformer = _TransformerParams(dim, depth, dim_head, heads, ff_mult, dim_cond_mult,
                                              cross_attn=condition_on_prompt)
        self._ws: "OrderedDict[tuple, Dict[str, torch.Tensor]]" = OrderedDict()
        self.freeze_packed = False  # set True to skip the per-call parameter-version check (inference loops)
        self._prof = None           # bench.py: list collecting (op name, start event, end event)
        self.use_cuda_graphs = False  # replay one captured CUDA graph per problem shape instead of ~110 launches
        self._graphs: "OrderedDict[tuple, dict]" = OrderedDict()   # `_captured`: model and sampler steps
        self.max_cached_shapes = 4  # LRU bound on per-(B, N) workspaces (~1.3 GB each at cfg2); graphs: twice that

    @property
    def device(self):
        return next(self.parameters()).device

    # ----------------------------------------------------------------------------------------------
    # weight packing: fp32 parameters -> bf16 tensor-core layouts (rebuilt whenever a parameter changes)
    # ----------------------------------------------------------------------------------------------
    def invalidate_packed(self) -> None:
        """`_PackedCache.invalidate_packed`, which here also drops every captured CUDA graph (they hold pointers into
        the packed copies)."""
        super().invalidate_packed()
        self._graphs.clear()

    def _apply(self, fn, *args, **kwargs):
        out = super()._apply(fn, *args, **kwargs)
        self._ws.clear()
        return out

    def packed(self) -> Dict[str, torch.Tensor]:
        if self._packed is not None and self.freeze_packed:
            return self._packed
        return super().packed()

    def _pack(self) -> Dict[str, torch.Tensor]:
        D, G = self.dim, self.wavenet_layers
        P: Dict[str, torch.Tensor] = {}
        # ---- every FiLM projection as one stacked (rows, dim_cond) matrix ----
        film_w, film_b = [], []
        for st in self.wavenet.stacks:
            for blk in st.blocks:
                film_w.append(blk.to_time_cond.weight)
                film_b.append(blk.to_time_cond.bias)
        self._film_tr_off = len(film_w) * 2 * D
        self._norms_per_layer = 3 if self.condition_on_prompt else 2
        for layer in self.transformer.layers:
            for idx in (0, 2, 4):
                if layer[idx] is not None:
                    film_w.append(layer[idx].to_gamma_beta.weight)
                    film_b.append(layer[idx].to_gamma_beta.bias)
        P["film_w"] = _bf(torch.cat(film_w, dim=0))
        P["film_b"] = torch.cat(film_b, dim=0).detach().float().contiguous()
        # ---- wavenet ----
        wn = self.wavenet
        P["wn_init_w"] = _pack_conv(wn.init_conv.weight)
        P["wn_init_b"] = wn.init_conv.bias.detach().float().contiguous()
        for s, st in enumerate(wn.stacks):
            ws, bc, br = [], [], []
            for blk in st.blocks:
                ws.append(torch.cat((_pack_conv(blk.conv.weight), _bf(blk.res_conv.weight[:, :, 0])), dim=1))
                bc.append(blk.conv.bias)
                br.append(blk.res_conv.bias)
            P[f"wn{s}_w"] = _bf(torch.cat(ws, dim=0))                      # (G*D, 4*D)
            P[f"wn{s}_b"] = torch.cat(bc + br).detach().float().contiguous()   # [conv biases | res biases]
        last = wn.stacks[-1]
        P["wn_skip_w"] = _bf(torch.cat([b.skip_conv.weight[:, :, 0] for b in last.blocks], dim=1))
        P["wn_skip_b"] = torch.stack([b.skip_conv.bias for b in last.blocks]).sum(0).detach().float().contiguous()
        P["wn_final_w"] = _bf(wn.final_conv.weight[:, :, 0])
        P["wn_final_b"] = wn.final_conv.bias.detach().float().contiguous()
        # ---- transformer ----
        kv_all = []
        for l, layer in enumerate(self.transformer.layers):
            attn = layer[1]
            P[f"l{l}_qkv"] = _bf(torch.cat((attn.to_q.weight, attn.to_kv.weight), dim=0))
            P[f"l{l}_o"] = _bf(attn.to_out.weight)
            if layer[3] is not None:
                P[f"l{l}_xq"] = _bf(layer[3].to_q.weight)
                P[f"l{l}_xo"] = _bf(layer[3].to_out.weight)
                kv_all.append(layer[3].to_kv.weight)
            ff = layer[5]
            for k, v in _pack_geglu(ff[0], ff[-1]).items():
                P[f"l{l}_ff_{k}"] = v
            conv, Dp = ff[2][1], P[f"l{l}_ff_w2"].shape[1]
            P[f"l{l}_ff_wc"] = _pack_conv(conv.weight, Dp, Dp)
            P[f"l{l}_ff_bc"] = torch.zeros(Dp, device=conv.bias.device)
            P[f"l{l}_ff_bc"][:self.ff_inner] = conv.bias
        # the forward runs each FFN's conv and output projection as one conv (wc / bc / w2 stay for the backward)
        ffs = [layer[5] for layer in self.transformer.layers]
        folded = _fold_conv_linear([ff[2][1] for ff in ffs], [ff[-1] for ff in ffs], P["l0_ff_w2"].shape[1])
        for l, (wo, bo) in enumerate(folded):
            P[f"l{l}_ff_wo"], P[f"l{l}_ff_bo"] = wo, bo                     # (D, 3*Dp), (D,)
        if kv_all:
            P["x_kv_all"] = _bf(torch.cat(kv_all, dim=0))  # (depth*2*inner, D): cross K/V of all layers
        P["pred_gamma"] = self.transformer.to_pred[0].gamma.detach().float().contiguous()
        P["pred_w"] = _bf(self.transformer.to_pred[1].weight)
        # ---- conditioning ----
        if self.condition_on_prompt:
            pr = self.perceiver_resampler
            if isinstance(pr.proj_context, nn.Linear):
                P["pr_proj_w"] = _bf(pr.proj_context.weight)
                P["pr_proj_b"] = pr.proj_context.bias.detach().float().contiguous()
            for i, (attn, ff) in enumerate(pr.layers):
                P[f"pr{i}_q"] = _bf(attn.to_q.weight)
                P[f"pr{i}_kv"] = _bf(attn.to_kv.weight)
                P[f"pr{i}_o"] = _bf(attn.to_out.weight)
                for k, v in _pack_geglu(ff[0], ff[-1]).items():
                    P[f"pr{i}_ff_{k}"] = v
            P["cond_w"] = _bf(self.cond_to_model_dim.weight[:, :, 0])
            P["cond_b"] = self.cond_to_model_dim.bias.detach().float().contiguous()
        return P

    def _pack_transposed(self, P: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        D, G = self.dim, self.wavenet_layers
        T: Dict[str, torch.Tensor] = {}
        t = lambda w: w.t().contiguous()  # noqa: E731
        T["film_w"] = t(P["film_w"])                                        # (dim_cond, rows)
        for s in range(self.wavenet_stacks):
            w = P[f"wn{s}_w"].view(G, D, 4, D)                              # [group][out][tap0,tap1,tap2,res][in]
            T[f"wn{s}_w"] = w.permute(0, 3, 2, 1).reshape(G * D, 4 * D).contiguous()   # [group][in][tap][out]
        T["wn_skip_w"] = t(P["wn_skip_w"])                                  # (G*D, D)
        T["wn_final_w"] = t(P["wn_final_w"])
        for l in range(self.depth):
            T[f"l{l}_qkv"] = t(P[f"l{l}_qkv"])                              # (D, 3*inner)
            T[f"l{l}_o"] = t(P[f"l{l}_o"])                                  # (inner, D)
            T[f"l{l}_ff_w1"] = t(P[f"l{l}_ff_w1"])                          # (D, 2*Dp)
            T[f"l{l}_ff_wc"] = _transpose_conv(P[f"l{l}_ff_wc"], 3)         # (Dp, 3*Dp)
            T[f"l{l}_ff_w2"] = t(P[f"l{l}_ff_w2"])                          # (Dp, D)
            T[f"l{l}_ff_wo"] = _transpose_conv(P[f"l{l}_ff_wo"], 3)         # (Dp, 3*D)
        T["pred_w"] = t(P["pred_w"])
        T["wn_init_w"] = _transpose_conv(P["wn_init_w"], 3)
        if self.condition_on_prompt:
            T["cond_w"] = t(P["cond_w"])                                   # (dim_prompt, D): d cond
            if "pr_proj_w" in P:
                T["pr_proj_w"] = t(P["pr_proj_w"])                         # (dim_prompt, D): d prompt
            T["x_kv_all"] = t(P["x_kv_all"])                               # (D, depth*2*inner)
            for l in range(self.depth):
                T[f"l{l}_xq"] = t(P[f"l{l}_xq"])
                T[f"l{l}_xo"] = t(P[f"l{l}_xo"])
            for i in range(len(self.perceiver_resampler.layers)):
                for k in ("q", "kv", "o", "ff_w1", "ff_w2"):
                    T[f"pr{i}_{k}"] = t(P[f"pr{i}_{k}"])
        return T

    # ----------------------------------------------------------------------------------------------
    # workspaces (stable addresses per problem shape so a forward can be captured in a CUDA graph)
    # ----------------------------------------------------------------------------------------------
    @staticmethod
    def _ws_key(B: int, N: int, dev) -> tuple:
        return (B, N, str(dev))

    def _workspace(self, B: int, N: int, dev) -> Dict[str, torch.Tensor]:
        key = self._ws_key(B, N, dev)
        ws = self._ws.get(key)
        if ws is not None:
            self._ws.move_to_end(key)
            return ws
        while len(self._ws) >= self.max_cached_shapes:   # LRU: variable-length serving must not grow without bound
            old_key, _ = self._ws.popitem(last=False)
            for gk in [k for k, e in self._graphs.items() if e["ws_key"] == old_key]:
                del self._graphs[gk]                      # graphs captured on the evicted workspace die with it
        D, G, inner = self.dim, self.wavenet_layers, self.inner
        Dp = _round_up(self.ff_inner, 128)
        bf, f32 = torch.bfloat16, torch.float32
        e = lambda *s, dt=bf: torch.empty(*s, device=dev, dtype=dt)
        ws = {
            "t": e(B, self.dim_cond, dt=f32), "t_bf": e(1, B, self.dim_cond),
            "film": e(1, B, self.packed()["film_w"].shape[0], dt=f32),
            "x_bf": e(B, N, D), "h": e(B, N, D),
            "wn_a": e(B, N, G * D), "wn_b": e(B, N, G * D),
            "x_res": e(B, N, D, dt=f32),
            "qkv": e(B, N, 3 * inner), "attn_o": e(B, N, inner),
            "ff_g": e(B, N, Dp),
        }
        if self.condition_on_prompt:
            M = self.num_latents_m
            ws.update({"xq": e(B, N, inner), "c_bf": e(B, M, D),
                       "xkv": e(B, M, self.depth * 2 * inner)})
        self._ws[key] = ws
        return ws

    def _captured(self, key, ws_key, conditioning, build) -> dict:
        """The one cache of the CUDA graphs that replay on this model's workspaces (its forward, the sampler's step).
        The entry for `key` holds "graph" and every buffer the graph reads or writes.  On a miss, `build(cond)` takes
        the static copy of `conditioning` and returns (buffers, step), and the step is captured on workspace `ws_key`.
        An entry goes with that workspace, with a repack, or as the least recent of 2 * max_cached_shapes."""
        self.packed()   # a parameter-version change repacks, which drops every entry
        entry = self._graphs.get(key)
        if entry is None:
            while len(self._graphs) >= 2 * self.max_cached_shapes:
                self._graphs.popitem(last=False)
            cond = None
            if conditioning is not None:   # static copies: the graph must not pin (or depend on) the caller's tensors
                cond = Conditioning({k: (v.clone() if torch.is_tensor(v) else v) for k, v in conditioning.items()})
            entry, step = build(cond)
            entry.update(graph=_capture(step), cond=cond, ws_key=ws_key)
            self._graphs[key] = entry
        elif conditioning is not None and (entry["cond_ref"] is None or entry["cond_ref"]() is not conditioning):
            for k, v in conditioning.items():    # a different (prompt, cond) of the same shapes: refresh the copies
                if torch.is_tensor(v):
                    entry["cond"][k].copy_(v)
        self._graphs.move_to_end(key)
        entry["cond_ref"] = weakref.ref(conditioning) if isinstance(conditioning, Conditioning) else None
        return entry

    # ----------------------------------------------------------------------------------------------
    # conditioning (timestep-invariant; cache across sampling steps via `precompute_conditioning`)
    # ----------------------------------------------------------------------------------------------
    def _perceiver(self, prompt: torch.Tensor, P: Dict[str, torch.Tensor], saved: Optional[dict] = None,
                   prompt_lens: Optional[torch.Tensor] = None) -> torch.Tensor:
        """PerceiverResampler.forward (ns2.py:568-579) -> (B, M, D) fp32.  With `saved`, every layer's activations are
        kept (fresh buffers per layer) for `training._conditioning_backward_tokens`.  prompt_lens: validated per-sample
        prompt lengths; the keys [latents ; prompt] of sample b are then its first M + prompt_lens[b]."""
        D, M, inner, H = self.dim, self.num_latents_m, self.inner, self.heads
        pr = self.perceiver_resampler
        B, Np, _ = prompt.shape
        dev = prompt.device
        e = lambda *s, dt=torch.bfloat16: torch.empty(*s, device=dev, dtype=dt)  # noqa: E731
        keep = saved is not None
        p_bf = ops.cast_bf16(prompt.contiguous().float(), e(B, Np, self.dim_prompt))
        kv_lens = None
        if prompt_lens is not None:   # padded rows are never attended to, but their keys must be finite
            ops.mask_rows(p_bf, prompt_lens)
            kv_lens = prompt_lens + M
        proj = p_bf
        if "pr_proj_w" in P:
            proj = ops.gemm(p_bf, P["pr_proj_w"], e(B, Np, D), n=D, epilogue=ops.EPI_BF16, bias=P["pr_proj_b"])
        # a copy: updated in place below, and for B = 1 `.contiguous()` would hand back the parameter's own storage
        lat = pr.latents.detach().float().unsqueeze(0).expand(B, M, D).clone(memory_format=torch.contiguous_format)
        Dp = _round_up(pr.ff_inner, 128)
        layers = []
        for i in range(len(pr.layers)):
            if keep or i == 0:   # inference reuses the first layer's buffers
                L = {"lat_bf": e(B, M, D), "cat": e(B, M + Np, D), "q": e(B, M, inner), "kv": e(B, M + Np, 2 * inner),
                     "lse": e(B, H, M, dt=torch.float32) if keep else None, "o": e(B, M, inner), "g": e(B, M, Dp)}
                L["lat_bf2"] = e(B, M, D) if keep else L["lat_bf"]
                L["cat"][:, M:].copy_(proj)   # [latents ; projected prompt]
                layers.append(L)
            ops.cast_bf16(lat, L["lat_bf"])
            L["cat"][:, :M].copy_(L["lat_bf"])  # cross_attn_include_queries: keys = cat(latents, context) (ns2.py:1060-1061)
            ops.gemm(L["lat_bf"], P[f"pr{i}_q"], L["q"], n=inner, epilogue=ops.EPI_BF16)
            ops.gemm(L["cat"], P[f"pr{i}_kv"], L["kv"], n=2 * inner, epilogue=ops.EPI_BF16)
            ops.attention(L["q"], L["kv"][:, :, :inner], L["kv"][:, :, inner:], L["o"], heads=H, lse=L["lse"],
                          kv_lens=kv_lens)
            ops.gemm(L["o"], P[f"pr{i}_o"], lat, n=D, epilogue=ops.EPI_F32, resid=lat)
            ops.cast_bf16(lat, L["lat_bf2"])
            ops.gemm(L["lat_bf2"], P[f"pr{i}_ff_w1"], L["g"], n=2 * Dp, epilogue=ops.EPI_GEGLU, bias=P[f"pr{i}_ff_b1"])
            ops.gemm(L["g"], P[f"pr{i}_ff_w2"], lat, n=D, epilogue=ops.EPI_F32, bias=P[f"pr{i}_ff_b2"], resid=lat)
        if keep:
            saved.update(pr_layers=layers, pr_lat=lat, pr_p_bf=p_bf, pr_Np=Np)
        out = e(B, M, D, dt=torch.float32)
        ops.rmsnorm_f32(lat, out, pr.norm.gamma.detach().float().contiguous())
        return out

    def precompute_conditioning(self, prompt: torch.Tensor, cond: torch.Tensor, length: int,
                                saved: Optional[dict] = None, *, prompt_lens=None, cond_lens=None) -> dict:
        """Everything in `forward` that depends on (prompt, cond) but not on the timestep or x:
        prompt FiLM vector, perceiver latents, projected aligned condition (ns2.py:947-992).  `saved`: see
        `_forward_impl`.
        prompt_lens (B,): sample b's prompt is prompt[b, :prompt_lens[b]] (the mean, the perceiver's keys); cond_lens (B,):
        its condition ends at frame cond_lens[b] (kept in the result as "cond_lens" for `forward`).  With them each
        sample's conditioning is that of the sample alone, and nothing in the padded rows is read.  With `saved` (the
        training forward) prompt_lens is recorded for the backward; cond_lens is for sampling only."""
        assert self.condition_on_prompt
        P, D = self.packed(), self.dim
        B = prompt.shape[0]
        dev = prompt.device
        if saved is not None and cond_lens is not None:
            raise NotImplementedError("cond_lens is supported for sampling only")
        plens = None if prompt_lens is None else ops.lengths(prompt_lens, B, prompt.shape[1], device=dev,
                                                             name="prompt_lens")
        prompt = prompt.float().contiguous()
        mean = ops.mean_rows(prompt, torch.empty(B, self.dim_prompt, device=dev), lens=plens)
        lin = self.to_prompt_cond[1]
        prompt_cond = ops.small_linear(mean, lin.weight.detach().float().contiguous(),
                                       lin.bias.detach().float().contiguous(),
                                       torch.empty(B, self.dim_time, device=dev), act=1)
        tokens = self._perceiver(prompt, P, saved, plens)
        L = cond.shape[-1]
        cond_bf = ops.transpose_cast(cond.float().contiguous(), torch.empty(B, L, self.dim_prompt, device=dev,
                                                                            dtype=torch.bfloat16))
        cond_proj = ops.gemm(cond_bf, P["cond_w"], torch.empty(B, L, D, device=dev), n=D, epilogue=ops.EPI_F32,
                             bias=P["cond_b"])
        if saved is not None:
            saved.update(prompt_mean=mean, cond_bf=cond_bf, Lc=L, prompt_lens=plens)
        c = Conditioning(prompt_cond=prompt_cond, tokens=tokens, cond_proj=cond_proj, length=length)
        if cond_lens is not None:
            c["cond_lens"] = ops.lengths(cond_lens, B, None, device=dev, name="cond_lens", lo=0)
        return c

    def _run(self, name, fn, *args, **kwargs):
        """Call one kernel wrapper; when profiling is on, bracket it with CUDA events on the current stream."""
        if self._prof is None:
            return fn(*args, **kwargs)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn(*args, **kwargs)
        b.record()
        self._prof.append((name, a, b))
        return out

    # ----------------------------------------------------------------------------------------------
    # forward
    # ----------------------------------------------------------------------------------------------
    def forward_with_cond_scale(self, *args, cond_scale=1., **kwargs):
        """ns2.py:914-927: one forward, or conditional + null forwards combined when cond_scale != 1."""
        logits = self.forward(*args, cond_drop_prob=0., **kwargs)
        if cond_scale == 1.:
            return logits
        null_logits = self.forward(*args, cond_drop_prob=1., **kwargs)
        return ops.cfg_combine(logits, null_logits, cond_scale, logits)   # in place into the (fresh) first output

    def forward(self, x, times, prompt=None, prompt_mask=None, cond=None, cond_drop_prob=None, *,
                out: Optional[torch.Tensor] = None, _conditioning: Optional[dict] = None, prompt_lens=None,
                cond_lens=None, lengths=None):
        """x (B, N, dim) fp32, times (B,) in [0, 1] -> (B, N, dim) fp32   (ns2.py:929-1000).

        Returns a fresh tensor, like the reference; pass `out=` (contiguous fp32 (B, N, dim)) to have the prediction
        written into a buffer the caller owns instead.  In train mode (`model.train()`, the nn.Module default) with
        gradients enabled the call records one autograd node whose backward runs the hand-written backward kernels
        (`training.py`); after `model.eval()` or under `torch.no_grad()` it is the inference path and nothing is saved.

        With `use_cuda_graphs` the whole step (every kernel launch below) is captured once per
        (B, N, drop-prob, conditioning shapes) and replayed; eligible when no RNG draw and no per-call host work is
        involved, i.e. unconditional models or cached conditioning with cond_drop_prob in {0, 1}.

        prompt_lens / cond_lens (B,): per-sample prompt lengths and condition lengths of a batch padded at the end, see
        `precompute_conditioning`; cached conditioning carries its own.  Training takes prompt_lens (each sample's
        prediction and gradients are those of the sample alone, d prompt is zero past its length); cond_lens is for
        inference only: in training the condition spans the latents' frames, zero past each sample's durations.

        lengths (B,): per-sample latent lengths of a batch padded at the end, in [1, N], at most 64 samples.  Sample b's
        prediction rows [0, lengths[b]) are then bit-identical to the call on x[b:b+1, :lengths[b]] alone, rows past it
        are exact zeros, and nothing in x's (or the condition's) padded rows is read.  In inference the GEMMs, the
        attention and the norms skip the 128-row tiles that lie wholly in a sample's padding.  In training every row is
        computed (the backward reads every saved activation) with the self-attention's keys limited to each sample's
        length; the gradient rows past a length are exact zeros and add nothing to any parameter gradient, so
        each sample's gradients are those of the sample alone."""
        lens = None
        if lengths is not None:
            lens = self._latent_lens(lengths, x)
        ragged = prompt_lens is not None or cond_lens is not None
        if ragged and _conditioning is not None:
            raise ValueError("prompt_lens / cond_lens go to precompute_conditioning when the conditioning is cached")
        if ragged and not self.condition_on_prompt:
            raise ValueError("prompt_lens / cond_lens apply to models with condition_on_prompt=True")
        if _records_graph(self):
            # training: one autograd node whose backward runs the hand-written kernels (training.py)
            from .training import DenoiserFunction
            if prompt_mask is not None or out is not None or _conditioning is not None or cond_lens is not None:
                raise NotImplementedError("training mode takes (x, times[, prompt, cond, prompt_lens]): no out=, "
                                          "prompt_mask, cond_lens or cached conditioning")
            return DenoiserFunction.apply(self, x, times, prompt, cond, cond_drop_prob, prompt_lens, lens,
                                          *self.parameters())
        if ragged:
            with torch.no_grad():   # eager: the prompt work is per call anyway
                return self._forward_impl(x, times, prompt, prompt_mask, cond, cond_drop_prob, None, out,
                                          prompt_lens=prompt_lens, cond_lens=cond_lens, lengths=lens)
        with torch.no_grad():
            return self._forward_nograd(x, times, prompt, prompt_mask, cond, cond_drop_prob, out, _conditioning, lens)

    def _latent_lens(self, lengths, x: torch.Tensor) -> torch.Tensor:
        """`lengths` as the validated int32 CUDA (B,) tensor the kernels read.  A tensor that already is one is used as
        it is (its range is read once per tensor version), so a sampling loop passes the same lengths every step
        without a host round trip."""
        B, N = x.shape[0], x.shape[1]
        if B > ops._lib.NS2_GEMM_ROW_LENS_MAX_BATCHES:
            raise ValueError(f"lengths: at most {ops._lib.NS2_GEMM_ROW_LENS_MAX_BATCHES} samples per call, got {B}")
        if (isinstance(lengths, torch.Tensor) and lengths.dtype == torch.int32 and lengths.is_cuda
                and lengths.is_contiguous() and tuple(lengths.shape) == (B,) and lengths.device == x.device):
            ops._check_lens(lengths, 1, N, "lengths")
            return lengths
        return ops.lengths(lengths, B, N, device=x.device, name="lengths")

    def _forward_nograd(self, x, times, prompt, prompt_mask, cond, cond_drop_prob, out, _conditioning, lens=None):
        if out is not None:
            if not (out.is_cuda and out.dtype == torch.float32 and out.is_contiguous()
                    and tuple(out.shape) == tuple(x.shape)):
                raise ValueError("out must be a contiguous CUDA float32 tensor with x's shape")
        p_eff = self.cond_drop_prob if cond_drop_prob is None else cond_drop_prob
        if (self.use_cuda_graphs and self._prof is None and prompt_mask is None and x.is_cuda
                and not torch.cuda.is_current_stream_capturing()
                and (not self.condition_on_prompt or (_conditioning is not None and p_eff in (0, 0., 1, 1.)))):
            return self._forward_graphed(x, times, p_eff, _conditioning, out, lens)
        return self._forward_impl(x, times, prompt, prompt_mask, cond, cond_drop_prob, _conditioning, out, lengths=lens)

    def _forward_graphed(self, x, times, p_eff, conditioning, out, lens=None):
        B, N, _ = x.shape
        dev = x.device
        cond_sig = None
        if conditioning is not None:
            cond_sig = tuple(tuple(conditioning[k].shape) for k in ("prompt_cond", "tokens", "cond_proj"))
            cond_sig += (conditioning.get("cond_lens") is not None,)   # a different cond_inject launch

        def build(cond):
            xs = torch.empty(B, N, self.dim, device=dev, dtype=torch.float32)
            ts = torch.empty(B, device=dev, dtype=torch.float32)
            static_out = torch.empty(B, N, self.dim, device=dev, dtype=torch.float32)
            static_lens = None if lens is None else lens.clone()
            xs.copy_(x)
            ts.copy_(times)
            step = lambda: self._forward_impl(xs, ts, cond_drop_prob=p_eff, _conditioning=cond,  # noqa: E731
                                              out=static_out, lengths=static_lens)
            return {"xs": xs, "ts": ts, "out": static_out, "lens": static_lens}, step

        # lengths live in a static device buffer: one graph serves every set of lengths of a shape
        key = (B, N, float(p_eff), cond_sig, lens is not None, str(dev))
        entry = self._captured(key, self._ws_key(B, N, dev), conditioning, build)
        entry["xs"].copy_(x)
        entry["ts"].copy_(times)
        if lens is not None:
            entry["lens"].copy_(lens)
        entry["graph"].replay()
        if out is None:
            return entry["out"].clone()
        out.copy_(entry["out"])
        return out

    @torch.no_grad()
    def _forward_impl(self, x, times, prompt=None, prompt_mask=None, cond=None, cond_drop_prob=None,
                      _conditioning: Optional[dict] = None, out: Optional[torch.Tensor] = None,
                      saved: Optional[dict] = None, prompt_lens=None, cond_lens=None, lengths=None):
        """The denoiser's forward.  Without `saved` every intermediate lives in the per-shape workspace, so the call can
        be captured in a CUDA graph.  With `saved` (a dict; the training forward of `training.DenoiserFunction`) the
        workspace is not touched: each activation `training.train_backward` reads goes to a fresh tensor recorded
        there, together with the residual stream before each branch and the attention log-sum-exps.

        lengths: validated int32 CUDA (B,) latent lengths (see `forward`).  The input rows past them (x and condition)
        are zeroed on entry, the self-attention takes them as key lengths, and the prediction's padded rows are zeroed
        at the end.  Without `saved`, every GEMM over latent rows and every norm also skips the 128-row tiles (norm:
        rows) wholly past a sample's length, and both attentions take them as query lengths.  With `saved` every row is
        computed, so every saved activation is finite.  The workspace rows of the
        skipped tiles keep whatever an earlier call left there.  No valid row reads them: the causal convs read only
        earlier rows, the other GEMMs and the norms are per row, and the self-attention never loads a key tile past a
        sample's length.  Rows past a length inside a computed tile are computed from the zeroed input and rows of the
        same computed tiles (the norm's skipped rows keep this call's skip-conv output), so the keys the attention
        masks there are finite."""
        if prompt_mask is not None:
            raise NotImplementedError("prompt_mask is unsupported (the reference itself fails on it, SURVEY T9)")
        if not x.is_cuda:
            raise RuntimeError("naturalspeech2_pytorch_b200.Model runs on CUDA (sm_90a) tensors only")
        B, N, D = x.shape
        assert D == self.dim, f"expected last dim {self.dim}, got {D}"
        dev = x.device
        P = self.packed()
        G, inner, H = self.wavenet_layers, self.inner, self.heads
        Dp = _round_up(self.ff_inner, 128)
        keep = saved is not None
        lens = None if keep else lengths   # tile skipping: inference only
        if keep:
            buf = lambda name, *s, dt=torch.bfloat16: torch.empty(*s, device=dev, dtype=dt)  # noqa: E731
        else:
            ws = self._workspace(B, N, dev)
            buf = lambda name, *s, dt=None: ws[name]  # noqa: E731
        cond_drop_prob = self.cond_drop_prob if cond_drop_prob is None else cond_drop_prob

        # ---- time / prompt conditioning vector t: (B, dim_cond) ----
        times = times.float().contiguous()
        t = buf("t", B, self.dim_cond, dt=torch.float32)
        tc = self.to_time_cond
        self._run("time_cond", ops.time_cond, times, tc[0].weights.detach().float().contiguous(),
                      tc[1].weight.detach().float().contiguous(), tc[1].bias.detach().float().contiguous(),
                      t[:, :self.dim_time])
        c_tokens = None
        cond_drop_mask = None
        if self.condition_on_prompt:
            if _conditioning is None:
                assert _exists(prompt), "prompt is required when condition_on_prompt=True"
                assert _exists(cond), "cond is required when condition_on_prompt=True"
                _conditioning = self.precompute_conditioning(prompt, cond, N, saved, prompt_lens=prompt_lens,
                                                             cond_lens=cond_lens)
            # two independent draws, in the reference's order (ns2.py:950, 980): kept in torch for RNG-stream parity
            drop_mask = _prob_mask_like((B,), cond_drop_prob, dev)
            cond_drop_mask = _prob_mask_like((B,), cond_drop_prob, dev)
            ops.select_rows(drop_mask, self.null_prompt_cond.detach().float().contiguous(),
                            _conditioning["prompt_cond"], t[:, self.dim_time:])
            c_tokens = ops.select_rows(drop_mask, self.null_prompt_tokens.detach().float().contiguous(),
                                       _conditioning["tokens"], buf("c_bf", B, self.num_latents_m, D))
            if keep:
                saved.update(drop=drop_mask, cdrop=cond_drop_mask, c_bf=c_tokens)

        # ---- all FiLM (gamma, beta) vectors in one GEMM ----
        rows = P["film_w"].shape[0]
        t_bf = self._run("cast", ops.cast_bf16, t, buf("t_bf", 1, B, self.dim_cond))
        film = self._run("film", ops.gemm, t_bf, P["film_w"], buf("film", 1, B, rows, dt=torch.float32), n=rows,
                         epilogue=ops.EPI_F32, bias=P["film_b"])[0]  # (B, rows)

        # ---- wavenet ----
        if self.condition_on_prompt:
            # x + pad_or_curtail(where(cond_drop_mask, null_cond, cond_proj)) -> bf16 in one pass (ns2.py:982-992)
            x_bf = self._run("cast", ops.cond_inject, x.float().contiguous(), _conditioning["cond_proj"],
                             buf("x_bf", B, N, D), drop_mask=cond_drop_mask,
                             null_cond=self.null_cond.detach().float().reshape(-1),
                             cond_lens=_conditioning.get("cond_lens"))
        else:
            x_bf = self._run("cast", ops.cast_bf16, x.float().contiguous(), buf("x_bf", B, N, D))
        if lengths is not None:   # the padded rows of x + condition: zeros, whatever the caller's padding holds
            self._run("mask", ops.mask_rows, x_bf, lengths)
        h0 = self._run("wn_init", ops.gemm, x_bf, P["wn_init_w"], buf("h", B, N, D), n=D, epilogue=ops.EPI_BF16,
                       bias=P["wn_init_b"], segs=ops.conv3_segs(D), row_lens=lens)
        segs = ops.conv3_segs(D) + [(0, 3 * D, D, 0, 1)]
        dil = [2 ** i for i in range(G)]
        src, stack_out = h0, []
        for s in range(self.wavenet_stacks):
            dst = buf(("wn_a", "wn_b")[s % 2], B, N, G * D)
            self._run("wn_stack", ops.gemm, src, P[f"wn{s}_w"], dst, n=D, epilogue=ops.EPI_WAVENET, bias=P[f"wn{s}_b"],
                     bias1_off=G * D, segs=segs, film=film[:, s * G * 2 * D:], film_group_stride=2 * D,
                     groups=G, a_group_col_stride=0 if s == 0 else D, b_group_row_stride=D,
                     out_group_col_stride=D, dil=dil, row_lens=lens)
            stack_out.append(dst)
            src = dst
        skip = self._run("wn_skip", ops.gemm, src, P["wn_skip_w"], buf("h", B, N, D), n=D, epilogue=ops.EPI_BF16,
                         bias=P["wn_skip_b"], row_lens=lens)
        xr = self._run("wn_final", ops.gemm, skip, P["wn_final_w"], buf("x_res", B, N, D, dt=torch.float32), n=D,
                       epilogue=ops.EPI_F32, bias=P["wn_final_b"], row_lens=lens)
        if keep:
            saved.update(B=B, N=N, times=times, t=t, film=film, x_bf=x_bf, h0=h0, stack_out=stack_out, skip=skip)

        # ---- transformer ----
        lse = lambda: torch.empty(B, H, N, device=dev, dtype=torch.float32) if keep else None  # noqa: E731
        if c_tokens is not None:
            xkv = self._run("x_kv", ops.gemm, c_tokens, P["x_kv_all"], buf("xkv", B, self.num_latents_m, self.depth * 2 * inner),
                            n=self.depth * 2 * inner, epilogue=ops.EPI_BF16)
            if keep:
                saved["xkv"] = xkv
        npl = self._norms_per_layer
        layers = []
        for l in range(self.depth):
            fo = self._film_tr_off + l * npl * 2 * D
            L = {"x_in": xr.clone()} if keep else {}
            L["h1"] = self._run("norm", ops.rmsnorm_film, xr, buf("h", B, N, D), film=film[:, fo:fo + 2 * D], lens=lens)
            qkv = L["qkv"] = self._run("qkv", ops.gemm, L["h1"], P[f"l{l}_qkv"], buf("qkv", B, N, 3 * inner),
                                       n=3 * inner, epilogue=ops.EPI_BF16, row_lens=lens)
            L["lse"] = lse()
            L["ao"] = self._run("attn", ops.attention, qkv[:, :, :inner], qkv[:, :, inner:2 * inner],
                                qkv[:, :, 2 * inner:], buf("attn_o", B, N, inner), heads=H, lse=L["lse"],
                                kv_lens=lengths, q_lens=lens)
            self._run("attn_out", ops.gemm, L["ao"], P[f"l{l}_o"], xr, n=D, epilogue=ops.EPI_F32, resid=xr,
                      row_lens=lens)
            if c_tokens is not None:   # cross attention over the perceiver latents (ns2.py:800-803)
                fo2 = fo + 2 * D
                if keep:
                    L["x_c"] = xr.clone()
                L["h_x"] = self._run("norm", ops.rmsnorm_film, xr, buf("h", B, N, D), film=film[:, fo2:fo2 + 2 * D],
                                     lens=lens)
                L["xq"] = self._run("x_q", ops.gemm, L["h_x"], P[f"l{l}_xq"], buf("xq", B, N, inner), n=inner,
                                    epilogue=ops.EPI_BF16, row_lens=lens)
                kv = xkv[:, :, l * 2 * inner:(l + 1) * 2 * inner]
                L["lse2"] = lse()
                L["ao2"] = self._run("x_attn", ops.attention, L["xq"], kv[:, :, :inner], kv[:, :, inner:],
                                     buf("attn_o", B, N, inner), heads=H, lse=L["lse2"], q_lens=lens)
                self._run("x_out", ops.gemm, L["ao2"], P[f"l{l}_xo"], xr, n=D, epilogue=ops.EPI_F32, resid=xr,
                          row_lens=lens)
            if keep:
                L["x_mid"] = xr.clone()
            fo3 = fo + (npl - 1) * 2 * D
            L["h2"] = self._run("norm", ops.rmsnorm_film, xr, buf("h", B, N, D), film=film[:, fo3:fo3 + 2 * D],
                                lens=lens)
            L["ff_g"] = self._run("ff_in", ops.gemm, L["h2"], P[f"l{l}_ff_w1"], buf("ff_g", B, N, Dp), n=2 * Dp,
                                  epilogue=ops.EPI_GEGLU, bias=P[f"l{l}_ff_b1"], row_lens=lens)
            # causal conv with the output projection folded in: x += W' * g + b' straight from the GEGLU output
            self._run("ff_conv", ops.gemm, L["ff_g"], P[f"l{l}_ff_wo"], xr, n=D, epilogue=ops.EPI_F32,
                      bias=P[f"l{l}_ff_bo"], resid=xr, segs=ops.conv3_segs(Dp), row_lens=lens)
            layers.append(L)
        hf = self._run("norm", ops.rmsnorm_film, xr, buf("h", B, N, D), gamma=P["pred_gamma"], lens=lens)
        if keep:
            saved.update(layers=layers, x_final=xr, hf=hf, lens=lengths)
        if out is None:
            out = torch.empty(B, N, D, device=dev, dtype=torch.float32)   # fresh tensor, like the reference
        self._run("pred", ops.gemm, hf, P["pred_w"], out, n=D, epilogue=ops.EPI_F32, row_lens=lens)
        if lengths is not None:
            self._run("mask", ops.mask_rows, out, lengths)
        return out
