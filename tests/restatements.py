"""Float64 compositions and fixtures that more than one GPU suite reads: the restatements of the encoders, the
Conditioner, the predictor (with and without its dropout masks), the denoiser port and the whole training objective,
the configuration tables the float64 suites sweep, and the small training fixtures.  Everything here is built from the
pinned restatements only (`oracle.*`, tests/dropout_oracle.py, tests/rvq_ce_restatement.py); nothing touches CUDA at
import time, so CPU tests read it too."""
import numpy as np
import torch
import torch.nn.functional as F
from torch import nn

import dropout_oracle as do
from fp64_check import autograd, round_params
from helpers import GOLDEN, oracle_config
from oracle import denoiser_torch_port as tp
from oracle import diffusion_oracle as dfo
from oracle import encoders_oracle as eo
from param_fill import fill_module
from rvq_ce_restatement import residual_vq_ce

SEED_HIGH = 2 ** 63 - 1
# test_ragged_training_gpu.py: the batch against the alone calls where every attention fits one key tile
RTOL = 2.0 ** -19


def drawn_seed(torch_seed):
    """The dropout seed a module draws right after torch.manual_seed(torch_seed)."""
    torch.manual_seed(torch_seed)
    return int(torch.randint(0, SEED_HIGH, ()))


# ---- the conditioning encoders at their default dims ----
DIM, HEADS, DEPTH, DROP_P = 512, 8, 6, 0.2         # the encoders' default transformer and dropout


def encoder_masks(cls, seed, B, N):
    """(attention masks per layer, conv mask) as keep * scale fp64 tensors of the drawn seed (None: no dropout)."""
    if seed is None:
        return None, None
    if cls == "SpeechPromptEncoder":       # `dropout` goes to every attention; there is no conv dropout
        return [do.mask_tensor(do.attention_mask(seed, 1 + l, DROP_P, B, HEADS, N, N), DROP_P).cuda()
                for l in range(DEPTH)], None
    # PhonemeEncoder: conv_dropout 0.2 on the causal conv's SiLU output (site 0), attn_dropout 0
    return None, do.mask_tensor(do.elementwise_mask(seed, 0, DROP_P, B * N * DIM).reshape(B, N, DIM), DROP_P).cuda()


def encoder_fwd(cls, x, masks, phoneme_encoder=None):
    """The restatement of one encoder: P (a state_dict of `dtype` tensors) -> {"out": (B, N, 512)}."""
    attn, conv = masks

    def fwd(P, dtype):
        if cls == "SpeechPromptEncoder":
            if attn is None:
                return {"out": eo.speech_prompt_encoder(P, x.to(dtype))}
            return {"out": do.speech_prompt_encoder(P, x.to(dtype), attn_masks=[m.to(dtype) for m in attn])}
        if phoneme_encoder is not None:
            return {"out": phoneme_encoder(P, x)}
        if conv is None:
            return {"out": eo.phoneme_encoder(P, x)}
        return {"out": do.phoneme_encoder(P, x, conv_mask=conv.to(dtype))}
    return fwd


def conditioner_fwd(prompt, text, mask, onehot):
    """Conditioner(mode="train") restated: prompt_enc and cond = length-regulated phoneme encodings + coarse-pitch
    embeddings (ns2.py:1449-1455) with the host-built alignment `mask` (B, T, L) and pitch one-hot (B, T, bins)."""
    def fwd(P, dtype):
        sub = lambda pfx: {k[len(pfx):]: v for k, v in P.items() if k.startswith(pfx)}  # noqa: E731
        pe = eo.speech_prompt_encoder(sub("prompt_enc."), prompt.to(dtype))
        ph = eo.phoneme_encoder(sub("phoneme_enc."), text)
        m = mask.to(dtype)
        pitch = onehot.to(dtype) @ P["pitch_emb.weight"]
        cond = torch.einsum("btl,bdt->bdl", m, ph.transpose(1, 2)) + torch.einsum("btl,bdt->bdl", m, pitch.transpose(1, 2))
        return {"out prompt_enc": pe, "out cond": cond}
    return fwd


# ---- the duration / pitch predictor ----
TRUNKS = ("to_duration_pred.", "to_pitch_pred.")
DPP_DIM, DPP_HEADS, DPP_DEPTH = 512, 8, 10          # the predictor's default dims


def predictor_fwd(x, prompts, table, groups=8, trunk=None, heads=DPP_HEADS):
    """fwd(P, dtype) = {"duration": ..., "pitch": ...} of the restatement; the leaves P["x"] / P["prompts"], where
    present, stand for `x` / `prompts`.  `x` are ids when `table`."""
    trunk = trunk or eo._trunk

    def fwd(P, dtype):
        xs, ps = P.get("x", x), P.get("prompts", prompts)
        h = P["phoneme_token_emb.weight"][xs] if table else xs.to(dtype)
        sub = lambda pfx: {k: v for k, v in P.items() if k.startswith(pfx)}  # noqa: E731
        return {"duration": trunk(sub(TRUNKS[0]), TRUNKS[0], h, ps.to(dtype), heads, groups=groups),
                "pitch": trunk(sub(TRUNKS[1]), TRUNKS[1], h, ps.to(dtype), heads, groups=groups)}
    return fwd


def set_head_biases(m, x, prompts, table, heads=DPP_HEADS):
    """Head biases (bf16 values) that keep every fp64 pre-activation away from 0; returns them per trunk."""
    P = {n: p.detach().double() for n, p in m.named_parameters()}
    for t in TRUNKS:
        P[t + "to_pred.0.bias"] = torch.full_like(P[t + "to_pred.0.bias"], 1e3)
    with torch.backends.cudnn.flags(enabled=False):
        outs = predictor_fwd(x, prompts, table, heads=heads)(P, torch.float64)
    biases = {}
    for t, key in zip(TRUNKS, ("duration", "pitch")):
        pre = (outs[key] - 1e3).flatten().sort().values           # pre-activations without the bias
        spread = float(pre[-1] - pre[0]) + 1e-3
        lo, hi = int(0.2 * pre.numel()), int(0.8 * pre.numel())
        gaps = pre[lo + 1:hi + 1] - pre[lo:hi] if hi > lo else pre[:0]
        if gaps.numel() and float(gaps.max()) > 0.2 * spread:     # room for dead and live rows on both sides
            i = lo + int(gaps.argmax())
            b = -0.5 * float(pre[i] + pre[i + 1])
        else:                                                       # every row alive
            b = 0.25 * spread - float(pre[0])
        biases[t] = torch.tensor(b).bfloat16().float().item()
        with torch.no_grad():
            m.get_submodule(t[:-1]).to_pred[0].bias.fill_(biases[t])
    m.invalidate_packed()
    return biases


def site(t, l):
    """Dropout site of the cross attention of layer l of trunk t (0 duration, 1 pitch)."""
    return t * DPP_DEPTH + l


def masks_for(seed, p, B, T, Np, site_of=site, block_sites=None):
    """{trunk: (block masks [l][j] (B, T, D) or None, attention masks [l] (B, H, T, T + Np))}, keep * scale in fp64 on
    the GPU.  block_sites(t, l, j): sites for masks after every Block's SiLU (only a wrong reference has them)."""
    out = {}
    for t, pre in enumerate(TRUNKS):
        blocks = None if block_sites is None else [
            [do.mask_tensor(do.elementwise_mask(seed, block_sites(t, l, j), p, B * T * DPP_DIM).reshape(B, T, DPP_DIM),
                            p).cuda() for j in range(6)] for l in range(DPP_DEPTH)]
        attn = [do.mask_tensor(do.attention_mask(seed, site_of(t, l), p, B, DPP_HEADS, T, T + Np), p).cuda()
                for l in range(DPP_DEPTH)]
        out[pre] = (blocks, attn)
    return out


def masked_trunk(P, pre, x, prompts, heads, block_masks=None, attn_masks=None, groups=8, eps=1e-5):
    """eo._trunk with the attention mask after the softmax (attend.py:149) and, for a wrong reference only, Block j's
    mask after its SiLU; masks None = no dropout."""
    for l in range(DPP_DEPTH):
        lp = f"{pre}layers.{l}."
        j = 0
        for r in range(3):
            h = x.transpose(1, 2)
            for c in range(2):
                bp = f"{lp}0.{r}.blocks.{c}."
                w = P[bp + "proj.weight"]
                h = F.conv1d(h, w, P[bp + "proj.bias"], padding=w.shape[-1] // 2)
                h = F.silu(F.group_norm(h, groups, P[bp + "norm.weight"], P[bp + "norm.bias"], eps))
                if block_masks is not None:
                    h = h * block_masks[l][j].transpose(1, 2).to(h.dtype)
                j += 1
            x = h.transpose(1, 2) + x
        nx = eo._rmsnorm(x, P[lp + "1.gamma"])
        ctx = torch.cat((nx, prompts), dim=-2)
        q = nx @ P[lp + "2.to_q.weight"].T
        k, v = (ctx @ P[lp + "2.to_kv.weight"].T).chunk(2, dim=-1)
        b, n, _ = q.shape
        q, k, v = (t.view(b, t.shape[1], heads, -1).transpose(1, 2) for t in (q, k, v))
        attn = (torch.einsum("bhid,bhjd->bhij", q, k) * (q.shape[-1] ** -0.5)).softmax(dim=-1)
        if attn_masks is not None:
            attn = attn * attn_masks[l].to(attn.dtype)
        o = torch.einsum("bhij,bhjd->bhid", attn, v).transpose(1, 2).reshape(b, n, -1)
        x = o @ P[lp + "2.to_out.weight"].T + x
    return F.relu(x @ P[pre + "to_pred.0.weight"].T + P[pre + "to_pred.0.bias"]).squeeze(-1)


def masked_predictor_fp64(params, x, prompts, d_outs, masks=None, only=None):
    """fp64 autograd of the (masked) restatement -> {name: gradient} plus "out duration" / "out pitch"; with
    d_outs=None the outputs alone."""
    P = {n: p.detach().double().requires_grad_(True) for n, p in params.items()}
    leaves = dict(P, x=x.detach().double().requires_grad_(True), prompts=prompts.detach().double().requires_grad_(True))
    outs = {}
    with torch.backends.cudnn.flags(enabled=False):
        for pre, key in zip(TRUNKS, ("duration", "pitch")):
            sub = {k: v for k, v in P.items() if k.startswith(pre)}
            bm, am = masks[pre] if masks is not None else (None, None)
            outs[key] = masked_trunk(sub, pre, leaves["x"], leaves["prompts"], DPP_HEADS, bm, am)
        if d_outs is None:
            return {k: o.detach() for k, o in outs.items()}
        names = list(leaves) if only is None else list(only)
        g = torch.autograd.grad([outs["duration"], outs["pitch"]], [leaves[n] for n in names],
                                [d_outs["duration"].double(), d_outs["pitch"].double()], allow_unused=True)
    res = {n: torch.zeros_like(leaves[n]) if gi is None else gi.detach() for n, gi in zip(names, g)}
    res.update({"out " + k: o.detach() for k, o in outs.items()})
    return res


def set_head_biases_masked(m, params, x, prompts, masks):
    """bf16 head biases that keep every fp64 pre-activation, with and without the masks, well above 0."""
    P = dict(params)
    for pre in TRUNKS:
        P[pre + "to_pred.0.bias"] = torch.full_like(P[pre + "to_pred.0.bias"], 1e3)
    outs = [masked_predictor_fp64(P, x, prompts, None, mk) for mk in (None, masks)]
    for pre, key in zip(TRUNKS, ("duration", "pitch")):
        pres = torch.cat([(o[key] - 1e3).flatten() for o in outs])   # pre-activations without the bias
        b = 0.25 * float(pres.max() - pres.min()) + 1e-3 - float(pres.min())
        with torch.no_grad():
            m.get_submodule(pre[:-1]).to_pred[0].bias.fill_(torch.tensor(b).bfloat16().float().item())
    m.invalidate_packed()


# ---- the encoder configurations the float64 suites sweep ----
SPE, PHON, DPP = "SpeechPromptEncoder", "PhonemeEncoder", "DurationPitchPredictor"
ENCODER_CONFIGS = {
    # name: (class, constructor kwargs, ragged lengths, ragged prompt lengths (predictor))
    "spe_k3_narrow": (SPE, dict(dim_codebook=64, dims=(64, 192, 128), kernel_size=3, padding=1, depth=2, heads=3),
                      (1, 129, 50), None),
    "spe_k1_wide": (SPE, dict(dim_codebook=128, dims=(1024,), kernel_size=1, padding=0, depth=1, heads=16),
                    (1, 300), None),
    "spe_k11": (SPE, dict(dim_codebook=128, dims=(256, 384), kernel_size=11, padding=5, depth=1, heads=4),
                (1, 103), None),
    "phon_d64": (PHON, dict(num_tokens=30, dim=64, dim_hidden=384, kernel_size=3, depth=2, heads=5), (1, 37, 20), None),
    "phon_k12": (PHON, dict(num_tokens=30, dim=256, dim_hidden=256, kernel_size=12, depth=1, heads=2), (1, 100), None),
    "phon_k1": (PHON, dict(num_tokens=30, dim=512, dim_hidden=1024, kernel_size=1, depth=1, heads=8), (1, 64), None),
    "dpp_128": (DPP, dict(dim=128, dim_hidden=128, kernel_size=5, depth=2, heads=2, num_convs_per_resnet_block=1,
                          num_convolutions_per_block=2), (1, 40, 17), (7, 1, 4)),
    "dpp_384": (DPP, dict(dim=384, dim_hidden=384, kernel_size=7, depth=1, heads=3, num_convs_per_resnet_block=3,
                          num_convolutions_per_block=1), (1, 65), (129, 1)),
    "dpp_640": (DPP, dict(dim=640, dim_hidden=640, kernel_size=1, depth=1, heads=10), (33, 1), (1, 64)),
    "dpp_1024": (DPP, dict(dim=1024, dim_hidden=1024, kernel_size=3, depth=1, heads=16), (1, 100), (103, 1)),
    "dpp_table": (DPP, dict(num_phoneme_tokens=60, dim=256, dim_hidden=256, kernel_size=3, depth=2), (1, 50), (40, 1)),
}


def config_heads(cfg):
    return ENCODER_CONFIGS[cfg][1].get("heads", 8)


def build_config(cfg):
    """The module of one configuration, filled and rounded to bf16, on the GPU."""
    from naturalspeech2_pytorch_b200 import encoders
    cls, kw, _, _ = ENCODER_CONFIGS[cfg]
    m = getattr(encoders, cls)(**kw)
    fill_module(m, 1234)
    m.cuda()
    round_params(m)
    return m


def config_fwd(cfg, x, prompts=None, **kw):
    """fwd(P, dtype) of the configuration's restatement; x: prompt frames (the leaf P["x"] where present), ids (-1 =
    padding) or phoneme encodings."""
    cls, ckw, _, _ = ENCODER_CONFIGS[cfg]
    heads = config_heads(cfg)
    if cls == DPP:
        return predictor_fwd(x, prompts, "num_phoneme_tokens" in ckw, heads=heads, **kw)

    def fwd(P, dtype):
        if cls == SPE:
            return {"encoding": eo.speech_prompt_encoder(P, P.get("x", x).to(dtype), heads=heads,
                                                         padding=ckw["padding"])}
        return {"encoding": eo.phoneme_encoder(P, x, heads=heads)}
    return fwd


# ---- the denoiser ----
COND = dict(condition_on_prompt=True)
DENOISER_CASES = {
    # name: (model kwargs, B, N, prompt length, cond frames, cond_drop_prob)
    "g1_h1": (dict(dim=256, depth=1, heads=1, wavenet_layers=1, wavenet_stacks=1), 3, 200, None, None, 0.),
    "g5_d3": (dict(dim=384, depth=3, heads=5, wavenet_layers=5, wavenet_stacks=3, dim_cond_mult=2), 2, 129, None, None, 0.),
    "ff2_cond": (dict(dim=128, depth=2, heads=2, ff_mult=2, wavenet_layers=3, wavenet_stacks=2, dim_prompt=192, **COND),
                 3, 160, 40, 150, .5),
    "ff8_cond": (dict(dim=128, depth=1, heads=4, ff_mult=8, dim_cond_mult=1, wavenet_layers=2, wavenet_stacks=2,
                      dim_prompt=128, **COND), 2, 97, 25, 200, 0.),
    "w640_m1": (dict(dim=640, depth=2, heads=10, wavenet_layers=7, wavenet_stacks=2, dim_cond_mult=3, dim_prompt=64,
                     num_latents_m=1, resampler_depth=1, **COND), 2, 300, 1, 300, 0.),
    "w1024_b50": (dict(dim=1024, depth=1, heads=16, wavenet_layers=8, wavenet_stacks=1, dim_prompt=1088, num_latents_m=33,
                       resampler_depth=3, **COND), 50, 37, 19, 20, 0.),
    "n1_b33": (dict(dim=128, depth=1, heads=2, wavenet_layers=8, wavenet_stacks=2), 33, 1, None, None, 0.),
}


def drop_masks(B, p):
    """(seed, prompt-drop mask, cond-drop mask) as Model.forward draws them after torch.manual_seed(seed): prompt first,
    cond second (`model._prob_mask_like`); for 0 < p < 1 the first seed where each mask drops some samples and keeps
    others."""
    if p == 0:
        zeros = torch.zeros(B, dtype=torch.bool, device="cuda")
        return None, zeros, zeros
    for seed in range(100):
        torch.manual_seed(seed)
        dp = torch.zeros((B,), device="cuda").float().uniform_(0, 1) < p
        dc = torch.zeros((B,), device="cuda").float().uniform_(0, 1) < p
        if 0 < int(dp.sum()) < B and 0 < int(dc.sum()) < B:
            return seed, dp, dc
    raise AssertionError("no seed gives mixed drop masks")


def port_grads(params, kwargs, inp, drop, d_out, autocast=False, dilations=None, only=None):
    """{name: d out-weighted gradient} of the torch port on `params` (the model's rounded fp32 values) in fp64, or in
    fp32 under bf16 autocast; names are the parameters' and "d prompt" / "d cond"."""
    def fwd(P, dtype):
        return {"out": tp.model_forward_autograd(P, oracle_config(kwargs), inp["x"].to(dtype), inp["times"].to(dtype),
                                                 P.get("d prompt"), P.get("d cond"), drop_prompt=drop[0],
                                                 drop_cond=drop[1], dilations=dilations)}
    inputs = {f"d {k}": inp[k] for k in ("prompt", "cond") if k in inp}
    return autograd(fwd, params, {"out": d_out}, autocast=autocast, inputs=inputs, only=only)


# ---- the whole training objective ----
def objective(P, dtype, c, wrong=None):
    """The scalar NaturalSpeech2.forward returns, as one graph over P ({"model." / "prompt_enc." / "phoneme_enc." /
    "pitch_emb." / "duration_pitch." + name: tensor}) -> {"loss", "duration_loss", "pitch_loss"} and the boundary
    tensors "pe" (prompt encoder output), "pe_model" (what the Model receives), "cond", "ph" (phoneme encodings).
    `c` holds the inputs and host-side glue (alignment mask, coarse-pitch one-hot, per-phoneme pitch, alpha / sigma,
    drop masks, dropout masks); `wrong` selects a deliberately wrong variant."""
    sub = lambda pfx: {k[len(pfx):]: v for k, v in P.items() if k.startswith(pfx)}  # noqa: E731
    attn, conv, pred_masks = c.get("masks", (None, None, None))
    if attn is None:
        pe = eo.speech_prompt_encoder(sub("prompt_enc."), c["prompt"].to(dtype), heads=c["heads"][0],
                                      padding=c["padding"])
    else:
        pe = do.speech_prompt_encoder(sub("prompt_enc."), c["prompt"].to(dtype), heads=c["heads"][0],
                                      padding=c["padding"], attn_masks=[m.to(dtype) for m in attn])
    if conv is None:
        ph = eo.phoneme_encoder(sub("phoneme_enc."), c["text"], heads=c["heads"][1])
    else:
        ph = do.phoneme_encoder(sub("phoneme_enc."), c["text"], heads=c["heads"][1], conv_mask=conv.to(dtype))
    if "enc_values" in c:     # the downstream graph evaluated at given encoder outputs; gradients pass unchanged
        pe = pe + (c["enc_values"][0].to(dtype) - pe).detach()
        ph = ph + (c["enc_values"][1].to(dtype) - ph).detach()
    # expand_encodings (ns2.py:1449-1455) with the alignment of the durations over L frames and the coarse pitch
    m = c["mask"].to(dtype)
    pitch = c["onehot"].to(dtype) @ P["pitch_emb.weight"]
    cond = torch.einsum("btl,bdt->bdl", m, ph.transpose(1, 2)) + torch.einsum("btl,bdt->bdl", m, pitch.transpose(1, 2))
    out = {"pe": pe, "ph": ph, "cond": cond}
    if "duration_pitch.to_duration_pred.to_pred.0.bias" in P:
        ph_in = ph.detach() if wrong == "predictor without phoneme stream" else ph
        Pd = sub("duration_pitch.")
        if wrong == "predictor on the null-substituted prompt":
            dp = c["drop"][0]
            null = P["model.null_prompt_tokens"][None].expand(int(dp.sum()), -1, -1)
            keep, drop = predict(Pd, ph_in[~dp], pe[~dp], c, None), predict(Pd, ph_in[dp], null, c, None)
            preds = [torch.empty(*ph_in.shape[:2], dtype=k.dtype, device=k.device).index_put((~dp,), k)
                     .index_put((dp,), d) for k, d in zip(keep, drop)]
        else:
            preds = predict(Pd, ph_in, pe, c, pred_masks)
        out["duration_loss"] = F.l1_loss(c["duration"].to(device=ph.device, dtype=dtype), preds[0].to(dtype))
        out["pitch_loss"] = F.l1_loss(c["ph_pitch"].to(device=ph.device, dtype=dtype), preds[1].to(dtype))
        out["duration_pred"], out["pitch_pred"] = preds
    pe_model = pe.view_as(pe)              # the Model's share of d prompt_enc
    cfg = c["cfg"]
    a, s = c["alpha"].to(dtype), c["sigma"].to(dtype)
    audio, noise = c["audio"].to(dtype), c["noise"].to(dtype)
    noised = a[:, None, None] * audio + s[:, None, None] * noise
    pred = tp.model_forward_autograd(sub("model."), oracle_config(c["model_kwargs"]), noised, c["times"].to(dtype),
                                     pe_model, cond, drop_prompt=c["drop"][0], drop_cond=c["drop"][1]).to(dtype)
    loss, _ = dfo.diffusion_loss(pred, audio, noise, a, s, cfg["objective"], cfg["min_snr_loss_weight"],
                                 cfg["min_snr_gamma"])
    if c.get("codebooks") is not None:
        x_start = pred if wrong == "ce x_start = pred" else dfo.x_start_from_pred(audio, pred, a, s, cfg["objective"])
        _, ce, _ = residual_vq_ce(x_start, c["codebooks"].to(dtype), c["codes"], own=c.get("own"))
        loss = loss + cfg["ce_weight"] * ce
    if "duration_loss" in out:
        wd, wp = cfg["weights"][::-1] if wrong == "loss weights swapped" else cfg["weights"]
        loss = loss + (wd * out["duration_loss"] + wp * out["pitch_loss"])
    out.update(loss=loss, pe_model=pe_model)
    return out


def predict(Pd, x, prompts, c, masks):
    """The predictor's two predictions inside `objective` (masked trunks with the predictor's dropout masks)."""
    heads = c["heads"][2]
    if masks is None:
        return eo.duration_pitch_predictor(Pd, x, prompts, heads=heads)
    return tuple(masked_trunk(Pd, pre, x, prompts, heads, None, [m.to(x.dtype) for m in masks[pre][1]])
                 for pre in TRUNKS)


# ---- training fixtures ----
_E2E_GOLDEN = None


def e2e_golden():
    """tests/golden/grads_cond_train.npz, loaded once."""
    global _E2E_GOLDEN
    if _E2E_GOLDEN is None:
        _E2E_GOLDEN = np.load(GOLDEN / "grads_cond_train.npz")
    return _E2E_GOLDEN


def e2e_front_end(case):
    """Our modules for one end-to-end golden case, filled like the reference's (param_fill, by state_dict key)."""
    from golden.make_golden_cond_train import COND_TRAIN_CASES
    from naturalspeech2_pytorch_b200 import Model
    from naturalspeech2_pytorch_b200.encoders import Conditioner, PhonemeEncoder, SpeechPromptEncoder
    mkw, skw, pkw, tshape, *_ = COND_TRAIN_CASES[case]
    mods = {"model": Model(**mkw), "prompt_enc": SpeechPromptEncoder(**skw), "phoneme_enc": PhonemeEncoder(**pkw),
            "pitch_emb": nn.Embedding(*tshape)}
    for m in mods.values():
        fill_module(m, seed=1234)
        m.cuda().train()
    cond_net = Conditioner.__new__(Conditioner)            # a Conditioner around these (small) sub-modules
    nn.Module.__init__(cond_net)
    cond_net.phoneme_enc, cond_net.prompt_enc, cond_net.pitch_emb = mods["phoneme_enc"], mods["prompt_enc"], mods["pitch_emb"]
    cond_net.grad_reducer = None
    return mods, cond_net


def e2e_inputs(case):
    from golden.make_golden_cond_train import cond_train_inputs
    z = e2e_golden()
    inp = cond_train_inputs(case)
    for k in ("text", "duration"):   # the seeded inputs regenerate exactly what the fixture was made from
        assert np.array_equal(inp[k].numpy(), z[f"{case}::in_{k}"]), k
    return inp


def e2e_loss(ns, inp):
    return ns(inp["latents"].cuda(), text=inp["text"].cuda(), prompt=inp["prompt"].cuda(), pitch=inp["pitch"].cuda(),
              duration=inp["duration"].cuda(), times=inp["times"], noise=inp["noise"])


DPP_TRAIN_SHAPE = (2, 24, 40, 96)     # B, text length, prompt frames, pitch frames


def dpp_train_inputs():
    """A small seeded batch for the predictor trained jointly with the conditional model."""
    B, T_TEXT, NP, L = DPP_TRAIN_SHAPE
    g = torch.Generator().manual_seed(5)
    dur = torch.randint(1, 6, (B, T_TEXT), generator=g)
    dur[:, -1] = 0
    dur[0, 3] = 0
    pitch = 100 + 200 * torch.rand(B, L, generator=g)
    pitch[:, ::5] = 0.0                                              # unvoiced frames
    return dict(latents=torch.randn(B, L, 128, generator=g).cuda(), prompt=torch.randn(B, NP, 128, generator=g).cuda(),
                text=torch.randint(0, 50, (B, T_TEXT), generator=g).cuda(), duration=dur.cuda(), pitch=pitch.cuda(),
                times=torch.rand(B, generator=g).cuda(), noise=torch.randn(B, L, 128, generator=g).cuda())


def dpp_train_loss(ns, inp):
    return ns(inp["latents"], text=inp["text"], prompt=inp["prompt"], pitch=inp["pitch"], duration=inp["duration"],
              times=inp["times"], noise=inp["noise"])
