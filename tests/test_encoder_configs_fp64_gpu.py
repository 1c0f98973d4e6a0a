"""GPU: the conditioning encoders against float64 across the configurations their constructors accept.

`tests/test_conditioning_backward_fp64_gpu.py` and `tests/test_duration_pitch_backward_fp64_gpu.py` check
`SpeechPromptEncoder`, `PhonemeEncoder` and `DurationPitchPredictor` at the reference's default dims (k = 9 convs,
dim 512, 8 heads, k = 3 trunk convs, 2 convs per ResnetBlock, 3 ResnetBlocks per layer).  The constructors take much
more, and the host code turns each configuration into its own segment lists, pack layouts and kernel parameters:
  * conv kernel sizes 1, 3, 5, 7, 11 and 12 (`ops.conv_segs` / `conv_dgrad_segs` with that many segments, one
    `ops.wgrad` per tap at shifts up to +-5, taps that read only the padding when N < k);
  * GroupNorm groups of 16, 48, 80 and 128 channels: 48 and 80 (v4 = 12, 20 float4 per row) do not divide the 256
    threads of `groupnorm_silu_bwd_kernel`, which then leaves threads idle;
  * attention widths heads x 64 that differ from dim (fused qkv, the predictor's separate q / kv GEMMs, the out-projection
    dgrad), conv widths of 64 and 192 channels (partial n-tiles), GEGLU inner widths 341, 682, 1365 and 2730 (padded to
    384, 768, 1408 and 2816) and 1024 (no padding);
  * ResnetBlocks of 1 and 3 Blocks and layers of 1 and 2 ResnetBlocks (the backward's walk of the saved blocks).

Reference and protocol are those of the two default-dims modules, with the encoders' family of tests/fp64_check.py:
every parameter is rounded to bf16 in place, inputs and upstream gradients are bf16-representable, and the reference is the
float64 restatement (`oracle.encoders_oracle`, pinned to the reference modules at these knobs by
tests/test_encoders_cpu.py and tests/golden/encoder_configs.npz) on the GPU with cuDNN off.  A tensor passes when
  (i)   rel-L2 <= C x the rel-L2 of the same restatement in fp32 under torch.autocast("cuda", bfloat16) + floor,
  (ii)  rel-L2 <= ceiling,
  (iii) it is exactly zero wherever the fp64 value is exactly zero, and nothing is non-finite.
The self-attention to_q of the prompt and phoneme encoders is bounded by TO_Q_BOUND relative to the fused q / kv
gradient, for the reason test_conditioning_backward_fp64_gpu.py gives, under fp64_check.EITHER (below); the predictor's
to_q meets the common bound.
The predictor's head biases are chosen as in its module, away from the ReLU kink.

Per run: (1) the inference forward against fp64, and two calls bit-identical; (2) the training forward (autograd in
train() mode, no dropout) bit-identical to the inference forward; (3) the training backward: every parameter gradient,
d x of the prompt encoder and of the predictor (or its token table's gradient) and d prompts, from random bf16 upstream
gradients.  Per configuration, (4) a ragged batch: per-sample lengths including 1 and the full length, NaN in every
padded float input row (random ids past a text's length), each sample against float64 run on it alone, unpadded,
bit-identical to the module run on it alone, and exact zeros in the padded output rows.  The predictor's valid rows are
compared together there (a length-1 sample gives two numbers, too few for a rel-L2), with head biases that keep every
sample's pre-activations alive.  With every parameter frozen, an input that requires grad still gets its gradient.

Wrong references that the same bounds must reject: a GroupNorm whose statistics leave out each group's last channel
quad (dpp_384), "same" convs padded k//2 - 1 on the left (spe_k11), the causal conv padded k - 2 on the left
(phon_k12), and attention scaled by (heads x 64)^-1/2 instead of 64^-1/2 (spe_k3_narrow).

Two findings shaped the comparison, neither a kernel error:
  * to_q at five frames (spe_k11-N5): the attention is far from flat, so to_q's gradient is ~40 % of the fused q / kv
    gradient, and its ordinary bf16 error (rel-L2 9.2e-3, below the autocast twin's 1.09e-2) is 3.65e-3 of it, over
    TO_Q_BOUND.  TO_Q_BOUND exists for nearly flat attention, where the twin comparison says nothing; a self-attention
    to_q therefore passes under the common bound or under TO_Q_BOUND.
  * The predictor's output at T = 1 (dpp_128-T1): the pitch head has three values, and its head bias leaves live rows
    0.14 above the kink, where our 5.2e-3 absolute error (the twin's is 2.5x larger) is rel-L2 2.1e-2 of the pitch
    alone, over the ceiling.  The predictor's output is compared whole, both predictions as one tensor (1.9e-3 there).

Measured on an H100 80GB HBM3 (700 W power limit).  Worst tensor per run, rel-L2 ours / autocast-bf16 of the same
tensor, and the tightest use of a bound:
  spe_k3_narrow-N1    transformer.layers.1.3.0.weight                   8.7e-3 / 1.07e-2   54 %
  spe_k3_narrow-N2    x                                                 1.18e-2 / 1.35e-2  60 %
  spe_k3_narrow-N129  x                                                 8.5e-3 / 1.15e-2   62 %
  spe_k1_wide         transformer.layers.0.0.gamma                      4.4e-3 / 6.0e-3    42 %
  spe_k11-N5          conv.1.weight                                     8.5e-3 / 9.9e-3    51 %
  spe_k11-N103        x                                                 6.7e-3 / 9.6e-3    48 %
  phon_d64-T1         transformer.layers.0.2.gamma                      7.7e-3 / 1.05e-2   47 %
  phon_d64-T2         transformer.layers.0.2.gamma                      9.2e-3 / 1.11e-2   57 %
  phon_d64-T37        transformer.layers.0.2.gamma                      7.4e-3 / 7.0e-3    65 %
  phon_k12-T9         token_emb.weight                                  6.5e-3 / 7.1e-3    51 %
  phon_k12-T100       conv.1.weight                                     6.6e-3 / 7.8e-3    50 %
  phon_k1             conv.1.weight                                     6.9e-3 / 8.3e-3    51 %
  dpp_128-T1          to_duration_pred.layers.1.1.gamma                 8.0e-3 / 6.3e-3    70 %
  dpp_128-T2          to_duration_pred.layers.1.2.to_q.weight           7.0e-3 / 6.7e-3    60 %
  dpp_128-T40         to_duration_pred.layers.1.2.to_q.weight           7.1e-3 / 8.5e-3    49 %
  dpp_384             to_pitch_pred.layers.0.1.gamma                    6.4e-3 / 8.0e-3    46 %
  dpp_640             to_pitch_pred.layers.0.2.to_q.weight              5.4e-3 / 6.8e-3    44 %
  dpp_1024            to_pitch_pred.layers.0.2.to_out.weight            7.1e-3 / 9.0e-3    48 %
  dpp_1024-dur_only   to_duration_pred.layers.0.2.to_q.weight           5.7e-3 / 7.2e-3    44 %
  dpp_table           to_duration_pred.layers.0.0.2.blocks.0.norm.bias  1.37e-2 / 1.61e-2  69 %
The largest ours / autocast-bf16 ratio of any tensor is 1.27, and the tightest tensor uses 70 % of its bound.  The
whole inference output sits at 2.4e-3 ... 5.2e-3 for the encoders (autocast-bf16 4.5e-3 ... 7.9e-3) and 3.3e-4 ...
3.6e-3 for the predictor (8.7e-4 ... 4.8e-3).  Ragged samples against fp64 alone: 2.4e-3 ... 4.0e-3 (autocast-bf16
4.4e-3 ... 6.2e-3), the predictor's valid rows 4.2e-4 ... 2.3e-3.  The wrong references sit at rel-L2 2.1e-2 ... 4.2e-2
(GroupNorm without the last quad, the smallest margin: 2.8x the bound on d x), 1.1 ... 1.4 (conv taps one row off),
0.43 (causal conv padded k - 2) and 9.4e-2 ... 1.5 (attention scale; to_q 1.6e-2 ... 9.6e-2 of the q / kv gradient).
The whole module takes ~20 s.
"""
import functools
import time

import pytest
import torch
import torch.nn.functional as F

from fp64_check import (EITHER, ENCODERS, MARGIN, assert_rejected, autograd, bf, bound, compare, over,
                        use)
from oracle import encoders_oracle as eo
from restatements import DPP, PHON, SPE, TRUNKS, build_config, config_fwd, config_heads, set_head_biases
from restatements import ENCODER_CONFIGS as CONFIGS

pytestmark = pytest.mark.gpu

RUNS = {
    # name: (configuration, B, N (prompt frames / text length), predictor: Np / encoders: text lengths (-1 past),
    #        predictions that get a gradient)
    "spe_k3_narrow-N1": ("spe_k3_narrow", 3, 1, None, "both"),
    "spe_k3_narrow-N2": ("spe_k3_narrow", 3, 2, None, "both"),
    "spe_k3_narrow-N129": ("spe_k3_narrow", 3, 129, None, "both"),
    "spe_k1_wide": ("spe_k1_wide", 2, 300, None, "both"),
    "spe_k11-N5": ("spe_k11", 2, 5, None, "both"),
    "spe_k11-N103": ("spe_k11", 2, 103, None, "both"),
    "phon_d64-T1": ("phon_d64", 3, 1, (1, 1, 1), "both"),
    "phon_d64-T2": ("phon_d64", 3, 2, (2, 1, 2), "both"),
    "phon_d64-T37": ("phon_d64", 3, 37, (37, 20, 5), "both"),
    "phon_k12-T9": ("phon_k12", 2, 9, (9, 4), "both"),
    "phon_k12-T100": ("phon_k12", 2, 100, (100, 61), "both"),
    "phon_k1": ("phon_k1", 2, 64, (64, 30), "both"),
    "dpp_128-T1": ("dpp_128", 3, 1, 7, "both"),
    "dpp_128-T2": ("dpp_128", 3, 2, 1, "both"),
    "dpp_128-T40": ("dpp_128", 3, 40, 7, "both"),
    "dpp_384": ("dpp_384", 2, 65, 129, "both"),
    "dpp_640": ("dpp_640", 2, 33, 64, "both"),
    "dpp_1024": ("dpp_1024", 2, 100, 103, "both"),
    "dpp_1024-dur_only": ("dpp_1024", 2, 100, 103, "duration"),
    "dpp_table": ("dpp_table", 2, 50, 40, "both"),
}
RAGGED_RUN = {cfg: max((r for r in RUNS if RUNS[r][0] == cfg), key=lambda r: RUNS[r][2]) for cfg in CONFIGS}


def _is_self_q(cls, name):
    return cls != DPP and name.endswith(".1.to_q.weight")


def _outputs(fwd, params, inputs, autocast=False):
    """The restatement's outputs (fp64 values) without gradients."""
    dtype = torch.float32 if autocast else torch.float64
    P = {n: p.detach().to(dtype) for n, p in params.items()}
    P.update({n: t.to(dtype) for n, t in inputs.items() if t.is_floating_point()})
    with torch.no_grad(), torch.backends.cudnn.flags(enabled=False):
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
            return {k: o.double() for k, o in fwd(P, dtype).items()}


def _inputs(run):
    cfg, B, N, extra, _ = RUNS[run]
    cls, kw, _, _ = CONFIGS[cfg]
    g = torch.Generator().manual_seed(100 + list(RUNS).index(run))
    if cls == SPE:
        return {"x": bf(g, B, N, kw["dim_codebook"])}, g
    if cls == PHON:
        ids = torch.randint(0, kw["num_tokens"], (B, N), generator=g)
        for b, n in enumerate(extra):
            ids[b, n:] = -1
        return {"ids": ids.cuda()}, g
    if "num_phoneme_tokens" in kw:
        x = torch.randint(0, kw["num_phoneme_tokens"], (B, N), generator=g).cuda()
    else:
        x = bf(g, B, N, kw["dim_hidden"])
    return {"x": x, "prompts": bf(g, B, extra, kw["dim_hidden"])}, g


def _alive_biases(m, cfg, samples):
    """Head biases (bf16 values) under which every fp64 pre-activation of every (x, prompts) sample is at least a
    quarter of the pre-activations' spread above 0."""
    params = {n: p.detach() for n, p in m.named_parameters()}
    for t in TRUNKS:
        params[t + "to_pred.0.bias"] = torch.full_like(params[t + "to_pred.0.bias"], 1e3)
    pre = {k: [] for k in ("duration", "pitch")}
    for x, p in samples:
        for k, o in _outputs(config_fwd(cfg, x, p), params, {}).items():
            pre[k].append(o.flatten() - 1e3)
    with torch.no_grad():
        for t, k in zip(TRUNKS, ("duration", "pitch")):
            v = torch.cat(pre[k])
            b = torch.tensor(0.25 * float(v.max() - v.min() + 1e-3) - float(v.min())).bfloat16().float().item()
            m.get_submodule(t[:-1]).to_pred[0].bias.fill_(b)


# ---- one run ----
_CACHE = {}
KEEP = {   # our gradients kept for the wrong references
    "spe_k3_narrow-N129": ("conv.1.weight", "x", *(f"transformer.layers.{l}.1.{w}.weight" for l in range(2)
                                                   for w in ("to_q", "to_kv"))),
    "spe_k11-N103": ("conv.1.weight", "conv.3.weight", "x"),
    "phon_k12-T100": ("conv.1.weight", "token_emb.weight"),
    "dpp_384": ("to_duration_pred.layers.0.0.0.blocks.0.norm.weight", "to_pitch_pred.layers.0.0.0.blocks.2.norm.weight",
                "x"),
}


def _run(run):
    if run in _CACHE:
        return _CACHE[run]
    t0 = time.perf_counter()
    cfg, B, N, extra, which = RUNS[run]
    cls, kw, _, _ = CONFIGS[cfg]
    m = build_config(cfg)
    inputs, g = _inputs(run)
    table = cls == DPP and "num_phoneme_tokens" in kw
    if cls == DPP:
        x, prompts = inputs["x"], inputs["prompts"]
        biases = set_head_biases(m, x, prompts, table, heads=config_heads(cfg))
        d_outs = {"duration": bf(g, B, N, scale=0.05), "pitch": bf(g, B, N, scale=0.05) if which == "both" else None}
        fwd = config_fwd(cfg, x, prompts)
        args = (x, prompts)
    else:
        x = inputs.get("x", inputs.get("ids"))
        biases = None
        d_outs = {"encoding": bf(g, B, N, m.dim_out if cls == SPE else m.dim_hidden)}
        fwd = config_fwd(cfg, x)
        args = (x,)
    ref_inputs = {k: v for k, v in inputs.items() if v.is_floating_point()}

    # (1) inference, twice
    m.eval()
    with torch.no_grad():
        inf = [m(*args), m(*args)]
    inf = [o if isinstance(o, tuple) else (o,) for o in inf]
    # (2) + (3) training forward and backward
    m.train()
    leaves = [a.clone().requires_grad_(True) if a.is_floating_point() else a for a in args]
    outs = m(*leaves)
    outs = outs if isinstance(outs, tuple) else (outs,)
    keys = list(d_outs)
    used = [(o, d_outs[k]) for o, k in zip(outs, keys) if d_outs[k] is not None]
    torch.autograd.backward([o for o, _ in used], [d for _, d in used])
    ours = {n: p.grad for n, p in m.named_parameters()}
    for name, leaf in zip(("x", "prompts"), leaves):
        if leaf.is_floating_point():
            ours[name] = leaf.grad
    ours.update({"out " + k: o for k, o in zip(keys, inf[0])})
    twice = all(torch.equal(a, b) for a, b in zip(*inf))
    train_eq = all(torch.equal(a, b.detach()) for a, b in zip(inf[0], outs))

    params = {n: p.detach().clone() for n, p in m.named_parameters()}
    ref = autograd(fwd, params, d_outs, inputs=ref_inputs, cudnn=False, out_prefix="out ")
    ac = autograd(fwd, params, d_outs, autocast=True, inputs=ref_inputs, cudnn=False, out_prefix="out ")

    fails, stats, none_ok = [], {}, True
    if cls == DPP:   # the whole output: both predictions as one tensor
        for d in (ours, ref, ac):
            d["out duration, pitch"] = torch.stack((d.pop("out duration"), d.pop("out pitch")))
    for n, r in ref.items():
        o = ours.get(n)
        if which == "duration" and n.startswith(TRUNKS[1]):
            none_ok &= o is None
            continue
        if o is None or o.shape != r.shape:
            fails.append((n, "missing" if o is None else f"shape {tuple(o.shape)} != {tuple(r.shape)}"))
            continue
        s = compare(o, r, ac[n], ref[n.replace("to_q", "to_kv")] if _is_self_q(cls, n) else None)
        if isinstance(s, str):
            fails.append((n, s))
        elif s is not None:
            stats[n] = s
    fwd_err = min_pre = None
    if cls == DPP:   # the ReLU margin of the predictor module: every |pre| >= MARGIN x our forward's max-abs error
        fwd_err = float((ours["out duration, pitch"].double() - ref["out duration, pitch"]).abs().max())
        P = dict(params, **{t + "to_pred.0.bias": params[t + "to_pred.0.bias"] + 1e3 for t in TRUNKS})
        min_pre = min(float((o - 1e3).abs().min()) for o in _outputs(fwd, P, ref_inputs).values())
    res = dict(cls=cls, cfg=cfg, stats=stats, fails=fails, twice=twice, train_eq=train_eq, none_ok=none_ok,
               fwd_err=fwd_err, min_pre=min_pre, biases=biases, params=params, inputs=inputs, ref_inputs=ref_inputs,
               d_outs=d_outs, fwd=fwd, ours={n: ours[n].clone() for n in KEEP.get(run, ()) + ("x", "prompts")
                                              if ours.get(n) is not None})
    if run == RAGGED_RUN[cfg]:
        res["ragged"] = _ragged(m, cfg, inputs)
    del ours, ref, ac, m
    torch.cuda.empty_cache()
    res["seconds"] = time.perf_counter() - t0
    _CACHE[run] = res
    return res


def _ragged(m, cfg, inputs):
    """(4): one padded batch with per-sample lengths against each sample run alone -> {sample: stats or failure}."""
    cls, kw, lens, plens = CONFIGS[cfg]
    m.eval()
    g = torch.Generator().manual_seed(7)
    res = {}
    with torch.no_grad():
        if cls == DPP:
            x, prompts = inputs["x"], inputs["prompts"]
            alone_in = [(x[b:b + 1, :n], prompts[b:b + 1, :pn]) for b, (n, pn) in enumerate(zip(lens, plens))]
            _alive_biases(m, cfg, alone_in)
            if x.is_floating_point():
                xr = x.clone()
                for b, n in enumerate(lens):
                    xr[b, n:] = float("nan")
            else:
                xr = torch.randint(0, kw["num_phoneme_tokens"], x.shape, generator=g).cuda()   # random past the lengths
                for b, n in enumerate(lens):
                    xr[b, :n] = x[b, :n]
            pr = prompts.clone()
            for b, n in enumerate(plens):
                pr[b, n:] = float("nan")
            got = torch.stack(m(xr, pr, lengths=list(lens), prompt_lens=list(plens)), -1)     # (B, T, 2)
            alone = [torch.stack(m(*a), -1)[0] for a in alone_in]
            params = {n: p.detach() for n, p in m.named_parameters()}
            refs = [torch.stack(list(_outputs(config_fwd(cfg, *a), params, {}).values()), -1)[0] for a in alone_in]
            acs = [torch.stack(list(_outputs(config_fwd(cfg, *a), params, {}, autocast=True).values()), -1)[0]
                   for a in alone_in]
            valid = [got[b, :n] for b, n in enumerate(lens)]
            res["valid rows"] = compare(torch.cat(valid), torch.cat(refs), torch.cat(acs))
        else:
            if cls == SPE:
                xr = inputs["x"].clone()
                for b, n in enumerate(lens):
                    xr[b, n:] = float("nan")
                alone_in = [xr[b:b + 1, :n] for b, n in enumerate(lens)]
            else:
                xr = torch.randint(0, kw["num_tokens"], inputs["ids"].shape, generator=g).cuda()
                alone_in = [xr[b:b + 1, :n] for b, n in enumerate(lens)]
            got = m(xr, lengths=list(lens))
            alone = [m(a)[0] for a in alone_in]
            valid = [got[b, :n] for b, n in enumerate(lens)]
            params = {n: p.detach() for n, p in m.named_parameters()}
            for b, a in enumerate(alone_in):
                r = _outputs(config_fwd(cfg, a), params, {"x": a} if cls == SPE else {})["encoding"][0]
                ac = _outputs(config_fwd(cfg, a), params, {"x": a} if cls == SPE else {}, autocast=True)["encoding"][0]
                res[f"sample {b} (length {lens[b]})"] = compare(valid[b], r, ac)
    res["bit-identical to alone"] = all(torch.equal(v, a) for v, a in zip(valid, alone))
    res["padding zeros"] = all(int((got[b, n:] != 0).sum()) == 0 for b, n in enumerate(lens))
    return res


@pytest.mark.parametrize("run", list(RUNS))
def test_matches_fp64(run):
    r = _run(run)
    stats = r["stats"]
    rest = {n: s for n, s in stats.items() if s.share is None}
    worst = max(rest.items(), key=lambda kv: kv[1].rel)
    tight = max(stats.items(), key=lambda kv: use(ENCODERS, kv[1], EITHER))
    ratio = max(((n, s) for n, s in rest.items() if s.rel_ac > 0), key=lambda kv: kv[1].rel / kv[1].rel_ac)
    q = [s.share for s in stats.values() if s.share is not None]
    outs = {n: s for n, s in stats.items() if n.startswith("out ")}
    print(f"\n{run}: {len(stats)} tensors in {r['seconds']:.1f} s; worst {worst[0]} ours {worst[1].rel:.2e} / autocast "
          f"{worst[1].rel_ac:.2e}; max ratio {ratio[1].rel / ratio[1].rel_ac:.2f} ({ratio[0]}); tightest {tight[0]} at "
          f"{use(ENCODERS, tight[1], EITHER):.0%} of its bound" + (f"; worst to_q share {max(q):.2e}" if q else "") +
          "; forward " + ", ".join(f"{n[4:]} {s.rel:.2e} / {s.rel_ac:.2e}" for n, s in outs.items()) +
          (f"; forward max-abs {r['fwd_err']:.2e}, min |pre| {r['min_pre']:.2e}, head biases {r['biases']}"
           if r["cls"] == DPP else ""))
    assert r["twice"], "two inference calls differ"
    assert r["train_eq"], "the training forward must be bit-identical to the inference forward"
    assert r["none_ok"], "a trunk without an upstream gradient must leave its parameters' .grad None"
    if r["cls"] == DPP:
        assert r["min_pre"] >= MARGIN * r["fwd_err"], "fixture: a head pre-activation lies too close to 0"
    assert not r["fails"], r["fails"][:8]
    bad = [(n, s) for n, s in stats.items() if over(ENCODERS, s, EITHER)]
    assert not bad, f"{len(bad)} tensors over the bound (rel-L2, autocast rel-L2, to_q share): {bad[:8]}"


@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_ragged_batch_matches_each_sample_alone(cfg):
    rg = _run(RAGGED_RUN[cfg])["ragged"]
    checks = {k: v for k, v in rg.items() if k not in ("bit-identical to alone", "padding zeros")}
    print(f"\n{cfg} ragged {CONFIGS[cfg][2:]}: " + "; ".join(
        f"{k} {v}" if not isinstance(v, tuple) else f"{k} {v[0]:.2e} / {v[1]:.2e}" for k, v in checks.items()))
    assert rg["bit-identical to alone"], "a sample of the ragged batch differs from the sample run alone"
    assert rg["padding zeros"], "padded output rows must be exact zeros"
    for k, v in checks.items():
        assert not isinstance(v, str), (k, v)
        assert v is None or not over(ENCODERS, v, EITHER), (k, v, bound(ENCODERS, v[1]))


def test_input_grads_with_frozen_parameters():
    """Every parameter frozen, the input requiring grad: the prompt encoder and the predictor still record their node
    and give the inputs the gradients of the run with trainable parameters, bit for bit."""
    for run in ("spe_k3_narrow-N129", "dpp_128-T40"):
        r = _run(run)
        m = build_config(r["cfg"])
        if r["cls"] == DPP:
            set_head_biases(m, r["inputs"]["x"], r["inputs"]["prompts"], False, heads=config_heads(r["cfg"]))
        m.requires_grad_(False)
        m.train()
        leaves = [r["inputs"][k].clone().requires_grad_(True) for k in ("x", "prompts") if k in r["inputs"]]
        outs = m(*leaves)
        outs = outs if isinstance(outs, tuple) else (outs,)
        assert all(o.requires_grad for o in outs), run
        torch.autograd.backward(list(outs), [r["d_outs"][k] for k in r["d_outs"]])
        for k, leaf in zip(("x", "prompts"), leaves):
            assert torch.equal(leaf.grad, r["ours"][k]), (run, k)


# ---- wrong references ----
def _assert_rejected(run, fwd, names):
    r = _run(run)
    wrong = autograd(fwd, r["params"], r["d_outs"], inputs=r["ref_inputs"], only=names, cudnn=False)
    assert_rejected(r["ours"], wrong, r["stats"], names, ENCODERS, EITHER)


def _group_norm_without_last_quad(h, groups, weight, bias, eps):
    """GroupNorm whose mean and variance leave out the last 4 channels of every group (they are still normalised)."""
    B, C, N = h.shape
    hg = h.reshape(B, groups, C // groups, N)
    s = hg[:, :, :-4]
    mean = s.mean(dim=(2, 3), keepdim=True)
    var = s.var(dim=(2, 3), unbiased=False, keepdim=True)
    return ((hg - mean) / torch.sqrt(var + eps)).reshape(B, C, N) * weight[:, None] + bias[:, None]


def test_rejects_group_norm_without_the_last_channel_quad():
    r = _run("dpp_384")
    fwd = config_fwd("dpp_384", r["inputs"]["x"], r["inputs"]["prompts"],
                       trunk=functools.partial(eo._trunk, group_norm=_group_norm_without_last_quad))
    _assert_rejected("dpp_384", fwd, list(KEEP["dpp_384"]))


def test_rejects_same_conv_taps_one_row_off():
    """spe_k11's convs padded (k//2 - 1, k//2 + 1): every tap reads one row later."""
    k, heads = CONFIGS["spe_k11"][1]["kernel_size"], config_heads("spe_k11")

    def fwd(P, dtype):
        h = P["x"].to(dtype).transpose(1, 2)
        for i in (1, 3):
            h = F.silu(F.conv1d(F.pad(h, (k // 2 - 1, k // 2 + 1)), P[f"conv.{i}.weight"], P[f"conv.{i}.bias"]))
        return {"encoding": eo.transformer(h.transpose(1, 2), P, "transformer.", heads)}
    _assert_rejected("spe_k11-N103", fwd, list(KEEP["spe_k11-N103"]))


def test_rejects_causal_conv_padded_one_short():
    """phon_k12's causal conv padded (k - 2, 1) instead of (k - 1, 0)."""
    r = _run("phon_k12-T100")
    ids, heads = r["inputs"]["ids"], config_heads("phon_k12")

    def fwd(P, dtype):
        pad_id = P["token_emb.weight"].shape[0] - 1
        w = P["conv.1.weight"]
        h = P["token_emb.weight"][ids.masked_fill(ids < 0, pad_id)].transpose(1, 2)
        h = F.silu(F.conv1d(F.pad(h, (w.shape[-1] - 2, 1)), w, P["conv.1.bias"]))
        return {"encoding": eo.transformer(h.transpose(1, 2), P, "transformer.", heads)}
    _assert_rejected("phon_k12-T100", fwd, list(KEEP["phon_k12-T100"]))


def test_rejects_attention_scaled_by_the_attention_width():
    """spe_k3_narrow's attention scaled by (heads x 64)^-1/2: q scaled by heads^-1/2 inside the restatement."""
    r = _run("spe_k3_narrow-N129")
    heads = config_heads("spe_k3_narrow")
    base = config_fwd("spe_k3_narrow", r["inputs"]["x"])

    def fwd(P, dtype):
        q = {n: v * heads ** -0.5 for n, v in P.items() if n.endswith(".to_q.weight")}
        return base(dict(P, **q), dtype)
    _assert_rejected("spe_k3_narrow-N129", fwd, list(KEEP["spe_k3_narrow-N129"]))
