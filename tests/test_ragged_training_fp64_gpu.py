"""GPU: training on padded batches with per-sample lengths against float64, sample by sample, across the module
configurations and past the first key tile.

`tests/test_ragged_training_gpu.py` checks ragged training against our own single-sample ("alone") calls at shapes that
never leave one key tile.  This module checks the same calls against the float64 restatements, at padded lengths of
300 where every attention backward spans three 128-key tiles and five 64-query tiles, and across the configurations
the constructors accept:
  * SpeechPromptEncoder / PhonemeEncoder(lengths=): `spe_k3_narrow`, `spe_k1_wide`, `spe_k11`, `phon_d64`, `phon_k12`
    and `phon_k1` of restatements.ENCODER_CONFIGS (test_encoder_configs_fp64_gpu.py), and both encoders at their
    default dims;
  * Model(prompt_lens=): the conditional cases `ff2_cond` (cond_drop_prob 0.5: dropped and kept samples both carry
    lengths), `ff8_cond` (no perceiver projection), `w640_m1` (one latent) and `w1024_b50` (B 50, 33 latents, resampler
    depth 3) of restatements.DENOISER_CASES (test_denoiser_configs_fp64_gpu.py) with their prompts padded to 300
    frames, and `bench` (dim 512, 8 heads, depth 2, 32 latents: M + length lands on 33, 128, 129, 256 and 332 keys);
  * Conditioner(mode="train", prompt_lens=, phoneme_lens=) at the encoders' default dims;
  * NaturalSpeech2.forward(prompt_lens=, phoneme_lens=).
Each padded batch mixes lengths 1, 63 / 64 / 65, 127 / 128 / 129 and the full length, unsorted, with one length used
twice; a sample of length 1 or 40 at 300 frames leaves its last two key tiles to the backward's early exit, and 129
(or M + 97) puts the last valid key tile at tile 1.  spe_k11 also has lengths 2 and 4, below k // 2, so the taps reach
past both ends of a sample.  Padded float inputs hold NaN, and padded ids are tokens no valid position uses.

The reference of a padded batch is the float64 restatement run on each sample alone, unpadded (`oracle.encoders_oracle`
for the encoders and the Conditioner, `oracle.denoiser_torch_port.model_forward_autograd` for the denoiser; samples of
one length run together, which for the restatement is the same computation).  With the loss sum_b <out_b, up_b> and
bf16-representable upstream gradients, each sample's input gradient (d prompt rows, d cond, d x) is that sample's
float64 gradient and each parameter gradient the sum over samples.  The autocast-bf16 twin is computed the same way, so
the bounds of the default-dims modules apply unchanged: rel-L2 <= C x twin + floor and <= ceiling
(the encoders' constants and to_q rule for the encoders and the Conditioner, the denoiser's for the Model), exact zeros
wherever float64 is exactly zero, nothing non-finite.  Per case also:
  * forward: each sample's output is bit-identical to the alone call, and padded output rows are exact zeros;
  * the batch against the sum of our alone calls, per gradient tensor (parameters, and each sample's input
    gradients), with the spread of two runs of the same batch call printed;
  * exact zeros: d prompt rows past prompt_lens[b], every d prompt row of a null-substituted sample, token-table rows
    that only padded ids reach, pitch-table rows with no valid frame, and in the phoneme encoder the padded rows of
    every intermediate gradient its backward forms (the argument of encoders.PhonemeEncoder._train_backward that the
    causal conv and the zero d K / d V rows keep them zero without a mask).

The batch against the alone calls: RTOL = 2^-19 of test_ragged_training_gpu.py holds only where every attention fits
one key tile.  Past it the attention backward adds each key tile's dQ into the query tile's fp32 accumulator with
atomics, in an order that varies with the launch: a last-bit difference moves a bf16 rounding of dQ, and the roundings
after it in the backward move with it, so the gradients further down differ at the level of bf16 rounding noise.
Measured on an H100 80GB HBM3 (700 W power limit) over two runs of the module, two runs of the same batch call differ
by up to 5.9e-3 (bench, d cond), 4.8e-3 (w640_m1), 3.6e-3 (Conditioner), 3.3e-3 (spe_k3_narrow, 1.1e-7 in the other
run), 2.5e-3 (w1024_b50), 1.8e-3 (spe_default) and 1.75e-3 (ff2_cond), and the batch against the alone sums by up to
5.8e-3, 5.0e-3, 3.6e-3, 2.2e-3, 2.6e-3, 1.7e-3 and 1.75e-3; the other cases stay at 1e-7 ... 2e-5.  So here the batch
against the alone sums is held to the bound of the float64 comparison of the same tensor (it uses at most 51 % of it:
w640_m1, d prompt of sample 8); the float64 comparison is the check of correctness.
NaturalSpeech2.forward's loss is mean_b(mse_b) * mean_b(w_b) (see test_ragged_training_gpu.py), so each parameter
gradient is (mean(w) / B) sum_b g_b / w_b, with g_b the alone call's gradient at the same times and noise.  The bf16 cast
of d pred in the denoiser's backward does not commute with a scale that is not a power of two, so the alone calls are
run from d mse_b = the batch's own d mse (mean(w) / B, checked against it), which is g_b / w_b x mean(w) / B with the
batch's roundings, at shapes within one key tile.

Wrong references, with finite +-1e4 junk in the padded rows they read, must fail the same bounds: the perceiver
attending to one padded prompt row (M + length + 1 keys), the prompt mean-pool divided by the padded Np, spe_k11's
"same" convs reading the first padded rows instead of zeros, and the phoneme encoder's self-attention including one
padded token.

Measured on an H100 80GB HBM3 (700 W power limit).  Per case the tensor that uses the largest share of its bound,
with its rel-L2 ours / autocast-bf16 (a self-attention to_q under the to_q rule is marked q), and the largest ratio ours
/ autocast-bf16 of any tensor:
  spe_k3_narrow  transformer.layers.1.0.gamma                     5.7e-3 / 5.2e-3     59 %   3.92
  spe_k1_wide    x (sample 1)                                     4.0e-3 / 5.9e-3     37 %   4.06
  spe_k11        x (sample 8, length 2)                           8.6e-3 / 1.05e-2    48 %   2.98
  spe_default    x (sample 2, length 300)                         1.42e-2 / 1.12e-2   76 %   3.58
  phon_d64       transformer.layers.1.1.to_q.weight (q)           1.9e-1 / 1.7e-2     75 %   2.55
  phon_k12       transformer.layers.0.1.to_q.weight (q)           3.8e-2 / 1.0e-2     69 %   3.38
  phon_k1        transformer.layers.0.1.to_q.weight (q)           3.0e-2 / 1.6e-2     50 %   3.35
  phon_default   transformer.layers.5.1.to_q.weight (q)           4.3e1 / 2.5e-1      71 %   6.67
  ff2_cond       transformer.layers.0.2.to_gamma_beta.bias        1.06e-2 / 1.38e-2   71 %   0.77
  ff8_cond       d prompt (sample 2)                              5.8e-3 / 6.7e-3     67 %   0.87
  w640_m1        d prompt (sample 8)                              6.4e-3 / 7.3e-3     68 %   0.87
  w1024_b50      perceiver_resampler.layers.0.0.to_q.weight       9.2e-3 / 1.19e-2    66 %   0.80
  bench          transformer.layers.0.1.to_q.weight               1.05e-2 / 1.76e-2   70 %   0.75
  Conditioner    prompt_enc.transformer.layers.4.1.to_q.weight (q) 3.1e2 / 5.6e-1    80 %   3.39
The largest ratios (2.6 ... 6.7) are all on the last feed-forward bias of an encoder, where the twin's error is far
below the floor; every tensor is within its bound.  NaturalSpeech2.forward: the denoiser's gradients match the scaled
alone gradients to 8.6e-7, the conditioner's to 7.6e-3 (prompt_enc.conv.1.weight).  The wrong references sit at 106x
the bound (perceiver to_kv; 204x on latents, 437x on d prompt), 4.7x (mean-pool over Np, on d prompt of the 224-frame sample; 781x on to_prompt_cond),
21x (spe_k11 convs, on d x of the 129-frame sample; 59-65x on the conv weights) and 1.4x (phoneme attention over one
padded token, on layer 0's to_kv, the smallest margin; 6.9x on the token table and the conv).  The whole module takes
~85 s.
"""
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from fp64_check import DENOISER, EITHER, ENCODERS, assert_rejected, autograd, bf, compare, over, rel_qkv, round_params, use
from helpers import build_encoder, build_model
from oracle import denoiser_torch_port as tp
from oracle import encoders_oracle as eo
from param_fill import fill_module
from restatements import DENOISER_CASES as CASES
from restatements import ENCODER_CONFIGS as CONFIGS
from restatements import RTOL, build_config, conditioner_fwd, config_fwd, drop_masks, encoder_fwd, port_grads

pytestmark = pytest.mark.gpu

SPE, PHON = "SpeechPromptEncoder", "PhonemeEncoder"
FAMILY = {"enc": ENCODERS, "den": DENOISER}   # the Model's tensors take the denoiser's bounds, the rest the encoders'
NPAD = 300                                              # padded prompt frames / phonemes
LENS = (129, 1, 300, 64, 63, 128, 65, 40, 127, 64)      # unsorted, 64 twice
LENS_K11 = (129, 4, 300, 64, 1, 63, 128, 65, 2, 127, 64)
BENCH_LENS = (97, 1, 300, 96, 224, 64, 129, 40, 128, 96)   # M + length: 129, 33, 332, 128, 256, 96, 161, 72, 160, 128
_W = (1, 2, 40, 63, 64, 65, 94, 95, 96, 97, 127, 128, 129, 222, 223, 224, 255, 256, 257, 300)
B50_LENS = tuple(int(v) for v in np.random.default_rng(3).permutation(_W + _W + _W[:10]))
PHON_LENS = (64, 300, 1, 129, 128, 40, 63, 64, 65, 127)  # the Conditioner's phoneme lengths, paired with LENS
JUNK = 1e4

ENC_CASES = {
    # name: (a configuration of test_encoder_configs_fp64_gpu, or the class at its default dims; lengths)
    "spe_k3_narrow": ("spe_k3_narrow", LENS),
    "spe_k1_wide": ("spe_k1_wide", LENS),
    "spe_k11": ("spe_k11", LENS_K11),
    "spe_default": (SPE, LENS),
    "phon_d64": ("phon_d64", LENS),
    "phon_k12": ("phon_k12", LENS),
    "phon_k1": ("phon_k1", LENS),
    "phon_default": (PHON, LENS),
}
DEFAULT_KW = {SPE: dict(dim_codebook=128), PHON: dict(num_tokens=100)}
BENCH = dict(dim=512, depth=2, heads=8, dim_prompt=512, num_latents_m=32, condition_on_prompt=True)
DEN_CASES = {
    # name: (model kwargs, latent frames N, prompt lengths (padded to NPAD), cond frames, cond_drop_prob)
    "ff2_cond": (CASES["ff2_cond"][0], CASES["ff2_cond"][2], LENS, CASES["ff2_cond"][4], CASES["ff2_cond"][5]),
    "ff8_cond": (CASES["ff8_cond"][0], CASES["ff8_cond"][2], LENS, CASES["ff8_cond"][4], CASES["ff8_cond"][5]),
    "w640_m1": (CASES["w640_m1"][0], CASES["w640_m1"][2], LENS, CASES["w640_m1"][4], CASES["w640_m1"][5]),
    "w1024_b50": (CASES["w1024_b50"][0], CASES["w1024_b50"][2], B50_LENS, CASES["w1024_b50"][4], CASES["w1024_b50"][5]),
    "bench": (BENCH, 256, BENCH_LENS, 256, 0.),
}
assert DEN_CASES["ff2_cond"][4] == 0.5


def _groups(lens):
    """{length: sample indices} (samples of one length run together in the restatement)."""
    out = {}
    for b, n in enumerate(lens):
        out.setdefault(int(n), []).append(b)
    return out


def _is_self_q(name):
    return name.endswith(".1.to_q.weight") and name.startswith(("transformer.", "prompt_enc.", "phoneme_enc."))


def _acc(tot, grads, names):
    for n in names:
        g = grads[n]
        if g is not None:
            tot[n] = g.double() + tot[n] if n in tot else g.double().clone()


def _err(got, want):
    """Relative L2 error of `got` against `want` (0 when both are zero; inf when only `want` is; None is zero)."""
    if got is None or want is None:
        got, want = (torch.zeros(()) if t is None else t for t in (got, want))
    got, want = got.double(), want.double()
    d, w = float((got - want).norm()), float(want.norm())
    return 0.0 if d == 0 else (d / w if w > 0 else float("inf"))


def _against(res, ours, ref, ac, names):
    """Stats of ours against fp64 (ref) and its twin (ac) into res["stats"], failures into res["fails"]."""
    for n in names:
        o, r, a = ours.get(n), ref[n], ac[n]
        if o is None:
            if bool((r != 0).any()):
                res["fails"].append((n, "missing"))
            continue
        s = compare(o, r, a, ref[n.replace("to_q", "to_kv")] if res["family"] == "enc" and _is_self_q(n) else None)
        if isinstance(s, str):
            res["fails"].append((n, s))
        elif s is not None:
            res["stats"][n] = s


def _alone_spread(res, got, again, alone, names):
    """Run to run (printed) and the batch against the sum of the alone calls per tensor (rel-L2, and a self-attention
    to_q's share of its q / kv gradient); checked in _assert_case against the bound of the float64 comparison."""
    res["spread"] = max(((_err(again[n], got[n]), n) for n in names), default=(0.0, None))
    res["alone_errs"] = {}
    for n in names:
        share = None
        if res["family"] == "enc" and _is_self_q(n) and got[n] is not None:
            share = rel_qkv(got[n], alone[n], alone[n.replace("to_q", "to_kv")])
        res["alone_errs"][n] = (_err(got[n], alone.get(n)), share)


# ---- encoders ----
_CACHE = {}


def _enc_module(case):
    cfg, _ = ENC_CASES[case]
    if cfg in CONFIGS:
        return build_config(cfg), CONFIGS[cfg][0]
    m = build_encoder(cfg, DEFAULT_KW[cfg], seed=1234, device="cuda")
    round_params(m)
    return m, cfg


def _enc_fwd(case, x, cls, heads, padding):
    """fwd(P, dtype) of the restatement on one group of samples; the prompt frames are the leaf P["x"]."""
    cfg = ENC_CASES[case][0]
    if cfg in CONFIGS:
        return config_fwd(cfg, x)
    if cls == SPE:
        return lambda P, dtype: {"encoding": eo.speech_prompt_encoder(P, P["x"].to(dtype), heads=heads, padding=padding)}
    base = encoder_fwd(cls, x, (None, None))
    return lambda P, dtype: {"encoding": base(P, dtype)["out"]}


def _enc_inputs(case, m, cls):
    lens = ENC_CASES[case][1]
    B = len(lens)
    g = torch.Generator().manual_seed(50 + list(ENC_CASES).index(case))
    if cls == SPE:
        x = bf(g, B, NPAD, m.dim)
        junk = x.clone()
        for b, n in enumerate(lens):
            x[b, n:] = float("nan")
            junk[b, n:] = JUNK * torch.randn(NPAD - n, m.dim, generator=g).sign().cuda()
    else:
        V = m.pad_id
        x = torch.randint(0, V // 2, (B, NPAD), generator=g)
        for b, n in enumerate(lens):    # ids only the padding uses
            x[b, n:] = torch.randint(V // 2, V, (NPAD - n,), generator=g)
        x = junk = x.cuda()
    up = bf(g, B, NPAD, m.dim_out if cls == SPE else m.dim_hidden)
    return x, junk, up


def _spy_intermediates(monkeypatch, rows):
    """Record every intermediate gradient of the phoneme encoder's backward (after each kernel that forms one)."""
    from naturalspeech2_pytorch_b200 import ops

    def wrap(name, pick):
        fn = getattr(ops, name)

        def spy(*a, **kw):
            out = fn(*a, **kw)
            for label, t in pick(a, kw):
                rows.append((f"{name} {label}", t.detach().clone()))
            return out
        monkeypatch.setattr(ops, name, spy)
    wrap("attention_bwd", lambda a, kw: [("dQ", a[6]), ("dK", a[7]), ("dV", a[8]), ("dO", a[4])])
    wrap("rmsnorm_film_bwd", lambda a, kw: [("dh", a[1]), ("d residual", a[2]), ("d residual bf16", a[3])])
    wrap("silu_bwd", lambda a, kw: [("d pre", next(t for t in (kw.get("dpre"), a[2] if len(a) > 2 else None, a[0])
                                                   if t is not None))])
    wrap("embedding_bwd", lambda a, kw: [("d emb", a[1])])


def _enc_case(case):
    if case in _CACHE:
        return _CACHE[case]
    t0 = time.perf_counter()
    m, cls = _enc_module(case)
    m.train()
    lens = ENC_CASES[case][1]
    B = len(lens)
    x, junk, up = _enc_inputs(case, m, cls)
    names = [n for n, _ in m.named_parameters()]
    params = {n: p.detach() for n, p in m.named_parameters()}
    res = dict(family="enc", cls=cls, lens=lens, stats={}, fails=[], checks={})

    def batch(spy_rows=None):
        leaf = x.clone().requires_grad_(True) if cls == SPE else x
        with pytest.MonkeyPatch.context() as mp:
            if spy_rows is not None:
                _spy_intermediates(mp, spy_rows)
            out = m(leaf, lengths=list(lens))
            torch.autograd.backward(out, up)
        gr = {n: p.grad for n, p in m.named_parameters()}
        m.zero_grad(set_to_none=True)
        if cls == SPE:
            gr["x"] = leaf.grad
        return out.detach(), gr

    spy_rows = [] if cls == PHON else None
    out, got = batch(spy_rows)
    _, again = batch()
    # ours alone, one sample per call
    alone, alone_dx = {}, {}
    fwd_ok, pad_ok = True, True
    for b, n in enumerate(lens):
        leaf = x[b:b + 1, :n].clone().requires_grad_(True) if cls == SPE else x[b:b + 1, :n]
        ob = m(leaf)
        torch.autograd.backward(ob, up[b:b + 1, :n])
        _acc(alone, {k: p.grad for k, p in m.named_parameters()}, names)
        m.zero_grad(set_to_none=True)
        if cls == SPE:
            alone_dx[b] = leaf.grad[0]
        fwd_ok &= torch.equal(out[b, :n], ob.detach()[0])
        pad_ok &= int((out[b, n:] != 0).sum()) == 0
    res["checks"]["forward bit-identical to alone"] = fwd_ok
    res["checks"]["padded output rows are zeros"] = pad_ok
    if cls == SPE:
        for b, n in enumerate(lens):
            got[f"x {b}"], again[f"x {b}"], alone[f"x {b}"] = got["x"][b, :n], again["x"][b, :n], alone_dx[b]
        res["checks"]["d prompt rows past the lengths are zeros"] = all(
            int((got["x"][b, n:] != 0).sum()) == 0 for b, n in enumerate(lens))
    in_names = [f"x {b}" for b in range(B)] if cls == SPE else []
    _alone_spread(res, got, again, alone, names + in_names)
    if spy_rows is not None:
        bad = [(label, tuple(t.shape)) for label, t in spy_rows
               if t.dim() == 3 and t.shape[:2] == (B, NPAD) and
               any(int((t[b, n:] != 0).sum()) for b, n in enumerate(lens))]
        res["intermediates"] = (len(spy_rows), bad)
        emb = got["token_emb.weight"]
        res["checks"]["token rows only padded ids reach are zeros"] = int((emb[m.pad_id // 2:] != 0).sum()) == 0

    # float64 reference and its autocast-bf16 twin, per length group
    heads, padding = m.heads, getattr(m, "padding", None)
    ref, ac = {}, {}
    for dst, autocast in ((ref, False), (ac, True)):
        dx = {}
        for n, idx in _groups(lens).items():
            xs = x[idx, :n]
            extra = {"x": xs} if cls == SPE else {}
            gr = autograd(_enc_fwd(case, xs, cls, heads, padding), dict(params, **extra), {"encoding": up[idx, :n]},
                          autocast=autocast, only=names + list(extra), cudnn="twin")
            _acc(dst, gr, names)
            for i, b in enumerate(idx):
                if cls == SPE:
                    dst[f"x {b}"] = gr["x"][i].double()
    _against(res, got, ref, ac, names + in_names)
    res.update(params=params, x=x, junk=junk, up=up, heads=heads, padding=padding,
               ours={n: got[n].clone() for n in in_names + [k for k in names if k.startswith("conv.") and
                                                            k.endswith(".weight") or "layers.0.1." in k
                                                            or k == "token_emb.weight"]})
    del got, again, alone, ref, ac, m
    torch.cuda.empty_cache()
    res["seconds"] = time.perf_counter() - t0
    _CACHE[case] = res
    return res


def _alone_use(res):
    """{name: share of its bound} of the batch against the sum of the alone calls; inf where float64 is exactly zero
    and the two differ."""
    out = {}
    for n, (e, share) in res["alone_errs"].items():
        if n in res["stats"]:
            out[n] = use(FAMILY[res["family"]], (e, res["stats"][n].rel_ac, share), EITHER)
        else:
            out[n] = 0.0 if e == 0 else float("inf")
    return out


def _report(name, res):
    stats = res["stats"]
    fam = FAMILY[res["family"]]
    worst = max(stats.items(), key=lambda kv: kv[1].rel)
    tight = max(stats.items(), key=lambda kv: use(fam, kv[1], EITHER))
    ratio = max(((n, s) for n, s in stats.items() if s.rel_ac > 0 and s.share is None),
                key=lambda kv: kv[1].rel / kv[1].rel_ac)
    alone = max(_alone_use(res).items(), key=lambda kv: kv[1])
    print(f"\n{name}: {len(stats)} tensors in {res['seconds']:.1f} s; worst {worst[0]} ours {worst[1].rel:.2e} / "
          f"autocast {worst[1].rel_ac:.2e}; max ratio {ratio[1].rel / ratio[1].rel_ac:.2f} ({ratio[0]}); tightest "
          f"{tight[0]} at {use(fam, tight[1], EITHER):.0%} of its bound (ours {tight[1].rel:.2e} / autocast "
          f"{tight[1].rel_ac:.2e}); batch vs alone: largest {max(e for e, _ in res['alone_errs'].values()):.2e}, "
          f"tightest {alone[0]} at {alone[1]:.0%} of its bound; run to run {res['spread'][0]:.2e} ({res['spread'][1]})")


def _assert_case(res):
    bad_checks = [k for k, ok in res["checks"].items() if not ok]
    assert not bad_checks, bad_checks
    assert not res["fails"], res["fails"][:8]
    bad = [(n, s) for n, s in res["stats"].items() if over(FAMILY[res["family"]], s, EITHER)]
    assert not bad, f"{len(bad)} tensors over the bound (rel-L2, autocast rel-L2, to_q share): {bad[:8]}"
    over_alone = [(n, res["alone_errs"][n], u) for n, u in _alone_use(res).items() if u > 1]
    assert not over_alone, f"batch vs the sum of the alone calls over the bound: {over_alone[:8]}"


@pytest.mark.parametrize("case", list(ENC_CASES))
def test_encoder_matches_fp64_per_sample(case):
    res = _enc_case(case)
    _report(case, res)
    _assert_case(res)


@pytest.mark.parametrize("case", [c for c in ENC_CASES if c.startswith("phon")])
def test_phoneme_encoder_intermediate_gradients_are_zero_past_the_lengths(case):
    """The phoneme encoder masks only d out: the causal conv and the zero d K / d V rows must keep the padded rows of
    every gradient its backward forms (d residual, d h, dQ / dK / dV / dO, d pre, d emb) exact zeros."""
    count, bad = _enc_case(case)["intermediates"]
    print(f"\n{case}: {count} intermediate gradients checked")
    assert count >= 8 and not bad, bad[:8]


# ---- the denoiser ----
def _alone_seed(dp, dc, p):
    """A seed under which Model.forward on one sample draws (drop prompt, drop cond) = (dp, dc)."""
    for seed in range(200):
        torch.manual_seed(seed)
        a = bool(torch.zeros((1,), device="cuda").float().uniform_(0, 1) < p)
        c = bool(torch.zeros((1,), device="cuda").float().uniform_(0, 1) < p)
        if (a, c) == (dp, dc):
            return seed
    raise AssertionError("no seed draws these masks")


def _den_case(case):
    if case in _CACHE:
        return _CACHE[case]
    t0 = time.perf_counter()
    kwargs, N, lens, Lc, p = DEN_CASES[case]
    B = len(lens)
    model = build_model(kwargs, 1234, device="cuda").train()
    round_params(model)
    D, Dp = kwargs["dim"], kwargs["dim_prompt"]
    g = torch.Generator().manual_seed(60 + list(DEN_CASES).index(case))
    inp = {"x": bf(g, B, N, D), "times": torch.rand(B, generator=g).cuda(), "prompt": bf(g, B, NPAD, Dp),
           "cond": bf(g, B, Dp, Lc)}
    junk = inp["prompt"].clone()
    for b, n in enumerate(lens):
        inp["prompt"][b, n:] = float("nan")
        junk[b, n:] = JUNK * torch.randn(NPAD - n, Dp, generator=g).sign().cuda()
    d_out = bf(g, B, N, D)
    seed, dp, dc = drop_masks(B, p)
    names = [n for n, _ in model.named_parameters()]
    params = {n: prm.detach() for n, prm in model.named_parameters()}
    res = dict(family="den", lens=lens, stats={}, fails=[], checks={})

    def run(sl, n=None, s=None):
        X = {"prompt": inp["prompt"][sl, :n].clone().requires_grad_(True), "cond": inp["cond"][sl].clone().requires_grad_(True)}
        if s is not None:
            torch.manual_seed(s)
        out = model(inp["x"][sl], inp["times"][sl], **X, cond_drop_prob=p,
                    **({"prompt_lens": list(lens)} if n is None else {}))
        out.backward(d_out[sl])
        gr = {k: prm.grad for k, prm in model.named_parameters()}
        model.zero_grad(set_to_none=True)
        gr.update({"d prompt": X["prompt"].grad, "d cond": X["cond"].grad})
        return out.detach(), gr

    out, got = run(slice(None), s=seed)
    _, again = run(slice(None), s=seed)
    alone, fwd_ok = {}, True
    for b, n in enumerate(lens):
        s = None if seed is None else _alone_seed(bool(dp[b]), bool(dc[b]), p)
        ob, gb = run(slice(b, b + 1), n, s)
        fwd_ok &= torch.equal(out[b], ob[0])
        _acc(alone, gb, names)
        alone[f"d prompt {b}"], alone[f"d cond {b}"] = gb["d prompt"][0], gb["d cond"][0]
    res["checks"]["forward bit-identical to alone"] = fwd_ok
    for gr in (got, again):
        for b, n in enumerate(lens):
            gr[f"d prompt {b}"], gr[f"d cond {b}"] = gr["d prompt"][b, :n], gr["d cond"][b]
    res["checks"]["d prompt rows past the lengths are zeros"] = all(
        int((got["d prompt"][b, n:] != 0).sum()) == 0 for b, n in enumerate(lens))
    res["checks"]["d prompt of a null-substituted sample is zero"] = all(
        int((got["d prompt"][b] != 0).sum()) == 0 for b in range(B) if bool(dp[b]))
    res["dropped"] = (int(dp.sum()), int(dc.sum()))
    in_names = [f"d {k} {b}" for b in range(B) for k in ("prompt", "cond")]
    _alone_spread(res, got, again, alone, names + in_names)

    ref, ac = {}, {}
    for dst, kw in ((ref, {}), (ac, dict(autocast=True))):
        for n, idx in _groups(lens).items():
            sub = {"x": inp["x"][idx], "times": inp["times"][idx], "prompt": inp["prompt"][idx, :n],
                   "cond": inp["cond"][idx]}
            gr = port_grads(params, kwargs, sub, (dp[idx], dc[idx]), d_out[idx], **kw)
            _acc(dst, gr, names)
            for i, b in enumerate(idx):
                dst[f"d prompt {b}"], dst[f"d cond {b}"] = gr["d prompt"][i].double(), gr["d cond"][i].double()
    _against(res, got, ref, ac, names + in_names)
    keep = ("perceiver_resampler.latents", "perceiver_resampler.layers.0.0.to_kv.weight", "to_prompt_cond.1.weight")
    res.update(kwargs=kwargs, params=params, inp=inp, junk=junk, d_out=d_out, drop=(dp, dc),
               ours={n: got[n].clone() for n in keep + tuple(f"d prompt {b}" for b in range(B))})
    del got, again, alone, ref, ac, model
    torch.cuda.empty_cache()
    res["seconds"] = time.perf_counter() - t0
    _CACHE[case] = res
    return res


@pytest.mark.parametrize("case", list(DEN_CASES))
def test_model_prompt_lens_matches_fp64_per_sample(case):
    res = _den_case(case)
    _report(case, res)
    if DEN_CASES[case][4] > 0:
        print(f"  dropped prompts / conds: {res['dropped']} of {len(res['lens'])}")
        assert 0 < res["dropped"][0] < len(res["lens"])
    _assert_case(res)


# ---- Conditioner(mode="train") and NaturalSpeech2.forward ----
NUM_TOKENS, PITCH_BINS, L_FRAMES = 100, 256, 600
NS_NP, NS_T, NS_L = 96, 64, 128                     # NaturalSpeech2.forward: every attention within one key tile
NS_LENS, NS_PHON_LENS = (96, 1, 63, 64, 65, 40, 95, 64), (64, 1, 33, 63, 17, 40, 64, 5)
NS_COND_BOUND = ENCODERS.ceiling   # the conditioner behind the denoiser: see the docstring of the test below


def _cond_inputs(prompt_lens=LENS, phon_lens=PHON_LENS, Np=NPAD, T=NPAD, L=L_FRAMES):
    """Prompts (NaN past prompt_lens), ids (tokens of the upper half past phoneme_lens), durations 0-2 (zero past
    phoneme_lens) and frame-level pitch at the centre of a coarse bin per phoneme, a quarter of the frames unvoiced."""
    rng = np.random.default_rng(11)
    B = len(prompt_lens)
    g = torch.Generator().manual_seed(12)
    prompt = bf(g, B, Np, 128)
    for b, n in enumerate(prompt_lens):
        prompt[b, n:] = float("nan")
    text = rng.integers(0, NUM_TOKENS // 2, (B, T))
    dur = rng.choice(3, (B, T), p=(0.1, 0.45, 0.45))
    for b, t in enumerate(phon_lens):
        text[b, t:] = rng.integers(NUM_TOKENS // 2, NUM_TOKENS, T - t)
        dur[b, t:] = 0
    dur[:, 0] = np.maximum(dur[:, 0], 1)
    mel_min, mel_max = 1127 * np.log(1 + 50 / 700), 1127 * np.log(1 + 1100 / 700)
    bins = rng.integers(2, PITCH_BINS - 1, (B, T))
    f0 = np.round(700 * (np.exp(((bins - 1) * (mel_max - mel_min) / (PITCH_BINS - 2) + mel_min) / 1127) - 1))
    pitch = np.full((B, L), 150.0)
    for b in range(B):
        end = np.cumsum(dur[b])
        for t in range(T):
            s, e = end[t] - dur[b, t], end[t]
            pitch[b, s:e] = f0[b, t] * (rng.random(e - s) > 0.25)
            pitch[b, s:e][:1] = f0[b, t]
    return prompt, text, dur, pitch, bins


def _conditioner():
    from naturalspeech2_pytorch_b200.encoders import Conditioner
    net = Conditioner(dim_codebook=128, num_phoneme_tokens=NUM_TOKENS)
    fill_module(net, 1234)
    net.cuda()
    round_params(net)
    return net.train()


def _cond_case():
    if "conditioner" in _CACHE:
        return _CACHE["conditioner"]
    t0 = time.perf_counter()
    net = _conditioner()
    prompt, text_np, dur, pitch_np, bins = _cond_inputs()
    B = len(LENS)
    text, duration, pitch = (torch.from_numpy(a).cuda() for a in (text_np, dur, pitch_np.astype(np.float32)))
    g = torch.Generator().manual_seed(13)
    up = {"out prompt_enc": bf(g, B, NPAD, 512), "out cond": bf(g, B, 512, L_FRAMES)}
    names = [n for n, _ in net.named_parameters() if not n.startswith("duration_pitch.")]
    res = dict(family="enc", stats={}, fails=[], checks={})

    def run(sl, n=None, t=None):
        kw = dict(prompt_lens=list(LENS), phoneme_lens=list(PHON_LENS)) if n is None else {}
        pe, cond = net(prompt=prompt[sl, :n], text=text[sl, :t], duration=duration[sl, :t], pitch=pitch[sl],
                       mode="train", **kw)
        torch.autograd.backward([pe, cond], [up["out prompt_enc"][sl, :n], up["out cond"][sl]])
        gr = {k: p.grad for k, p in net.named_parameters()}
        net.zero_grad(set_to_none=True)
        return pe.detach(), cond.detach(), gr

    pe, cond, got = run(slice(None))
    _, _, again = run(slice(None))
    alone, fwd_ok, pad_ok = {}, True, True
    for b, (n, t) in enumerate(zip(LENS, PHON_LENS)):
        pa, ca, gb = run(slice(b, b + 1), n, t)
        fwd_ok &= torch.equal(pe[b, :n], pa[0]) and torch.equal(cond[b], ca[0])
        pad_ok &= int((pe[b, n:] != 0).sum()) == 0
        _acc(alone, gb, names)
    res["checks"].update({"forward bit-identical to alone": fwd_ok, "padded output rows are zeros": pad_ok})
    res["checks"]["no duration / pitch predictor gradient"] = all(
        got[n] is None for n in got if n.startswith("duration_pitch."))
    _alone_spread(res, got, again, alone, names)

    # reference operands per sample, from the restatements
    params = {n: p.detach() for n, p in net.named_parameters() if not n.startswith("duration_pitch.")}
    used = torch.zeros(PITCH_BINS, dtype=torch.bool)
    ref, ac = {}, {}
    for b, (n, t) in enumerate(zip(LENS, PHON_LENS)):
        d = dur[b:b + 1, :t]
        end = np.cumsum(d[0])
        ph = np.array([[(lambda v: v[v != 0].mean() if (v != 0).any() else 0.0)(pitch_np[b, end[i] - d[0, i]:end[i]])
                        for i in range(t)]])
        coarse = eo.f0_to_coarse(torch.from_numpy(ph).float()).long()
        assert torch.equal(coarse[torch.from_numpy(d > 0)], torch.from_numpy(bins[b:b + 1, :t][d > 0]))
        used[coarse[torch.from_numpy(d > 0)]] = True
        mask = eo.generate_mask_from_repeats(torch.from_numpy(d))
        mask = F.pad(mask, (0, L_FRAMES - mask.shape[-1])).cuda()
        fwd = conditioner_fwd(prompt[b:b + 1, :n], text[b:b + 1, :t], mask, F.one_hot(coarse, PITCH_BINS).cuda())
        d_outs = {"out prompt_enc": up["out prompt_enc"][b:b + 1, :n], "out cond": up["out cond"][b:b + 1]}
        for dst, autocast in ((ref, False), (ac, True)):
            _acc(dst, autograd(fwd, params, d_outs, autocast=autocast, only=names, cudnn="twin"), names)
    _against(res, got, ref, ac, names)
    res["checks"]["pitch rows without a valid frame are zeros"] = (
        int((got["pitch_emb.weight"].cpu()[~used] != 0).sum()) == 0 and 0 < int(used.sum()) < PITCH_BINS)
    res["checks"]["token rows only padded ids reach are zeros"] = int(
        (got["phoneme_enc.token_emb.weight"][NUM_TOKENS // 2:] != 0).sum()) == 0
    del got, again, alone, ref, ac, net
    torch.cuda.empty_cache()
    res["seconds"] = time.perf_counter() - t0
    _CACHE["conditioner"] = res
    return res


def test_conditioner_train_matches_fp64_per_sample():
    res = _cond_case()
    _report("conditioner", res)
    _assert_case(res)


def test_natural_speech2_forward_gradients_are_the_scaled_alone_gradients(monkeypatch):
    """loss = mean_b(mse_b) mean_b(w_b): d loss / d mse_b = mean(w) / B for every b, so each parameter gradient is
    (mean(w) / B) sum_b g_b / w_b.  The alone calls start from that d mse_b (see the module docstring).  Every
    attention here fits one key tile (96 prompt frames, 32 + 96 perceiver keys, 64 phonemes, 128 frames).  The
    denoiser's parameter gradients must match within RTOL.  Its d prompt and d cond match the alone ones only to fp32
    rounding (test_ragged_training_gpu.py), and the encoders' backward starts by casting them to bf16: a rounding that
    moves there changes the bf16 roundings after it, so the conditioner's gradients differ at the level of bf16 rounding
    noise and are bounded by the float64 comparisons' ceiling, NS_COND_BOUND."""
    from naturalspeech2_pytorch_b200 import Model, NaturalSpeech2, training
    from naturalspeech2_pytorch_b200.diffusion import gamma_to_alpha_sigma
    t0 = time.perf_counter()
    cn = _conditioner()
    torch.manual_seed(0)
    model = Model(dim=128, depth=2, heads=2, wavenet_layers=2, wavenet_stacks=1, dim_prompt=512,
                  condition_on_prompt=True, cond_drop_prob=0.0).cuda().train()
    ns = NaturalSpeech2(model, target_sample_hz=24000, timesteps=3, conditioner=cn)
    prompt, text_np, dur, pitch_np, _ = _cond_inputs(NS_LENS, NS_PHON_LENS, NS_NP, NS_T, NS_L)
    text, duration, pitch = (torch.from_numpy(a).cuda() for a in (text_np, dur, pitch_np.astype(np.float32)))
    B = len(NS_LENS)
    rows = []
    mse_apply = training.MseRowsFunction.apply

    def spy(pred, target):
        r = mse_apply(pred, target)
        rows.append(r)
        return r
    monkeypatch.setattr(training.MseRowsFunction, "apply", spy)
    g = torch.Generator(device="cuda").manual_seed(9)
    audio = torch.randn(B, NS_L, 128, device="cuda", generator=g)
    times = torch.rand(B, device="cuda", generator=g)
    noise = torch.randn(B, NS_L, 128, device="cuda", generator=g)
    mods = {"conditioner": cn, "model": model}
    named = [(f"{k}.{n}", p) for k, m in mods.items() for n, p in m.named_parameters()
             if not n.startswith("duration_pitch.")]

    def grads():
        out = {n: p.grad for n, p in named}
        cn.zero_grad(set_to_none=True)
        model.zero_grad(set_to_none=True)
        return out

    d_rows = []
    loss = ns(audio, text=text, prompt=prompt, duration=duration, pitch=pitch, times=times, noise=noise,
              prompt_lens=list(NS_LENS), phoneme_lens=list(NS_PHON_LENS))
    rows[-1].register_hook(lambda gr: d_rows.append(gr.clone()))
    loss.backward()
    got = grads()
    missing = [n for n, gr in got.items() if gr is None]
    assert not missing, f"parameters without a gradient: {missing[:8]}"
    assert all(bool(torch.isfinite(gr).all()) for gr in got.values())
    alpha, sigma = gamma_to_alpha_sigma(ns.gamma_schedule(times), ns.scale)
    snr = (alpha * alpha) / (sigma * sigma)
    w = snr.clamp(max=ns.min_snr_gamma) / (snr + 1) if ns.min_snr_loss_weight else snr / (snr + 1)
    c = d_rows[0]
    want_c = w.double().mean() / B
    assert float((c.double() - want_c).abs().max()) <= 1e-6 * float(want_c), (c, want_c)
    alone = {}
    for b, (n, t) in enumerate(zip(NS_LENS, NS_PHON_LENS)):
        ns(audio[b:b + 1], text=text[b:b + 1, :t], prompt=prompt[b:b + 1, :n], duration=duration[b:b + 1, :t],
           pitch=pitch[b:b + 1], times=times[b:b + 1], noise=noise[b:b + 1])
        torch.autograd.backward(rows[-1], c[b:b + 1])      # = g_b / w_b x mean(w) / B, with the batch's roundings
        _acc(alone, grads(), [k for k, _ in named])
    errs = {n: _err(got[n], alone[n]) for n in alone}
    assert set(errs) == set(got)
    worst = {m: max(((e, n) for n, e in errs.items() if n.startswith(m + ".")), default=(0.0, None)) for m in mods}
    print(f"\nNaturalSpeech2.forward: {len(errs)} parameter gradients against (mean(w) / B) sum_b g_b / w_b in "
          f"{time.perf_counter() - t0:.1f} s; worst " + ", ".join(f"{m} {e:.2e} ({n})" for m, (e, n) in worst.items()))
    bad = [(n, e) for n, e in errs.items() if e > (RTOL if n.startswith("model.") else NS_COND_BOUND)]
    assert not bad, bad[:8]


# ---- cases reach the tile edges ----
def test_cases_reach_the_key_and_query_tile_edges():
    """A key tile skipped by the early exit (start >= length), a last valid key tile other than tile 0, more than one
    64-query tile, lengths 1 / 63-65 / 127-129 / full, a repeated length; for the perceiver M + length on 128 / 129."""
    BKV, BQ = 128, 64
    for name, (_, lens) in ENC_CASES.items():
        tiles = -(-NPAD // BKV)
        assert any(tiles - (-(-n // BKV)) >= 2 for n in lens), name
        assert any((n - 1) // BKV >= 1 and n < NPAD for n in lens), name
        assert NPAD > BQ and len(set(lens)) < len(lens), name
        assert {1, 63, 64, 65, 127, 128, 129, NPAD} <= set(lens) or name == "spe_k11", name
    assert {1, 2, 4} <= set(LENS_K11) and CONFIGS["spe_k11"][1]["kernel_size"] // 2 == 5
    keys = [32 + n for n in BENCH_LENS]
    assert {33, 128, 129, 256, 332} <= set(keys)
    for name, (kw, _, lens, _, _) in DEN_CASES.items():
        M = kw.get("num_latents_m", 32)
        kv = [M + n for n in lens]
        assert any(-(-(M + NPAD) // BKV) - (-(-k // BKV)) >= 1 for k in kv), name
        assert any((k - 1) // BKV >= 1 for k in kv), name
    with_proj = {n for n, (kw, *_) in DEN_CASES.items() if kw["dim_prompt"] != kw["dim"]}
    assert with_proj and with_proj != set(DEN_CASES)


# ---- wrong references: the same bounds must reject them ----
def _assert_rejected(res, wrong, names):
    return assert_rejected(res["ours"], wrong, res["stats"], names, FAMILY[res["family"]], EITHER)[0]


def _wrong_port(res, names, perceiver_rows, mean_rows):
    """The denoiser's fp64 reference where the perceiver sees `perceiver_rows(b, n)` prompt rows and the mean-pool
    `mean_rows(b, n)` rows (rows past n: the junk of the padded prompt, or zeros)."""
    lens, inp = res["lens"], res["inp"]
    dp, dc = res["drop"]
    tot = {}
    orig = tp.perceiver_resampler
    for b, n in enumerate(lens):
        kp, km = perceiver_rows(n), mean_rows(n)
        full = res["junk"][b:b + 1, :max(kp, km)].clone()
        if km > n:
            full[:, n:] = 0
        sub = {"x": inp["x"][b:b + 1], "times": inp["times"][b:b + 1], "prompt": full[:, :km], "cond": inp["cond"][b:b + 1]}
        jrows = res["junk"][b:b + 1, n:kp].double()

        def perceiver(P, cfg, prompt, n=n, jrows=jrows):
            return orig(P, cfg, torch.cat((prompt[:, :n], jrows.to(prompt.dtype)), 1))
        tp.perceiver_resampler = perceiver
        try:
            gr = port_grads(res["params"], res["kwargs"], sub, (dp[b:b + 1], dc[b:b + 1]), res["d_out"][b:b + 1],
                             only=[k for k in names if not k.startswith("d ")] + ["d prompt"])
        finally:
            tp.perceiver_resampler = orig
        _acc(tot, gr, [k for k in names if not k.startswith("d ")])
        tot[f"d prompt {b}"] = gr["d prompt"][0, :n]
    return tot


def _target_sample(lens):
    """The sample with the longest prompt short of the padded length (the smallest effect of a length error)."""
    return max((b for b, n in enumerate(lens) if n < NPAD), key=lambda b: lens[b])


def test_rejects_perceiver_attending_one_padded_row():
    res = _den_case("bench")
    b = _target_sample(res["lens"])
    names = ["perceiver_resampler.latents", "perceiver_resampler.layers.0.0.to_kv.weight", f"d prompt {b}"]
    wrong = _wrong_port(res, names, lambda n: min(n + 1, NPAD), lambda n: n)
    print(f"\nperceiver over M + length + 1 keys: smallest margin {_assert_rejected(res, wrong, names):.1f}x")


def test_rejects_mean_pool_over_the_padded_length():
    res = _den_case("bench")
    b = _target_sample(res["lens"])
    names = ["to_prompt_cond.1.weight", f"d prompt {b}"]
    wrong = _wrong_port(res, names, lambda n: n, lambda n: NPAD)
    print(f"\nmean-pool divided by Np: smallest margin {_assert_rejected(res, wrong, names):.1f}x")


def test_rejects_same_conv_reading_the_first_padded_rows():
    """spe_k11: the k = 11 convs read the first five padded rows (junk) instead of zeros."""
    res = _enc_case("spe_k11")
    lens, k, pad = res["lens"], CONFIGS["spe_k11"][1]["kernel_size"], res["padding"]
    b = _target_sample(lens)
    names = ["conv.1.weight", "conv.3.weight", f"x {b}"]
    wrong = {}
    for n, idx in _groups(lens).items():
        ext = min(n + pad, NPAD)
        xs = res["junk"][idx, :ext]

        def fwd(P, dtype, n=n):
            h = P["x"].to(dtype).transpose(1, 2)
            for i in (1, 3):
                h = F.silu(F.conv1d(h, P[f"conv.{i}.weight"], P[f"conv.{i}.bias"], padding=k // 2))
            return {"encoding": eo.transformer(h.transpose(1, 2)[:, :n], P, "transformer.", res["heads"])}
        up = res["up"][idx, :n]
        gr = autograd(fwd, dict(res["params"], x=xs), {"encoding": up}, only=names[:2] + ["x"], cudnn="twin")
        _acc(wrong, gr, names[:2])
        for i, s in enumerate(idx):
            wrong[f"x {s}"] = gr["x"][i, :n]
    print(f"\nspe_k11 convs reading padded rows: smallest margin {_assert_rejected(res, wrong, names):.1f}x")


def test_rejects_phoneme_attention_with_one_padded_token():
    """phon_default: the self-attention of every sample shorter than the padding also attends to its first padded
    token (the reference runs on length + 1 tokens; the extra row's output gets no upstream gradient)."""
    res = _enc_case("phon_default")
    lens = res["lens"]
    names = ["transformer.layers.0.1.to_kv.weight", "token_emb.weight", "conv.1.weight"]
    wrong = {}
    for n, idx in _groups(lens).items():
        ext = min(n + 1, NPAD)
        up = torch.zeros(len(idx), ext, res["up"].shape[-1], device="cuda")
        up[:, :n] = res["up"][idx, :n]
        fwd = _enc_fwd("phon_default", res["x"][idx, :ext], PHON, res["heads"], None)
        _acc(wrong, autograd(fwd, res["params"], {"encoding": up}, only=names, cudnn="twin"), names)
    print(f"\nphoneme attention with one padded token: smallest margin {_assert_rejected(res, wrong, names):.1f}x")
