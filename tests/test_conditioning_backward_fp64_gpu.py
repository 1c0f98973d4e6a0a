"""GPU: the conditioning front end's hand-written backward (`encoders._EncoderFunction` for `SpeechPromptEncoder` and
`PhonemeEncoder`, `_ExpandFunction` / `ops.expand_encodings_bwd` for the pitch table) against float64 autograd on the
GPU at the encoders' default dims: the prompt encoder's eight k=9 convs 128 -> 256 -> 2048 x4 -> 512 x3, and both
encoders' depth-6, dim-512, 8-head transformer with the 1365-wide GEGLU (padded to 1408 in the packs).

The reference is built only from the restatements pinned to the reference modules: `oracle.encoders_oracle`
(speech_prompt_encoder, phoneme_encoder, generate_mask_from_repeats, f0_to_coarse; tests/test_encoders_cpu.py) and, with
dropout, tests/dropout_oracle.py with the masks of the seed the call drew.  Both sides see the same operands: every
parameter is rounded to bf16 in place (the packs hold exactly the parameters), and prompts and upstream gradients are
bf16-representable (`_start_backward` casts d out to bf16).  The fp64 reference runs with cuDNN off, so a conv tap that
only reads the zero padding gets an exactly zero gradient whatever algorithm cuDNN would pick.  The output and every
parameter gradient are compared whole, with the encoders' family of tests/fp64_check.py:
  (i)  rel-L2 <= C x the rel-L2 of the same restatement in fp32 under torch.autocast("cuda", bfloat16) (the
       reference's own reduced-precision mode, same rounded operands) + floor;
  (ii) rel-L2 <= ceiling;
every element whose fp64 value is exactly zero must be exactly zero in ours, and nothing may be non-finite.  Five
deliberately wrong references (reversed conv taps, a causal conv one frame off, one tile of d out rows missing, the
dropout masks of another seed, one phoneme's frames given to its neighbour) must be rejected by the same bounds.

to_q has its own bound, because of one rounding choice.  The attention backward (csrc/attn_bwd.cu) forms
dS = P (dP - D) with D = rowsum(dO * O) taken from the bf16 attention output, as FlashAttention-2 does.  The rounding
error of D is the same for every key of a query row, so dQ = dS K picks up that error times the attention-weighted mean
key, and the keys' shared component does not cancel.  With these weights the attention of layers 1-5 is nearly flat:
the exact to_q gradient there is ~1e-5 of to_kv's, below that error.  An fp64 restatement that rounds only O and dO to
bf16 inside D reproduces the effect (prompt encoder, B 2, N 103, layer 5: rel-L2 176 against exact fp64).  The
autocast-bf16 twin uses plain softmax autograd, whose D comes from the same dP it is subtracted from.  So to_q's
rel-L2 is not compared with its twin (ours is 1e1-1e2 rel-L2 where the twin is 0.1-0.8).  Its error is bounded
instead relative to the gradient of the fused q / kv projection that one wgrad produces: TO_Q_BOUND, and here a
self-attention to_q is judged by that share alone (fp64_check.SHARE_ONLY).

Measured on an H100 80GB HBM3 (700 W power limit).  Worst tensor per case (to_q aside), rel-L2 ours / autocast-bf16
of the same tensor; the largest ours / autocast-bf16 ratio of the case; to_q's worst error as a share of the q / kv
gradient:
  P_bench  prompt, B 4, N 103          conv.1.weight                   1.38e-2 / 1.29e-2   1.15   1.85e-3
  P_long   prompt, B 2, N 300          conv.1.weight                   1.50e-2 / 1.20e-2   1.25   2.03e-3
  P_short  prompt, B 3, N 3            conv.1.weight                   1.08e-2 / 1.26e-2   1.00   2.39e-3
  P_drop   prompt, dropout 0.2         conv.1.weight                   1.21e-2 / 1.17e-2   1.20   1.60e-3
  T_main   phoneme, B 4, T 100         transformer.layers.5.2.gamma    7.8e-3 / 9.4e-3     1.07   2.00e-3
  T_short  phoneme, B 3, T 5           transformer.layers.0.0.gamma    8.0e-3 / 8.7e-3     1.14   2.28e-3
  T_drop   phoneme, conv dropout 0.2   conv.1.weight                   7.3e-3 / 8.0e-3     1.17   1.97e-3
  C_train  Conditioner                 prompt_enc.conv.1.weight        1.28e-2 / 1.17e-2   1.18   2.01e-3
The worst ratio, 1.25, is the first conv's weight at P_long.  That conv's input gradient is the bf16 d pre of
`_conv_silu_backward`, which recomputes the SiLU pre-activation in bf16.  Against the bounds below the tightest
tensor uses 75 % of its bound (P_long conv.1.weight, at 1.5 x autocast + floor), and to_q uses 80 % (P_short).  The
wrong references sit at rel-L2 0.16-0.65 (reversed taps), 0.11-0.12 (conv one frame off), 0.36 (row tile), 0.08-0.12
on to_kv and 0.42 on conv.1 (masks of seed + 1), and 0.22 on pitch_emb / 0.030 on token_emb (phoneme given to its
neighbour, the smallest margin: 1.9x its bound).  The whole module takes ~35 s.
"""
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from fp64_check import ENCODERS, SHARE_ONLY, assert_rejected, autograd, bf, bound, compare, over, round_params
from helpers import build_encoder
from oracle import encoders_oracle as eo
from param_fill import fill_module
from restatements import (DEPTH, DIM, DROP_P, HEADS, conditioner_fwd, drawn_seed, encoder_fwd,
                          encoder_masks)

pytestmark = pytest.mark.gpu

SPE = ("SpeechPromptEncoder", {"dim_codebook": 128})
PHON = ("PhonemeEncoder", {"num_tokens": 100})
CASES = {
    # name: (encoder, B, length, train_dropout, phoneme lengths (the rest of a row is -1 padding))
    "P_bench": (SPE, 4, 103, False, None),
    "P_long": (SPE, 2, 300, False, None),
    "P_short": (SPE, 3, 3, False, None),
    "P_drop": (SPE, 2, 103, True, None),
    "T_main": (PHON, 4, 100, False, (100, 93, 64, 37)),
    "T_short": (PHON, 3, 5, False, (5, 5, 3)),
    "T_drop": (PHON, 2, 100, True, (100, 81)),
    "C_train": (None, 2, 103, False, None),        # Conditioner: B 2, Np 103, T 40, L 300
}
TORCH_SEED = {"P_drop": 1002, "T_drop": 1003}     # torch.manual_seed before the call that draws the dropout seed
NUM_TOKENS, PITCH_BINS = 100, 256
T_TEXT, L_FRAMES = 40, 300
SPE_CONVS = [f"conv.{2 * i + 1}.weight" for i in range(8)]
# gradients kept after a case for the sensitivity tests
KEEP = ("conv.1.weight", "conv.5.weight", "token_emb.weight", "transformer.layers.5.3.2.weight", "pitch_emb.weight",
        "phoneme_enc.token_emb.weight", *(f"transformer.layers.{l}.1.{w}.weight" for l in range(DEPTH)
                                           for w in ("to_q", "to_kv")))


def _is_q(name):
    return name.endswith(".1.to_q.weight")


def _ids(g, B, T, lengths):
    """Ids from the lower half of the table, every fifth one repeated in the next position, -1 past each length."""
    ids = torch.randint(0, NUM_TOKENS // 2, (B, T), generator=g)
    ids[:, 1::5] = ids[:, 0::5][:, :ids[:, 1::5].shape[1]]
    for b, n in enumerate(lengths):
        ids[b, n:] = -1
    return ids.cuda()


# ---- one run per case ----
_CACHE = {}


def _encoder_run(name):
    (cls, kw), B, N, drop, lengths = CASES[name]
    enc = build_encoder(cls, kw, seed=1234, device="cuda")
    round_params(enc)
    enc.train()
    enc.train_dropout = drop
    assert (enc.heads, len(enc.transformer.layers)) == (HEADS, DEPTH)
    if drop:
        assert (enc.attn_dropout, enc.conv_dropout) == ((DROP_P, 0.0) if cls == SPE[0] else (0.0, DROP_P))
    g = torch.Generator().manual_seed(20)
    x = bf(g, B, N, kw["dim_codebook"]) if cls == SPE[0] else _ids(g, B, N, lengths)
    d_outs = {"out": bf(g, B, N, DIM)}

    # ours: out.backward(d out) through _EncoderFunction
    if drop:
        torch.manual_seed(TORCH_SEED[name])
    out = enc(x)
    out.backward(d_outs["out"])
    seed = drawn_seed(TORCH_SEED[name]) if drop else None
    ours = {n: p.grad for n, p in enc.named_parameters()}
    ours["out"] = out.detach()
    params = {n: p.detach() for n, p in enc.named_parameters()}
    assert set(params) == set(enc.state_dict())
    ctx = dict(cls=cls, x=x, seed=seed, B=B, N=N)
    return ours, params, d_outs, encoder_fwd(cls, x, encoder_masks(cls, seed, B, N)), ctx, enc


def _conditioner_inputs():
    """Durations (with zeros; sample 0 fills L, sample 1 ends short of it and has a -1 text tail), ids and frame-level
    pitch.  Every phoneme with frames gets its own coarse-pitch bin, and no phoneme has more than 32 frames."""
    rng = np.random.default_rng(7)
    B = CASES["C_train"][1]
    dur = np.zeros((B, T_TEXT), dtype=np.int64)
    text = rng.integers(0, NUM_TOKENS, (B, T_TEXT))
    text[1, -4:] = -1
    for b, total in enumerate((L_FRAMES, 263)):
        d = rng.integers(1, 13, T_TEXT)
        d[rng.choice(T_TEXT - 4, 5, replace=False)] = 0
        if b == 1:
            d[-4:] = 0
        while d.sum() != total:
            i = rng.integers(T_TEXT)
            if d.sum() < total and 0 < d[i] < 32:
                d[i] += 1
            elif d.sum() > total and d[i] > 1:
                d[i] -= 1
        dur[b] = d
    # f0 at the centre of a distinct coarse bin (2 ... 254) per phoneme, rounded to whole Hz (< 0.2 bin off centre)
    mel_min, mel_max = 1127 * np.log(1 + 50 / 700), 1127 * np.log(1 + 1100 / 700)
    bins = rng.permutation(np.arange(2, PITCH_BINS - 1))[:B * T_TEXT].reshape(B, T_TEXT)
    f0 = np.round(700 * (np.exp(((bins - 1) * (mel_max - mel_min) / (PITCH_BINS - 2) + mel_min) / 1127) - 1))
    pitch = np.full((B, L_FRAMES), 150.0)                 # frames past a sample's total duration are ignored
    for b in range(B):
        end = np.cumsum(dur[b])
        for t in range(T_TEXT):
            s, e = end[t] - dur[b, t], end[t]
            pitch[b, s:e] = f0[b, t] * (rng.random(e - s) > 0.25)      # about a quarter of the frames unvoiced
            pitch[b, s:e][:1] = f0[b, t]                                # ... but never the first
    return dur, text, pitch, bins


def _conditioner_run():
    from naturalspeech2_pytorch_b200.encoders import Conditioner
    B, Np = CASES["C_train"][1:3]
    net = Conditioner(dim_codebook=128, num_phoneme_tokens=NUM_TOKENS)
    fill_module(net, 1234)
    net.cuda()
    round_params(net)
    net.train()
    dur, text_np, pitch_np, bins = _conditioner_inputs()
    g = torch.Generator().manual_seed(20)
    prompt = bf(g, B, Np, 128)
    d_outs = {"out prompt_enc": bf(g, B, Np, DIM), "out cond": bf(g, B, DIM, L_FRAMES)}
    text, duration, pitch = (torch.from_numpy(a).cuda() for a in (text_np, dur, pitch_np.astype(np.float32)))

    # ours, twice: d cond contiguous (B, D, L), then the channel-first view of a token-major (B, L, D) buffer
    d_phon = []

    def keep_d_phon(module, inputs, out):
        out.register_hook(lambda gr: d_phon.append(gr.clone()))

    hook = net.phoneme_enc.register_forward_hook(keep_d_phon)
    runs = []
    for d_cond in (d_outs["out cond"], d_outs["out cond"].transpose(1, 2).contiguous().transpose(1, 2)):
        net.zero_grad(set_to_none=True)
        pe, cond = net(prompt=prompt, text=text, mode="train", pitch=pitch, duration=duration)
        torch.autograd.backward([pe, cond], [d_outs["out prompt_enc"], d_cond])
        runs.append(({n: p.grad for n, p in net.named_parameters()}, pe.detach(), cond.detach()))
    hook.remove()
    grads, pe, cond = runs[0]
    no_grad = [n for n, p in grads.items() if n.startswith("duration_pitch.") and p is not None]
    layout = (runs[0][0]["pitch_emb.weight"], runs[1][0]["pitch_emb.weight"], d_phon[0], d_phon[1])
    ours = {n: v for n, v in grads.items() if not n.startswith("duration_pitch.")}
    ours.update({"out prompt_enc": pe, "out cond": cond})
    params = {n: p.detach() for n, p in net.named_parameters() if not n.startswith("duration_pitch.")}

    # reference operands, built on the host from the restatements
    ph_pitch = np.zeros((B, T_TEXT))
    for b in range(B):                                   # mean of the voiced frames of each phoneme (0 if none)
        end = np.cumsum(dur[b])
        for t in range(T_TEXT):
            v = pitch_np[b, end[t] - dur[b, t]:end[t]]
            ph_pitch[b, t] = v[v != 0].mean() if (v != 0).any() else 0.0
    coarse = eo.f0_to_coarse(torch.from_numpy(ph_pitch).float()).long()
    assert torch.equal(coarse[torch.from_numpy(dur > 0)], torch.from_numpy(bins[dur > 0]))
    mask = eo.generate_mask_from_repeats(torch.from_numpy(dur))
    mask = F.pad(mask, (0, L_FRAMES - mask.shape[-1])).cuda()
    onehot = F.one_hot(coarse, PITCH_BINS).cuda()
    ctx = dict(prompt=prompt, text=text, mask=mask, onehot=onehot, dur=dur, text_np=text_np, coarse=coarse,
               no_grad=no_grad, layout=layout)
    return ours, params, d_outs, conditioner_fwd(prompt, text, mask, onehot), ctx, net


def _case(name):
    """Run one case once: our backward, the fp64 reference and the autocast-bf16 run of the restatement; per-tensor
    statistics and what the other tests read."""
    if name in _CACHE:
        return _CACHE[name]
    t0 = time.perf_counter()
    ours, params, d_outs, fwd, ctx, module = _conditioner_run() if name == "C_train" else _encoder_run(name)
    # the fp64 run without cuDNN (exact zeros for taps that only read the padding), the twin with it
    ref = autograd(fwd, params, d_outs, cudnn="twin", out_prefix="")
    ac = autograd(fwd, params, d_outs, autocast=True, cudnn="twin", out_prefix="")
    assert set(ref) == set(ours) == set(ac)
    stats, fails = {}, []
    for n, r in ref.items():
        o = ours[n]
        assert o is not None and o.shape == r.shape, n
        s = compare(o, r, ac[n], ref[n.replace("to_q", "to_kv")] if _is_q(n) else None, max_abs=True)
        if isinstance(s, str):
            fails.append((n, s))
        elif s is not None:
            stats[n] = s
    res = dict(ctx, params=params, d_outs=d_outs, fwd=fwd, stats=stats, fails=fails,
               ours={n: ours[n].clone() for n in KEEP if n in ours})
    if name == "P_short":      # taps 0, 1, 7, 8 read only the padding at N = 3; taps 2 ... 6 read the sequence
        res["taps"] = {n: (ours[n][..., [0, 1, 7, 8]].clone(), ref[n][..., [0, 1, 7, 8]].clone(),
                           bool((ours[n][..., 2:7] != 0).any()), bool((ref[n][..., 2:7] != 0).any()))
                       for n in SPE_CONVS}
    if name == "T_short":
        res["taps"] = {"conv.1.weight": (ours["conv.1.weight"].clone(), ref["conv.1.weight"].clone())}
    if name == "T_main":
        res["emb"] = (ours["token_emb.weight"].clone(), ref["token_emb.weight"].clone())
    if name == "C_train":
        res["emb"] = (ours["pitch_emb.weight"].clone(), ref["pitch_emb.weight"].clone())
    module.zero_grad(set_to_none=True)
    del ours, ref, ac, module
    torch.cuda.empty_cache()
    res["seconds"] = time.perf_counter() - t0
    _CACHE[name] = res
    return res


@pytest.mark.parametrize("name", list(CASES))
def test_backward_matches_fp64_autograd(name):
    r = _case(name)
    stats = r["stats"]
    rest = {n: s for n, s in stats.items() if not _is_q(n)}
    q = {n: s for n, s in stats.items() if _is_q(n)}
    ranked = sorted(rest.items(), key=lambda kv: kv[1].rel / bound(ENCODERS, kv[1].rel_ac), reverse=True)
    worst_rel = max(rest.items(), key=lambda kv: kv[1].rel)
    ratio = max(((n, s) for n, s in rest.items() if s.rel_ac > 0), key=lambda kv: kv[1].rel / kv[1].rel_ac)
    worst_q = max(q.items(), key=lambda kv: kv[1].share)
    print(f"\n{name}: {len(stats)} tensors compared in {r['seconds']:.1f} s; worst rel-L2 {worst_rel[0]}: "
          f"ours {worst_rel[1].rel:.3e} autocast-bf16 {worst_rel[1].rel_ac:.3e}; max ratio ours / autocast-bf16 "
          f"{ratio[1].rel / ratio[1].rel_ac:.2f} ({ratio[0]}); worst to_q {worst_q[0]}: {worst_q[1].share:.3e} of the "
          f"q / kv gradient (rel-L2 ours {worst_q[1].rel:.3e} / autocast-bf16 {worst_q[1].rel_ac:.3e})")
    for n, s in ranked[:8]:
        print(f"  {n}: rel-L2 ours {s.rel:.3e} / autocast-bf16 {s.rel_ac:.3e} (bound {bound(ENCODERS, s.rel_ac):.3e}); "
              f"max-abs ours {s.max_abs:.3e} / autocast-bf16 {s.max_abs_ac:.3e} (max |ref| {s.max_ref:.3e})")
    assert not r["fails"], f"non-finite, or non-zero where the fp64 value is exactly zero: {r['fails'][:8]}"
    bad = [(n, s.rel, s.rel_ac, s.share) for n, s in stats.items() if over(ENCODERS, s, SHARE_ONLY)]
    assert not bad, f"{len(bad)} tensors over the bound (name, rel-L2, autocast rel-L2, to_q share): {bad[:8]}"


# ---- exact zeros ----
def test_short_prompt_conv_taps_beyond_the_sequence_are_exact_zeros():
    """N = 3 < the k=9 half-width: tap t reads x[n + t - 4], so taps 0, 1, 7, 8 of all eight convs only read padding."""
    r = _case("P_short")
    assert sorted(r["taps"]) == sorted(SPE_CONVS)
    for n, (o, ref, o_inner, ref_inner) in r["taps"].items():
        assert float(ref.abs().max()) == 0.0 and ref_inner, n
        assert int((o != 0).sum()) == 0 and o_inner, (n, float(o.abs().max()))


def test_short_text_causal_taps_before_the_sequence_are_exact_zeros():
    """T = 5: causal tap t reads x[n - (8 - t)], so taps 0 ... 3 only read the left padding."""
    o, ref = _case("T_short")["taps"]["conv.1.weight"]
    assert float(ref[..., :4].abs().max()) == 0.0 and float(ref[..., 4:].abs().min()) > 0
    assert int((o[..., :4] != 0).sum()) == 0 and bool((o[..., 4:] != 0).any())


def test_token_rows_that_never_occur_are_exact_zeros_and_the_pad_row_is_trained():
    r = _case("T_main")
    o, ref = r["emb"]
    used = torch.zeros(NUM_TOKENS + 1, dtype=torch.bool)
    used[r["x"].masked_fill(r["x"] < 0, NUM_TOKENS).flatten().cpu()] = True
    assert used[NUM_TOKENS] and not bool(used[NUM_TOKENS // 2:NUM_TOKENS].any())
    for g in (o.cpu(), ref.cpu()):
        assert int((g[~used] != 0).sum()) == 0
        assert bool((g[used].abs().sum(-1) > 0).all())


def test_conditioner_pitch_rows_without_frames_are_exact_zeros():
    r = _case("C_train")
    o, ref = r["emb"]
    used = torch.zeros(PITCH_BINS, dtype=torch.bool)
    used[r["coarse"][torch.from_numpy(r["dur"] > 0)]] = True
    assert 0 < int(used.sum()) < PITCH_BINS
    for g in (o.cpu(), ref.cpu()):
        assert int((g[~used] != 0).sum()) == 0
        assert bool((g[used].abs().sum(-1) > 0).all())


def test_conditioner_duration_predictor_gets_no_gradient():
    assert _case("C_train")["no_grad"] == []


def test_conditioner_token_major_d_cond_gives_bit_identical_gradients():
    """d cond as a contiguous (B, D, L) tensor and as the channel-first view of a token-major (B, L, D) buffer (what
    DenoiserFunction hands over) give the same pitch-table gradient and the same gradient into the phoneme encodings.
    The scatter accumulates with fp32 atomics; here every phoneme has at most 32 frames (at most two 32-frame blocks)
    and its own pitch bin, so each element sums at most two terms and its value does not depend on their order."""
    t0, t1, p0, p1 = _case("C_train")["layout"]
    assert torch.equal(t0, t1) and torch.equal(p0, p1)
    assert bool((t0 != 0).any()) and bool((p0 != 0).any())


# ---- sensitivity: wrong references must fail the same bounds ----
def _assert_rejected(r, wrong, names, at_least=None):
    """The bounds of test_backward_matches_fp64_autograd must reject `wrong` for every name, or for `at_least`."""
    assert_rejected(r["ours"], wrong, r["stats"], names, ENCODERS, SHARE_ONLY, at_least=at_least)


def test_rejects_reference_with_reversed_conv_taps():
    """conv.5 (2048 -> 2048) with its taps reversed: a mirrored shift sign in one conv's wgrad or dgrad."""
    r = _case("P_bench")
    base = r["fwd"]

    def fwd(P, dtype):
        return base(dict(P, **{"conv.5.weight": P["conv.5.weight"].flip(-1)}), dtype)
    names = ["conv.5.weight", "conv.1.weight"]
    _assert_rejected(r, autograd(fwd, r["params"], r["d_outs"], only=names, cudnn="twin"), names)


def test_rejects_reference_with_causal_conv_one_frame_off():
    """The phoneme encoder's causal conv padded (7, 1) instead of (8, 0)."""
    r = _case("T_main")

    def shifted(P, ids):
        ids = ids.masked_fill(ids < 0, P["token_emb.weight"].shape[0] - 1)
        h = P["token_emb.weight"][ids].transpose(1, 2)
        h = F.silu(F.conv1d(F.pad(h, (7, 1)), P["conv.1.weight"], P["conv.1.bias"]))
        return eo.transformer(h.transpose(1, 2), P, "transformer.", HEADS)
    names = ["conv.1.weight", "token_emb.weight"]
    fwd = encoder_fwd(r["cls"], r["x"], (None, None), phoneme_encoder=shifted)
    _assert_rejected(r, autograd(fwd, r["params"], r["d_outs"], only=names, cudnn="twin"), names)


def test_rejects_reference_with_one_row_tile_missing():
    """P_long's d out with the last 64 rows of sample 0 zeroed."""
    r = _case("P_long")
    d_out = r["d_outs"]["out"].clone()
    d_out[0, -64:] = 0
    names = ["transformer.layers.5.3.2.weight", "conv.1.weight"]
    _assert_rejected(r, autograd(r["fwd"], r["params"], {"out": d_out}, only=names, cudnn="twin"), names)


def test_rejects_reference_with_masks_of_another_seed():
    """P_drop's attention masks drawn from seed + 1."""
    r = _case("P_drop")
    fwd = encoder_fwd(r["cls"], r["x"], encoder_masks(r["cls"], r["seed"] + 1, r["B"], r["N"]))
    attn = [f"transformer.layers.{l}.1.{w}.weight" for l in range(DEPTH) for w in ("to_q", "to_kv")]
    wrong = autograd(fwd, r["params"], r["d_outs"], only=attn + ["conv.1.weight"], cudnn="twin")
    _assert_rejected(r, wrong, ["conv.1.weight"])
    _assert_rejected(r, wrong, attn, at_least=1)


def test_rejects_reference_with_one_phoneme_given_to_its_neighbour():
    """C_train with the frames of sample 0's longest phoneme attributed to the next one (whose id differs)."""
    r = _case("C_train")
    dur, text = r["dur"], r["text_np"]
    j = max((t for t in range(T_TEXT - 1) if dur[0, t + 1] > 0 and text[0, t] != text[0, t + 1]),
            key=lambda t: dur[0, t])
    mask = r["mask"].clone()
    mask[0, j + 1] |= mask[0, j]
    mask[0, j] = False
    fwd = conditioner_fwd(r["prompt"], r["text"], mask, r["onehot"])
    names = ["pitch_emb.weight", "phoneme_enc.token_emb.weight"]
    _assert_rejected(r, autograd(fwd, r["params"], r["d_outs"], only=names, cudnn="twin"), names)
