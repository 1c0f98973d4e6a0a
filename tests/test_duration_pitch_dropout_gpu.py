"""GPU: the duration / pitch predictor trained with the reference's dropout (`train_dropout=True`): p = `dropout` (0.2
by default) on the softmax probabilities of every layer's cross attention.  The reference's Blocks keep p = 0
(tests/test_duration_pitch_dropout_cpu.py reads that from the reference module), so nothing else is dropped.

The reference is `restatements.masked_trunk`, oracle.encoders_oracle._trunk with each layer's attention mask applied after its
softmax (attend.py:149), built from tests/dropout_oracle.py with the sites of the predictor's docstring and the seed the
call drew (re-drawn with torch.manual_seed).  At the reference's default dims (dim 512, depth 10, 8 heads, both
trunks) the GPU output, every parameter gradient, d x and d prompts are compared with fp64 autograd of it, with the
bounds of tests/test_encoder_dropout_training_gpu.py: gradient norms within 2 %, rel-L2 < max(3 %, 2 x the same
tensor's error without dropout) and cos > min(0.9995, 1 - 2 (1 - cos without dropout)).  As in
tests/test_duration_pitch_backward_fp64_gpu.py the parameters are bf16 values and the head biases are set from the fp64
pre-activations (masked and unmasked) so that no ReLU row lies within the forward error of 0.  Three wrong references
must fail the same bounds: the trunks' sites swapped, every attention mask taken from the next site, and p also drawn
after every Block's SiLU (dropout the reference does not apply there).

Measured on an H100 80GB HBM3 (700 W power limit), tightest tensor per case, rel-L2 with / without dropout:
  main  p 0.2   to_pitch_pred.layers.9.2.to_q.weight             1.15e-2 / 1.19e-2
  main  p 0.5   to_pitch_pred.layers.9.0.2.blocks.1.proj.bias    9.2e-3 / 6.8e-3
  short p 0.2   to_duration_pred.layers.6.2.to_q.weight          1.32e-2 / 1.27e-2
  short p 0.5   to_duration_pred.layers.7.0.0.blocks.0.proj.bias 1.09e-2 / 7.4e-3
so no tensor uses more than 44 % of its rel-L2 bound; forward max-abs error 3.5e-2 - 4.0e-2 against predictions >= 1.5;
d prompts is 82 - 215 x farther from the undropped reference than from the masked one; against the wrong references
every checked tensor is at least 0.095 rel-L2 away (bound 0.03).  Each case takes 3 - 5 s.

Semantics: torch.manual_seed reproduces a call and the next call draws other masks; no_grad and autograd draw the
same masks; eval() and train_dropout=False draw nothing and give the inference output bit for bit;
Conditioner(train_dropout=True) leaves the predictor deterministic; Conditioner(train_duration_pitch=True,
duration_pitch_dropout=True) lowers both L1 losses (evaluated without dropout) in a few AdamW steps.
"""
import time

import pytest
import torch
import torch.nn.functional as F

from param_fill import fill_module
from restatements import DPP_DEPTH as DEPTH
from restatements import DPP_DIM as DIM
from restatements import (dpp_train_inputs, dpp_train_loss, drawn_seed, masked_predictor_fp64, masks_for,
                          set_head_biases_masked, site)

pytestmark = pytest.mark.gpu
MARGIN = 20.0
CASES = {"main": (4, 100, 103), "short": (3, 5, 3)}   # (B, T, Np)


def _predictor():
    from naturalspeech2_pytorch_b200.encoders import DurationPitchPredictor
    m = DurationPitchPredictor(dim=DIM)
    fill_module(m, 4321)
    m.cuda()
    with torch.no_grad():
        for prm in m.parameters():
            prm.copy_(prm.bfloat16().float())
    assert (m.conv_dropout, m.attn_dropout, m.depth) == (0.0, 0.2, DEPTH)
    return m


def _gpu(m, x, prompts, d_outs):
    m.zero_grad(set_to_none=True)
    x_in, p_in = x.clone().requires_grad_(True), prompts.clone().requires_grad_(True)
    dur, pitch = m(x_in, p_in)
    torch.autograd.backward([dur, pitch], [d_outs["duration"], d_outs["pitch"]])
    res = {n: prm.grad.clone() for n, prm in m.named_parameters()}
    res.update({"x": x_in.grad, "prompts": p_in.grad, "out duration": dur.detach(), "out pitch": pitch.detach()})
    return res


def _rel_cos(got, ref):
    got, ref = got.detach().double().flatten(), ref.detach().double().flatten()
    rel = float((got - ref).norm() / ref.norm().clamp_min(1e-300))
    return rel, float(F.cosine_similarity(got, ref, dim=0))


def _bounds(rel0, cos0):
    return max(0.03, 2 * rel0), min(0.9995, 1 - 2 * (1 - cos0))


_CACHE = {}


def _case(name, p):
    if (name, p) in _CACHE:
        return _CACHE[(name, p)]
    t0 = time.perf_counter()
    B, T, Np = CASES[name]
    m = _predictor()
    m.attn_dropout = p
    g = torch.Generator().manual_seed(11 + list(CASES).index(name))
    bf = lambda *s, scale=1.0: (torch.randn(*s, generator=g) * scale).bfloat16().float().cuda()  # noqa: E731
    x, prompts = bf(B, T, DIM), bf(B, Np, DIM)
    d_outs = {"duration": bf(B, T, scale=0.05), "pitch": bf(B, T, scale=0.05)}
    torch_seed = 900 + int(p * 10) + 7 * list(CASES).index(name)
    seed = drawn_seed(torch_seed)
    assert seed >> 32, "the drawn seed should use the key's high word"
    masks = masks_for(seed, p, B, T, Np)
    set_head_biases_masked(m, {n: q.detach() for n, q in m.named_parameters()}, x, prompts, masks)
    params = {n: q.detach() for n, q in m.named_parameters()}
    m.train()
    m.train_dropout = False
    plain = _gpu(m, x, prompts, d_outs)
    m.train_dropout = True
    torch.manual_seed(torch_seed)
    ours = _gpu(m, x, prompts, d_outs)
    plain_ref = masked_predictor_fp64(params, x, prompts, d_outs)
    ref = masked_predictor_fp64(params, x, prompts, d_outs, masks)
    fwd_err = max(float((ours[k] - ref[k]).abs().max()) for k in ("out duration", "out pitch"))
    min_pre = min(float(o[k].abs().min()) for o in (ref, plain_ref) for k in ("out duration", "out pitch"))
    stats = {}
    for n in ref:
        stats[n] = (_rel_cos(ours[n], ref[n]), _rel_cos(plain[n], plain_ref[n]),
                    float(ours[n].double().norm()), float(ref[n].norm()), bool(torch.isfinite(ours[n]).all()))
    res = dict(stats=stats, fwd_err=fwd_err, min_pre=min_pre, params=params, x=x, prompts=prompts, d_outs=d_outs,
               seed=seed, B=B, T=T, Np=Np, p=p,
               differs=_rel_cos(ours["prompts"], plain_ref["prompts"])[0] / max(stats["prompts"][0][0], 1e-12),
               output_changed=not torch.equal(ours["out duration"], plain["out duration"]),
               ours={n: ours[n] for n in WRONG_NAMES}, seconds=time.perf_counter() - t0)
    del ref, plain_ref, plain, ours
    torch.cuda.empty_cache()
    _CACHE[(name, p)] = res
    return res


# d prompts reaches the prompts only through the dropped attention; the rest span both trunks, attention and convs
WRONG_NAMES = ("prompts", "x", "to_duration_pred.layers.9.2.to_kv.weight", "to_duration_pred.layers.9.2.to_out.weight",
               "to_pitch_pred.layers.0.2.to_q.weight", "to_duration_pred.layers.0.0.0.blocks.0.proj.weight",
               "to_pitch_pred.layers.9.0.2.blocks.1.norm.weight")


@pytest.mark.parametrize("p", [0.2, 0.5])
@pytest.mark.parametrize("name", list(CASES))
def test_predictor_dropout_matches_fp64_autograd(name, p):
    r = _case(name, p)
    worst = max(r["stats"].items(), key=lambda kv: kv[1][0][0] / _bounds(*kv[1][1])[0])
    print(f"\n{name} p{p}: {len(r['stats'])} tensors in {r['seconds']:.1f} s; tightest {worst[0]} rel-L2 "
          f"{worst[1][0][0]:.3e} (without dropout {worst[1][1][0]:.3e}); forward max-abs {r['fwd_err']:.3e}, "
          f"min |pred| {r['min_pre']:.3e}; d prompts vs the undropped reference {r['differs']:.0f} x its error")
    assert r["min_pre"] >= MARGIN * r["fwd_err"], "fixture: a head pre-activation lies too close to 0"
    assert r["output_changed"] and r["differs"] > 10, "the dropout must change what the undropped predictor computes"
    bad = []
    for n, ((rel, cos), (rel0, cos0), norm, ref_norm, finite) in r["stats"].items():
        max_rel, min_cos = _bounds(rel0, cos0)
        if not finite or abs(norm - ref_norm) >= 0.02 * ref_norm or rel >= max_rel or cos <= min_cos:
            bad.append((n, finite, norm / ref_norm, rel, rel0, cos, cos0))
    assert not bad, f"{len(bad)} tensors over the bounds: {bad[:8]}"


def _assert_rejected(r, wrong_masks):
    wrong = masked_predictor_fp64(r["params"], r["x"], r["prompts"], r["d_outs"], wrong_masks, only=WRONG_NAMES)
    for n in WRONG_NAMES:
        (rel, cos), (rel0, cos0) = r["stats"][n][:2]
        wrel, wcos = _rel_cos(r["ours"][n], wrong[n])
        max_rel, min_cos = _bounds(rel0, cos0)
        print(f"  {n}: vs the wrong reference rel-L2 {wrel:.3e} cos {wcos:.6f} (bound {max_rel:.3e} / {min_cos:.6f})")
        assert wrel >= max_rel or wcos <= min_cos, f"the bounds accept a wrong reference for {n}"


def test_rejects_the_trunks_sites_swapped():
    r = _case("main", 0.2)
    _assert_rejected(r, masks_for(r["seed"], r["p"], r["B"], r["T"], r["Np"], lambda t, l: site(1 - t, l)))


def test_rejects_attention_masks_moved_to_the_next_site():
    r = _case("main", 0.2)
    _assert_rejected(r, masks_for(r["seed"], r["p"], r["B"], r["T"], r["Np"], lambda t, l: site(t, l) + 1))


def test_rejects_dropout_after_every_block():
    """The reference's Blocks have p = 0: a restatement that also drops every Block's SiLU output (p after each of
    the 120 Blocks, on sites past the attention ones) must be rejected."""
    r = _case("main", 0.2)
    _assert_rejected(r, masks_for(r["seed"], r["p"], r["B"], r["T"], r["Np"],
                                  block_sites=lambda t, l, j: 2 * DEPTH + (t * DEPTH + l) * 6 + j))


# ---- semantics ----
def _small():
    from naturalspeech2_pytorch_b200.encoders import DurationPitchPredictor
    m = DurationPitchPredictor(dim=128, dim_hidden=128, depth=2, heads=2)
    fill_module(m, 55)
    m.cuda().train()
    g = torch.Generator().manual_seed(3)
    return m, torch.randn(2, 17, 128, generator=g).cuda(), torch.randn(2, 9, 128, generator=g).cuda()


def test_seed_draw_no_grad_autograd_and_eval():
    m, x, pr = _small()
    m.train_dropout = True
    with torch.no_grad():
        torch.manual_seed(7)
        a = m(x, pr)
        b = m(x, pr)                                  # the next call draws another seed
        torch.manual_seed(7)
        a2 = m(x, pr)                                 # torch.manual_seed reproduces the draw
    assert all(torch.equal(u, v) for u, v in zip(a, a2))
    assert not torch.equal(a[0], b[0]) and not torch.equal(a[1], b[1])
    torch.manual_seed(7)
    xg = x.clone().requires_grad_(True)
    g = m(xg, pr)                                     # the autograd path draws the same masks
    assert g[0].grad_fn is not None and all(torch.equal(u.detach(), v) for u, v in zip(g, a))
    m.eval()
    state = torch.get_rng_state()
    with torch.no_grad():
        e = m(x, pr)
    assert torch.equal(torch.get_rng_state(), state), "eval() draws nothing"
    m.train()
    m.train_dropout = False
    for grad in (False, True):
        state = torch.get_rng_state()
        with torch.set_grad_enabled(grad):
            t = m(x, pr)
        assert torch.equal(torch.get_rng_state(), state), "train_dropout=False draws nothing"
        assert all(torch.equal(u.detach(), v) for u, v in zip(t, e)), "it is the inference forward"
    assert not torch.equal(e[0], a[0])


def test_conditioner_train_dropout_leaves_the_predictor_deterministic():
    from naturalspeech2_pytorch_b200.encoders import Conditioner
    c = Conditioner(dim_codebook=128, num_phoneme_tokens=50, train_dropout=True, train_duration_pitch=True)
    fill_module(c, 77)
    c.cuda().train()
    dp = c.duration_pitch
    g = torch.Generator().manual_seed(9)
    x, pr = torch.randn(2, 12, 512, generator=g).cuda(), torch.randn(2, 20, 512, generator=g).cuda()
    state = torch.get_rng_state()
    with torch.no_grad():
        a, b = dp(x, pr), dp(x, pr)
    assert torch.equal(torch.get_rng_state(), state)
    assert all(torch.equal(u, v) for u, v in zip(a, b))


def test_conditional_training_with_predictor_dropout_lowers_both_losses():
    """AdamW steps with the predictor's dropout on lower both L1 losses, evaluated without dropout, on a fixed batch."""
    from naturalspeech2_pytorch_b200 import Model, NaturalSpeech2
    from naturalspeech2_pytorch_b200.encoders import Conditioner
    torch.manual_seed(0)
    cond_net = Conditioner(dim_codebook=128, num_phoneme_tokens=50, train_duration_pitch=True,
                           duration_pitch_dropout=True)
    fill_module(cond_net, 77)
    with torch.no_grad():
        for trunk, bias in ((cond_net.duration_pitch.to_duration_pred, 10.0), (cond_net.duration_pitch.to_pitch_pred, 3.0)):
            trunk.to_pred[0].weight.mul_(0.01)       # ReLU heads alive at random init, away from the targets
            trunk.to_pred[0].bias.fill_(bias)
    model = Model(dim=128, depth=1, heads=2, wavenet_layers=2, wavenet_stacks=1, dim_prompt=512, condition_on_prompt=True)
    fill_module(model, 78)
    cond_net.cuda().train()
    model.cuda().train()
    ns = NaturalSpeech2(model, target_sample_hz=24000, timesteps=4, conditioner=cond_net)
    inp = dpp_train_inputs()
    assert cond_net.duration_pitch.train_dropout and cond_net.duration_pitch.attn_dropout == 0.2

    def eval_losses():
        cond_net.eval()
        with torch.no_grad():
            _, _, l_dur, l_pitch = cond_net(prompt=ns.process_prompt(inp["prompt"]), text=inp["text"], mode="train",
                                            pitch=inp["pitch"], duration=inp["duration"])
        cond_net.train()
        return float(l_dur), float(l_pitch)

    before = eval_losses()
    opt = torch.optim.AdamW(list(cond_net.parameters()) + list(model.parameters()), lr=1e-5)
    torch.manual_seed(12)
    losses = []
    for _ in range(6):
        opt.zero_grad(set_to_none=True)
        loss = dpp_train_loss(ns, inp)
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    after = eval_losses()
    assert all(torch.isfinite(torch.tensor(losses))), losses
    assert after[0] < before[0] and after[1] < before[1], (before, after, losses)
