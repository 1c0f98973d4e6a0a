"""GPU: training on a batch of prompts and texts of different lengths, each padded at its end, with per-sample lengths.

The contract (SpeechPromptEncoder, PhonemeEncoder, Model with prompt_lens, Conditioner(mode="train"),
NaturalSpeech2.forward), with sample b = prompt[b, :prompt_lens[b]], text[b, :phoneme_lens[b]], its durations and the
shared-length latents and pitch:
  * forward: every output of sample b is bit-identical to the same call on sample b alone, unpadded;
  * backward, with an upstream gradient fixed per sample: every parameter gradient equals the sum of the
    per-sample-alone gradients and every input gradient the alone one, up to the fp32 summation order that already
    varies between two runs of the same call (dQ's atomics, the weight-gradient position splits), which then moves
    some bf16 roundings by one step.  The bound is a relative L2 error of RTOL = 2^-19 (1.9e-6) per gradient tensor.
    Measured on an NVIDIA H100 80GB HBM3 at 700 W (the tests print these with `-s`): two runs of the same batch call
    differ by at most 7.7e-8 (largest over every gradient tensor of every module); the batch against the sums of the
    alone runs by at most 4.7e-7 (the denoiser's parameter gradients: an alone call of one sample splits its
    weight-gradient positions differently), 1.1e-7 for the encoders' and the Conditioner's; input gradients against the
    alone ones by at most 1.5e-7 (the prompt encoder's d prompt is bit-identical); full lengths against no lengths by at
    most 7.5e-8.  RTOL is 25x the run-to-run spread and 4x the largest error seen;
  * padding: d prompt rows past prompt_lens and the token-table rows that only padded ids reach are exact zeros; NaN in
    the padded prompt frames and random ids in the padded text reach no output and no gradient;
  * full lengths reproduce the call without lengths: the forward bit for bit, the gradients within the bound above.
Shapes are those of the ragged-sampling tests: encoders at their default dims, a small conditional Model.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu
dev = "cuda"
NUM_TOKENS = 40
NP, T, N = 40, 25, 56   # N latent frames >= the largest total duration (25 phonemes x 2)
PROMPT_LENS = [1, 17, 40, 9, 40]
TEXT_LENS = [3, 1, 25, 12, 25]
B = len(PROMPT_LENS)
RTOL = 2.0 ** -19   # see the module docstring for the measured errors it bounds


@pytest.fixture(scope="module")
def mods():
    from naturalspeech2_pytorch_b200 import Model
    from naturalspeech2_pytorch_b200.encoders import Conditioner
    torch.manual_seed(0)
    cn = Conditioner(dim_codebook=128, num_phoneme_tokens=NUM_TOKENS)
    model = Model(dim=128, depth=2, heads=2, wavenet_layers=2, wavenet_stacks=1, dim_prompt=512,
                  condition_on_prompt=True, cond_drop_prob=0.0)
    return cn.to(dev).train(), model.to(dev).train()


@pytest.fixture(scope="module")
def inputs():
    g = torch.Generator().manual_seed(1)
    prompt = torch.randn(B, NP, 128, generator=g)
    text = torch.randint(0, 30, (B, T), generator=g)
    for b, (n, t) in enumerate(zip(PROMPT_LENS, TEXT_LENS)):
        prompt[b, n:] = float("nan")
        text[b, t:] = torch.randint(30, NUM_TOKENS, (T - t,), generator=g)   # ids only padding uses
    duration = torch.randint(1, 3, (B, T), generator=g)
    for b, t in enumerate(TEXT_LENS):
        duration[b, t:] = 0
    pitch = torch.rand(B, N, generator=g) * 300.0
    return dict(prompt=prompt.to(dev), text=text.to(dev), duration=duration.to(dev), pitch=pitch.to(dev))


def _grads(out, upstream, wrt):
    """torch.autograd.grad of sum(out * upstream) (tuples allowed) with respect to `wrt` (None: no gradient)."""
    outs = out if isinstance(out, tuple) else (out,)
    ups = upstream if isinstance(upstream, tuple) else (upstream,)
    loss = sum((o * u).sum() for o, u in zip(outs, ups))
    return list(torch.autograd.grad(loss, wrt, allow_unused=True))


def _close(got, want, what, rtol=RTOL):
    """Relative L2 error of `got` against `want` within rtol (None: no gradient, or an all-zero one); returns it."""
    if want is None:
        assert got is None or int((got != 0).sum()) == 0, what
        return 0.0
    got, want = got.double(), want.double()
    assert bool(torch.isfinite(got).all()), what
    err = (got - want).norm().item()
    rel = err / want.norm().item() if err > 0 else 0.0
    assert rel <= rtol, (what, rel)
    return rel


def _run_to_run(test, got, again, names):
    """The spread of two runs of the same batch call, checked against RTOL and printed (the docstring's number)."""
    worst = max(_close(g2, g, f"{n} run to run") for n, g, g2 in zip(names, got, again))
    print(f"\nrun-to-run spread {test}: {worst:.3e} relative L2 (largest over the gradient tensors)")


def _against_alone(test, got, ref, names):
    """Parameter gradients of the batch call against the sums of the alone ones; the largest error is printed."""
    worst = max(_close(g, r, n) for n, g, r in zip(names, got, ref))
    print(f"\nbatch vs alone {test}: {worst:.3e} relative L2 (largest over the parameter gradients)")


def _full_lengths(test, full, plain, names):
    worst = max(_close(f, p, f"{n} full lengths") for n, f, p in zip(names, full, plain))
    print(f"\nfull lengths vs no lengths {test}: {worst:.3e} relative L2")


def _sum(grads_list):
    out = []
    for gs in zip(*grads_list):
        present = [g for g in gs if g is not None]
        out.append(torch.stack([g.double() for g in present]).sum(0) if present else None)
    return out


def _zero(t, what):
    assert int((t != 0).sum()) == 0, what


def _check_rows(got, alone, lens, what, dim=1):
    for b, n in enumerate(lens):
        assert torch.equal(got[b].narrow(dim - 1, 0, n), alone[b][0]), (what, b, n)
        _zero(got[b].narrow(dim - 1, n, got.shape[dim] - n), (what, b, "padding"))


def _upstream(shape, seed):
    return torch.randn(*shape, device=dev, generator=torch.Generator(device=dev).manual_seed(seed))


def test_speech_prompt_encoder(mods, inputs):
    enc = mods[0].prompt_enc
    params = list(enc.parameters())
    x = inputs["prompt"].clone().requires_grad_(True)
    up = _upstream((B, NP, enc.dim_out), 3)
    out = enc(x, lengths=PROMPT_LENS)
    got = _grads(out, up, params + [x])
    again = _grads(enc(x, lengths=PROMPT_LENS), up, params + [x])
    alone_out, alone = [], []
    for b, n in enumerate(PROMPT_LENS):
        xb = inputs["prompt"][b:b + 1, :n].clone().requires_grad_(True)
        ob = enc(xb)
        alone_out.append(ob.detach())
        alone.append(_grads(ob, up[b:b + 1, :n], params + [xb]))
    _check_rows(out.detach(), alone_out, PROMPT_LENS, "prompt_enc")
    ref = _sum([a[:-1] for a in alone])
    names = [n for n, _ in enc.named_parameters()]
    _run_to_run("SpeechPromptEncoder", got, again, names + ["d prompt"])
    _against_alone("SpeechPromptEncoder", got, ref, names)
    dx = got[-1]
    assert bool(torch.isfinite(dx).all())
    worst = max(_close(dx[b, :n], alone[b][-1][0], f"d prompt sample {b}") for b, n in enumerate(PROMPT_LENS))
    print(f"\ninput gradients vs alone SpeechPromptEncoder: {worst:.3e} relative L2")
    for b, n in enumerate(PROMPT_LENS):
        _zero(dx[b, n:], ("d prompt padding", b))
    # full lengths: the call without lengths
    xf = inputs["prompt"].nan_to_num().requires_grad_(True)
    full_out = enc(xf, lengths=[NP] * B)
    full = _grads(full_out, up, params + [xf])
    plain_out = enc(xf)
    plain = _grads(plain_out, up, params + [xf])
    assert torch.equal(full_out, plain_out)
    _full_lengths("SpeechPromptEncoder", full, plain, names + ["d prompt"])


def test_phoneme_encoder(mods, inputs):
    enc = mods[0].phoneme_enc
    params = list(enc.parameters())
    text = inputs["text"]
    up = _upstream((B, T, enc.dim_hidden), 4)
    out = enc(text, lengths=torch.tensor(TEXT_LENS))
    got = _grads(out, up, params)
    again = _grads(enc(text, lengths=TEXT_LENS), up, params)
    alone_out, alone = [], []
    for b, n in enumerate(TEXT_LENS):
        ob = enc(text[b:b + 1, :n])
        alone_out.append(ob.detach())
        alone.append(_grads(ob, up[b:b + 1, :n], params))
    _check_rows(out.detach(), alone_out, TEXT_LENS, "phoneme_enc")
    _run_to_run("PhonemeEncoder", got, again, [n for n, _ in enc.named_parameters()])
    _against_alone("PhonemeEncoder", got, _sum(alone), [n for n, _ in enc.named_parameters()])
    table = dict(zip([n for n, _ in enc.named_parameters()], got))["token_emb.weight"]
    _zero(table[30:], "token rows only padded ids reach")
    full_out = enc(text, lengths=[T] * B)
    full = _grads(full_out, up, params)
    plain_out = enc(text)
    assert torch.equal(full_out, plain_out)
    _full_lengths("PhonemeEncoder", full, _grads(plain_out, up, params), [n for n, _ in enc.named_parameters()])


def _model_inputs(inputs, seed=5):
    g = torch.Generator(device=dev).manual_seed(seed)
    x = torch.randn(B, N, 128, device=dev, generator=g)
    times = torch.rand(B, device=dev, generator=g)
    prompt = torch.randn(B, NP, 512, device=dev, generator=g)
    for b, n in enumerate(PROMPT_LENS):
        prompt[b, n:] = float("nan")
    cond = torch.randn(B, 512, N, device=dev, generator=g)
    return x, times, prompt, cond


def test_model_prompt_lens(mods, inputs):
    model = mods[1]
    params = list(model.parameters())
    x, times, prompt, cond = _model_inputs(inputs)
    up = _upstream((B, N, 128), 6)

    def run(xs, ts, p, c, **kw):
        p = p.clone().requires_grad_(True)
        c = c.clone().requires_grad_(True)
        out = model(xs, ts, prompt=p, cond=c, **kw)
        return out.detach(), out, p, c

    o, out, p, c = run(x, times, prompt, cond, prompt_lens=PROMPT_LENS)
    got = _grads(out, up, params + [p, c])
    o2, out2, p2, c2 = run(x, times, prompt, cond, prompt_lens=PROMPT_LENS)
    again = _grads(out2, up, params + [p2, c2])
    assert torch.equal(o, o2)
    alone = []
    for b, n in enumerate(PROMPT_LENS):
        ob, outb, pb, cb = run(x[b:b + 1], times[b:b + 1], prompt[b:b + 1, :n], cond[b:b + 1])
        assert torch.equal(o[b], ob[0]), ("prediction", b)
        alone.append(_grads(outb, up[b:b + 1], params + [pb, cb]))
    names = [n for n, _ in model.named_parameters()]
    _run_to_run("Model", got, again, names + ["d prompt", "d cond"])
    _against_alone("Model", got, _sum([a[:-2] for a in alone]), names)
    dp, dc = got[-2], got[-1]
    assert bool(torch.isfinite(dp).all())
    worst = max(max(_close(dp[b, :n], alone[b][-2][0], f"d prompt sample {b}"),
                    _close(dc[b], alone[b][-1][0], f"d cond sample {b}")) for b, n in enumerate(PROMPT_LENS))
    print(f"\ninput gradients vs alone Model: {worst:.3e} relative L2")
    for b, n in enumerate(PROMPT_LENS):
        _zero(dp[b, n:], ("d prompt padding", b))
    pf = prompt.nan_to_num()
    of, outf, _, _ = run(x, times, pf, cond, prompt_lens=[NP] * B)
    full = _grads(outf, up, params)
    op, outp, _, _ = run(x, times, pf, cond)
    assert torch.equal(of, op)
    _full_lengths("Model", full, _grads(outp, up, params), names)


def test_conditioner_train(mods, inputs):
    cn = mods[0]
    params = [p for n, p in cn.named_parameters() if not n.startswith("duration_pitch.")]
    names = [n for n, _ in cn.named_parameters() if not n.startswith("duration_pitch.")]
    up = (_upstream((B, NP, 512), 7), _upstream((B, 512, N), 8))
    kw = dict(mode="train", pitch=inputs["pitch"])
    pe, cond = cn(prompt=inputs["prompt"], text=inputs["text"], duration=inputs["duration"], prompt_lens=PROMPT_LENS,
                  phoneme_lens=TEXT_LENS, **kw)
    got = _grads((pe, cond), up, params)
    again = _grads(cn(prompt=inputs["prompt"], text=inputs["text"], duration=inputs["duration"],
                      prompt_lens=PROMPT_LENS, phoneme_lens=TEXT_LENS, **kw), up, params)
    _run_to_run("Conditioner", got, again, names)
    alone = []
    for b, (n, t) in enumerate(zip(PROMPT_LENS, TEXT_LENS)):
        pa, ca = cn(prompt=inputs["prompt"][b:b + 1, :n], text=inputs["text"][b:b + 1, :t],
                    duration=inputs["duration"][b:b + 1, :t], pitch=inputs["pitch"][b:b + 1], mode="train")
        assert torch.equal(pe[b, :n], pa[0]) and torch.equal(cond[b], ca[0]), b
        _zero(pe[b, n:], ("prompt_enc padding", b))
        alone.append(_grads((pa, ca), (up[0][b:b + 1, :n], up[1][b:b + 1]), params))
    _against_alone("Conditioner", got, _sum(alone), names)
    table = dict(zip(names, got))["phoneme_enc.token_emb.weight"]
    _zero(table[30:], "token rows only padded ids reach")


def test_natural_speech2_forward(mods, inputs, monkeypatch):
    """Each sample's MSE row is bit-identical to its alone run.  The loss is not the mean of the alone losses: the
    reference's min-SNR weighting broadcasts the (B,) MSE rows against (B, 1, 1) weights (ns2.py:1651-1666), so the
    loss is mean(mse) * mean(weight).  Its gradients are checked in test_ragged_training_fp64_gpu.py."""
    from naturalspeech2_pytorch_b200 import NaturalSpeech2, training
    from naturalspeech2_pytorch_b200.diffusion import gamma_to_alpha_sigma
    cn, model = mods
    ns = NaturalSpeech2(model, target_sample_hz=24000, timesteps=3, conditioner=cn)
    rows = []
    mse_apply = training.MseRowsFunction.apply

    def spy(pred, target):
        r = mse_apply(pred, target)
        rows.append(r.detach().clone())
        return r
    monkeypatch.setattr(training.MseRowsFunction, "apply", spy)
    g = torch.Generator(device=dev).manual_seed(9)
    audio = torch.randn(B, N, 128, device=dev, generator=g)
    times = torch.rand(B, device=dev, generator=g)
    noise = torch.randn(B, N, 128, device=dev, generator=g)
    common = dict(pitch=inputs["pitch"], times=times, noise=noise)
    loss = ns(audio, text=inputs["text"], prompt=inputs["prompt"], duration=inputs["duration"],
              prompt_lens=PROMPT_LENS, phoneme_lens=TEXT_LENS, **common)
    batch_rows = rows[-1]
    for b, (n, t) in enumerate(zip(PROMPT_LENS, TEXT_LENS)):
        ns(audio[b:b + 1], text=inputs["text"][b:b + 1, :t], prompt=inputs["prompt"][b:b + 1, :n],
           duration=inputs["duration"][b:b + 1, :t], pitch=inputs["pitch"][b:b + 1], times=times[b:b + 1],
           noise=noise[b:b + 1])
        assert torch.equal(batch_rows[b], rows[-1][0]), b
    alpha, sigma = gamma_to_alpha_sigma(ns.gamma_schedule(times), ns.scale)
    snr = (alpha * alpha) / (sigma * sigma)
    weight = snr.clamp(max=ns.min_snr_gamma) / (snr + 1) if ns.min_snr_loss_weight else snr / (snr + 1)
    assert ns.objective == "v"
    want = batch_rows.double().mean() * weight.double().mean()
    assert abs(loss.item() - want.item()) <= 1e-5 * abs(want.item()), (loss.item(), want.item())
