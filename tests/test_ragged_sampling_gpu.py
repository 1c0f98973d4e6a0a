"""GPU: sampling a batch of prompts and texts of different lengths, each padded at its end, with per-sample lengths.

The contract: every sample's result is bit-identical to running that sample alone, unpadded, through the path without
lengths (which the golden tests pin to the reference); padded output rows are exact zeros; what the padded input rows
hold (NaN prompt frames, random phoneme ids) reaches no output; all-full lengths reproduce the call without lengths.
Checked at the encoders' default dims for SpeechPromptEncoder, PhonemeEncoder, DurationPitchPredictor, the Conditioner,
Model.precompute_conditioning and NaturalSpeech2.sample (3 DDIM steps, cond_scale 1 and 3, graphs on and off).
"""
import pytest
import torch

pytestmark = pytest.mark.gpu
dev = "cuda"
NUM_TOKENS = 40
NP, T, LENGTH = 40, 25, 48
PROMPT_LENS = [1, 17, 40, 9, 40]
TEXT_LENS = [3, 1, 25, 12, 25]
B = len(PROMPT_LENS)


@pytest.fixture(scope="module")
def mods():
    from naturalspeech2_pytorch_b200 import Model
    from naturalspeech2_pytorch_b200.encoders import Conditioner
    torch.manual_seed(0)
    cn = Conditioner(dim_codebook=128, num_phoneme_tokens=NUM_TOKENS)
    with torch.no_grad():   # durations of a few frames per phoneme, so every sample has a condition
        head = cn.duration_pitch.to_duration_pred.to_pred[0]
        head.weight.mul_(0.05)
        head.bias.fill_(2.5)
    model = Model(dim=128, depth=2, heads=2, wavenet_layers=2, wavenet_stacks=1, dim_prompt=512,
                  condition_on_prompt=True)
    return cn.to(dev).eval(), model.to(dev).eval()


@pytest.fixture(scope="module")
def inputs():
    g = torch.Generator().manual_seed(1)
    prompt = torch.randn(B, NP, 128, generator=g)
    text = torch.randint(0, NUM_TOKENS, (B, T), generator=g)   # padded ids stay random
    for b, n in enumerate(PROMPT_LENS):
        prompt[b, n:] = float("nan")
    return prompt.to(dev), text.to(dev)


def _nan_past(t, lens, dim=1):
    t = t.clone()
    for b, n in enumerate(lens):
        t[b].narrow(dim - 1, n, t.shape[dim] - n).fill_(float("nan"))
    return t


def _check_rows(got, alone, lens, what, dim=1):
    for b, n in enumerate(lens):
        assert torch.equal(got[b].narrow(dim - 1, 0, n), alone[b][0]), (what, b, n)
        assert int((got[b].narrow(dim - 1, n, got.shape[dim] - n) != 0).sum()) == 0, (what, b, "padding")


def test_prompt_encoder(mods, inputs):
    enc = mods[0].prompt_enc
    prompt = inputs[0]
    out = enc(prompt, lengths=PROMPT_LENS)
    _check_rows(out, [enc(prompt[b:b + 1, :n]) for b, n in enumerate(PROMPT_LENS)], PROMPT_LENS, "prompt_enc")
    full = prompt.nan_to_num()
    assert torch.equal(enc(full, lengths=[NP] * B), enc(full))


def test_phoneme_encoder(mods, inputs):
    enc = mods[0].phoneme_enc
    text = inputs[1]
    out = enc(text, lengths=torch.tensor(TEXT_LENS))
    _check_rows(out, [enc(text[b:b + 1, :n]) for b, n in enumerate(TEXT_LENS)], TEXT_LENS, "phoneme_enc")
    assert torch.equal(enc(text, lengths=[T] * B), enc(text))
    with pytest.raises(NotImplementedError):
        enc(text, mask=torch.ones(B, T, dtype=torch.bool, device=dev), lengths=TEXT_LENS)


def test_duration_pitch_predictor(mods, inputs):
    cn = mods[0]
    with torch.no_grad():
        pe = cn.prompt_enc(inputs[0].nan_to_num())
        ph = cn.phoneme_enc(inputs[1])
    x, p = _nan_past(ph, TEXT_LENS), _nan_past(pe, PROMPT_LENS)
    dur, pit = cn.duration_pitch(x, p, lengths=TEXT_LENS, prompt_lens=PROMPT_LENS)
    alone = [cn.duration_pitch(ph[b:b + 1, :n], pe[b:b + 1, :PROMPT_LENS[b]]) for b, n in enumerate(TEXT_LENS)]
    _check_rows(dur[..., None], [(a[0][0][..., None],) for a in alone], TEXT_LENS, "duration")
    _check_rows(pit[..., None], [(a[1][0][..., None],) for a in alone], TEXT_LENS, "pitch")
    assert bool((dur.sum(-1) > 0).all())
    full = cn.duration_pitch(ph, pe, lengths=[T] * B, prompt_lens=[NP] * B)
    plain = cn.duration_pitch(ph, pe)
    assert torch.equal(full[0], plain[0]) and torch.equal(full[1], plain[1])


def _alone_conditioner(cn, prompt, text):
    return [cn(prompt=prompt[b:b + 1, :PROMPT_LENS[b]], text=text[b:b + 1, :n], mode="sample")
            for b, n in enumerate(TEXT_LENS)]


def test_conditioner(mods, inputs):
    cn = mods[0]
    pe, cond, cond_lens = cn(prompt=inputs[0], text=inputs[1], mode="sample", prompt_lens=PROMPT_LENS,
                             phoneme_lens=TEXT_LENS)
    alone = _alone_conditioner(cn, *inputs)
    assert cond_lens.dtype == torch.int32 and cond_lens.tolist() == [a[1].shape[-1] for a in alone]
    _check_rows(pe, [(a[0][0],) for a in alone], PROMPT_LENS, "prompt_enc")
    _check_rows(cond, [(a[1][0],) for a in alone], cond_lens.tolist(), "cond", dim=2)
    with pytest.raises(NotImplementedError):
        cn(prompt=inputs[0], text=inputs[1], mode="train", prompt_lens=PROMPT_LENS)


def test_precompute_conditioning(mods, inputs):
    cn, model = mods
    pe, cond, cond_lens = cn(prompt=inputs[0], text=inputs[1], mode="sample", prompt_lens=PROMPT_LENS,
                             phoneme_lens=TEXT_LENS)
    c = model.precompute_conditioning(_nan_past(pe, PROMPT_LENS), _nan_past(cond, cond_lens.tolist(), dim=2), LENGTH,
                                      prompt_lens=PROMPT_LENS, cond_lens=cond_lens)
    for b, (pa, ca) in enumerate(_alone_conditioner(cn, *inputs)):
        a = model.precompute_conditioning(pa, ca, LENGTH)
        for k, got in (("prompt_cond", c["prompt_cond"][b]), ("tokens", c["tokens"][b]),
                       ("cond_proj", c["cond_proj"][b, :ca.shape[-1]])):
            assert torch.equal(got, a[k][0]), (k, b, (got - a[k][0]).abs().max().item())
    full = model.precompute_conditioning(pe, cond, LENGTH, prompt_lens=[NP] * B)
    plain = model.precompute_conditioning(pe, cond, LENGTH)
    for k in ("prompt_cond", "tokens", "cond_proj"):
        assert torch.equal(full[k], plain[k]), k


@pytest.mark.parametrize("graphs", [False, True], ids=["eager", "graphs"])
@pytest.mark.parametrize("cond_scale", [1.0, 3.0])
def test_sample(mods, inputs, cond_scale, graphs):
    from naturalspeech2_pytorch_b200 import NaturalSpeech2
    cn, model = mods
    ns = NaturalSpeech2(model, target_sample_hz=24000, timesteps=3, cuda_graphs=graphs, conditioner=cn)
    noise = torch.randn(B, LENGTH, 128, device=dev, generator=torch.Generator(device=dev).manual_seed(2))
    pe, cond, cond_lens = cn(prompt=inputs[0], text=inputs[1], mode="sample", prompt_lens=PROMPT_LENS,
                             phoneme_lens=TEXT_LENS)
    got = ns.sample(length=LENGTH, prompt_enc=_nan_past(pe, PROMPT_LENS), cond=_nan_past(cond, cond_lens.tolist(), 2),
                    prompt_lens=PROMPT_LENS, cond_lens=cond_lens, cond_scale=cond_scale, noise=noise)
    assert bool(torch.isfinite(got).all())
    for b, (pa, ca) in enumerate(_alone_conditioner(cn, *inputs)):
        alone = ns.sample(length=LENGTH, prompt_enc=pa, cond=ca, cond_scale=cond_scale, noise=noise[b:b + 1])
        assert torch.equal(got[b], alone[0]), b
    via_conditioner = ns.sample(length=LENGTH, prompt=inputs[0], text=inputs[1], prompt_lens=PROMPT_LENS,
                                phoneme_lens=TEXT_LENS, cond_scale=cond_scale, noise=noise)
    assert torch.equal(via_conditioner, got)
    full = ns.sample(length=LENGTH, prompt_enc=pe, cond=cond, prompt_lens=[NP] * B,
                     cond_lens=[cond.shape[-1]] * B, cond_scale=cond_scale, noise=noise)
    plain = ns.sample(length=LENGTH, prompt_enc=pe, cond=cond, cond_scale=cond_scale, noise=noise)
    assert torch.equal(full, plain)


def test_sample_rejects_raw_audio_prompt_with_lengths(mods, inputs):
    from naturalspeech2_pytorch_b200 import NaturalSpeech2
    cn, model = mods
    ns = NaturalSpeech2(model, target_sample_hz=24000, timesteps=3, conditioner=cn)
    with pytest.raises(ValueError, match="encoded latents"):
        ns.sample(length=LENGTH, prompt=torch.randn(B, 4800, device=dev), text=inputs[1], prompt_lens=PROMPT_LENS,
                  phoneme_lens=TEXT_LENS)
