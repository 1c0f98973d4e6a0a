"""GPU: the denoiser and the sampler on batches of latents of different lengths, each padded at its end.

The contract: sample b's prediction rows [0, L_b) are bit-identical to running x[b:b+1, :L_b] alone (unpadded, through
the path without lengths), rows past L_b are exact zeros, and NaN in the padded rows of x and of the condition reaches
nothing.  `NaturalSpeech2.sample(latent_lens=...)` matches sampling each sample alone with length=L_b and the first L_b
frames of its noise, bit for bit.  Checked unconditional, conditional and with classifier-free guidance, eager and with
CUDA graphs, at a small configuration and at dim 512 with N = 1024.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu
dev = "cuda"

SMALL = dict(dim=128, depth=2, heads=2, wavenet_layers=3, wavenet_stacks=2)
SMALL_N, SMALL_LENS = 300, [1, 7, 128, 129, 256, 300, 64]
BIG = dict(dim=512, depth=2, heads=8, wavenet_layers=8, wavenet_stacks=2)
BIG_N, BIG_LENS = 1024, [1024, 1, 300, 513, 1023, 640]
DIM_PROMPT, NP, LC = 128, 40, 200


def _model(cfg, cond):
    from naturalspeech2_pytorch_b200 import Model
    torch.manual_seed(0)
    kw = dict(cfg, dim_prompt=DIM_PROMPT, condition_on_prompt=True) if cond else cfg
    return Model(**kw).to(dev).eval()


def _nan_past(x, lens, dim=1):
    x = x.clone()
    for b, n in enumerate(lens):
        n = min(n, x.shape[dim])   # a condition shorter than the latent has no padding past the sample
        x[b].narrow(dim - 1, n, x.shape[dim] - n).fill_(float("nan"))
    return x


def _check(got, alone, lens):
    for b, n in enumerate(lens):
        assert torch.equal(got[b, :n], alone[b][0]), (b, n, (got[b, :n] - alone[b][0]).abs().max().item())
        assert int((got[b, n:] != 0).sum()) == 0, (b, n, "padding")


@pytest.fixture(scope="module", params=["small", "dim512"])
def case(request):
    return (SMALL, SMALL_N, SMALL_LENS) if request.param == "small" else (BIG, BIG_N, BIG_LENS)


@pytest.mark.parametrize("mode", ["uncond", "cond", "cfg"])
@pytest.mark.parametrize("graphs", [False, True], ids=["eager", "graphs"])
def test_forward_matches_each_sample_alone(case, mode, graphs):
    cfg, N, lens = case
    B = len(lens)
    model = _model(cfg, mode != "uncond")
    model.use_cuda_graphs = graphs
    g = torch.Generator(device=dev).manual_seed(1)
    x = torch.randn(B, N, cfg["dim"], device=dev, generator=g)
    times = torch.rand(B, device=dev, generator=g)
    kw, alone_kw = {}, [{} for _ in lens]
    if mode != "uncond":
        prompt = torch.randn(B, NP, DIM_PROMPT, device=dev, generator=g)
        cond = torch.randn(B, DIM_PROMPT, LC, device=dev, generator=g)
        c = model.precompute_conditioning(prompt, _nan_past(cond, lens, dim=2), N)
        kw = dict(_conditioning=c)
        alone_kw = [dict(_conditioning=model.precompute_conditioning(prompt[b:b + 1], cond[b:b + 1], n))
                    for b, n in enumerate(lens)]
    scale = 3.0 if mode == "cfg" else 1.0
    lt = torch.tensor(lens, dtype=torch.int32, device=dev)
    got = model.forward_with_cond_scale(_nan_past(x, lens), times, cond_scale=scale, lengths=lt, **kw)
    got2 = model.forward_with_cond_scale(_nan_past(x, lens), times, cond_scale=scale, lengths=lens, **kw)
    assert torch.equal(got, got2)
    alone = [model.forward_with_cond_scale(x[b:b + 1, :n], times[b:b + 1], cond_scale=scale, **alone_kw[b])
             for b, n in enumerate(lens)]
    _check(got, alone, lens)
    if mode != "uncond":   # conditioning without NaN, which the plain call would read
        kw = dict(_conditioning=model.precompute_conditioning(prompt, cond, N))
    full = model.forward_with_cond_scale(x, times, cond_scale=scale, lengths=[N] * B, **kw)
    plain = model.forward_with_cond_scale(x, times, cond_scale=scale, **kw)
    assert torch.equal(full, plain)


@pytest.mark.parametrize("mode", ["uncond", "cfg"])
@pytest.mark.parametrize("graphs", [False, True], ids=["eager", "graphs"])
def test_sample_matches_each_sample_alone(mode, graphs):
    from naturalspeech2_pytorch_b200 import NaturalSpeech2
    lens = SMALL_LENS
    B, N, D = len(lens), SMALL_N, SMALL["dim"]
    model = _model(SMALL, mode != "uncond")
    ns = NaturalSpeech2(model, target_sample_hz=24000, timesteps=3, cuda_graphs=graphs)
    g = torch.Generator(device=dev).manual_seed(2)
    noise = torch.randn(B, N, D, device=dev, generator=g)
    kw, alone_kw = dict(batch_size=B), [{} for _ in lens]
    if mode != "uncond":
        pe = torch.randn(B, NP, DIM_PROMPT, device=dev, generator=g)
        cond = torch.randn(B, DIM_PROMPT, LC, device=dev, generator=g)
        kw = dict(prompt_enc=pe, cond=cond, cond_scale=3.0)
        alone_kw = [dict(prompt_enc=pe[b:b + 1], cond=cond[b:b + 1], cond_scale=3.0) for b in range(B)]
    got = ns.sample(length=N, latent_lens=lens, noise=_nan_past(noise, lens), **kw)
    alone = [ns.sample(length=n, noise=noise[b:b + 1, :n], **alone_kw[b]) for b, n in enumerate(lens)]
    _check(got, alone, lens)
    again = ns.sample(length=N, latent_lens=torch.tensor(lens), noise=noise, **kw)   # other lengths object, same graph
    assert torch.equal(again, got)



@pytest.mark.parametrize("graphs", [False, True], ids=["eager", "graphs"])
def test_sample_with_prompt_and_cond_lens(graphs):
    """latent_lens together with prompt_lens / cond_lens: each sample as if sampled alone with its own prompt, condition
    and latent length."""
    from naturalspeech2_pytorch_b200 import NaturalSpeech2
    lens, plens, clens = [1, 130, 300, 64], [5, 40, 17, 40], [1, 100, 200, 64]
    B, N, D = len(lens), 300, SMALL["dim"]
    model = _model(SMALL, True)
    ns = NaturalSpeech2(model, target_sample_hz=24000, timesteps=3, cuda_graphs=graphs)
    g = torch.Generator(device=dev).manual_seed(5)
    noise = torch.randn(B, N, D, device=dev, generator=g)
    pe = torch.randn(B, NP, DIM_PROMPT, device=dev, generator=g)
    cond = torch.randn(B, DIM_PROMPT, LC, device=dev, generator=g)
    got = ns.sample(length=N, prompt_enc=_nan_past(pe, plens), cond=_nan_past(cond, clens, dim=2), prompt_lens=plens,
                    cond_lens=clens, latent_lens=lens, noise=noise, cond_scale=3.0)
    alone = [ns.sample(length=n, prompt_enc=pe[b:b + 1, :plens[b]], cond=cond[b:b + 1, :, :clens[b]],
                       noise=noise[b:b + 1, :n], cond_scale=3.0) for b, n in enumerate(lens)]
    _check(got, alone, lens)


def test_sample_with_codec_waveforms():
    """With a SEANet codec each waveform is zero past L_b * 320 samples, and for L_b >= 7 frames (longer than the first
    k7 conv's pad) its prefix is the waveform of the sample decoded alone: the decoder is causal.  L_b = 3 lies outside
    that guarantee (Encodec's short-input padding rule applies when it is decoded alone): only its zeros are checked."""
    from naturalspeech2_pytorch_b200 import EncodecRVQ, Model, NaturalSpeech2, SEANetDecoder
    torch.manual_seed(0)
    model = Model(dim=128, depth=1, heads=2, wavenet_layers=2, wavenet_stacks=1).to(dev).eval()
    codec = EncodecRVQ(torch.randn(4, 1024, 128), decoder=SEANetDecoder().eval()).to(dev)
    ns = NaturalSpeech2(model, codec=codec, timesteps=2)
    lens, N = [7, 40, 3, 21], 40
    B = len(lens)
    noise = torch.randn(B, N, 128, device=dev, generator=torch.Generator(device=dev).manual_seed(6))
    wav = ns.sample(length=N, batch_size=B, noise=noise, latent_lens=lens)
    assert tuple(wav.shape) == (B, 320 * N) and bool(torch.isfinite(wav).all())
    for b, n in enumerate(lens):
        assert int((wav[b, 320 * n:] != 0).sum()) == 0, b
        if n >= 7:
            alone = ns.sample(length=n, batch_size=1, noise=noise[b:b + 1, :n])
            assert torch.equal(wav[b, :320 * n], alone[0]), (b, (wav[b, :320 * n] - alone[0]).abs().max().item())
