"""GPU: a batch of waveforms of different lengths, padded at the end, through the codec and the training objective.

Sample b of a padded waveform batch is audio[b, :320 lengths[b]], lengths in frames.  The contract:
  * encoder / codec: sample b's frames, latents and codes are bit-identical to encoding its waveform alone; past its
    length frames and latents are exact zeros and codes -1; NaN in the padding reaches nothing; lengths all equal to
    N reproduce the call without lengths.  Lengths {7, 8, 63, 64, 65, 127, 128, 129, N - 1, N} at N = 1024, and 64
    samples in one batch;
  * training: `NaturalSpeech2.forward(raw_audio, latent_lens=)` gives the loss of `forward(alone-encoded latents,
    latent_lens=)` bit for bit and the same parameter gradients (up to the summation order of the float atomics in the
    bias and FiLM gradients: relative L2 <= 2^-19), unconditional and conditional with a raw prompt and prompt_lens;
  * the RVQ cross-entropy term with latent_lens is `codec.rq` on x_start with -1 targets past each length, bit for bit;
    its entries lie within the bounds of test_rvq_codec_edges_gpu.py against the float64 restatement on the valid
    frames, and d pred past the lengths is exactly zero;
  * sampling with a raw prompt and prompt_lens is bit-identical to sampling with the alone-encoded prompt latents.
Weights, audio and codebooks are the seeded ones of tests/golden/make_golden_seanet_encoder.py.
"""
import numpy as np
import pytest
import torch

from golden.make_golden_seanet_encoder import audio, codebooks, filled_state_dict
from kernel_check import acc_eps, assert_close
from rvq_ce_restatement import residual_vq_ce

pytestmark = pytest.mark.gpu
dev = "cuda"
NAN = float("nan")
RTOL = 2.0 ** -19
ERR_MULT, FLOOR = 4.0, 2.0 ** -16   # the entry bound of test_rvq_codec_edges_gpu.py


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(golden_dir / "seanet_encoder.npz")


@pytest.fixture(scope="module")
def enc(golden):
    from naturalspeech2_pytorch_b200 import SEANetEncoder
    keys_shapes = [(k, tuple(int(v) for v in s.split(","))) for k, s in zip(golden["keys"], golden["shapes"])]
    e = SEANetEncoder()
    e.load_state_dict({k: v.float() for k, v in filled_state_dict(keys_shapes).items()})
    return e.to(dev).eval()


@pytest.fixture(scope="module")
def codec(golden, enc):
    from naturalspeech2_pytorch_b200 import EncodecRVQ
    return EncodecRVQ(codebooks(golden["cb_scale"]).float(), encoder=enc).to(dev)


def _padded(B, N, lens, fill=NAN):
    """(B, 320 N) fp32 waveforms, each `fill` past its 320 lens[b] samples."""
    x = audio(B, N).float().to(dev)
    for b, n in enumerate(lens):
        x[b, 320 * n:] = fill
    return x


def _alone(codec, x, lens):
    """Per sample: (frames, emb, codes) of its waveform encoded alone."""
    out = []
    for b, n in enumerate(lens):
        w = x[b:b + 1, :320 * n]
        emb, codes, _ = codec(w, return_encoded=True)
        out.append((codec.encoder(w), emb, codes))
    return out


def _check_encoding(codec, x, lens):
    frames = codec.encoder(x, lengths=lens)
    emb, codes, _ = codec(x, return_encoded=True, lengths=lens)
    N = x.shape[1] // 320
    lens = [int(n) for n in lens]
    assert frames.shape == emb.shape == (len(lens), N, 128) and codes.shape == (len(lens), N, codec.num_quantizers)
    assert codes.dtype == torch.int64 and codes.is_contiguous()
    for b, (n, (f1, e1, c1)) in enumerate(zip(lens, _alone(codec, x, lens))):
        assert torch.equal(frames[b, :n], f1[0]), ("frames", b, n)
        assert torch.equal(emb[b, :n], e1[0]), ("emb", b, n)
        assert torch.equal(codes[b, :n], c1[0]), ("codes", b, n)
        assert int((frames[b, n:] != 0).sum()) == 0 and int((emb[b, n:] != 0).sum()) == 0, ("zeros", b, n)
        assert bool((codes[b, n:] == -1).all()), ("codes -1", b, n)
    return frames, emb, codes


def test_lengths_at_tile_edges_are_each_sample_alone(codec):
    N = 1024
    lens = [7, 8, 63, 64, 65, 127, 128, 129, N - 1, N]
    _check_encoding(codec, _padded(len(lens), N, lens), lens)


def test_64_samples_in_one_batch(codec):
    N = 160
    g = torch.Generator().manual_seed(5)
    edges = [7, 8, 63, 64, 65, 127, 128, 129, N - 1, N]
    lens = edges + torch.randint(7, N + 1, (64 - len(edges),), generator=g).tolist()
    x = _padded(64, N, lens)
    frames, emb, codes = _check_encoding(codec, x, torch.tensor(lens, dtype=torch.int32, device=dev))
    # zero padding gives the same result as NaN padding
    e0, c0, _ = codec(_padded(64, N, lens, fill=0.0), return_encoded=True, lengths=lens)
    assert torch.equal(e0, emb) and torch.equal(c0, codes)


def test_full_lengths_reproduce_the_call_without_lengths(codec):
    B, N = 3, 200
    x = audio(B, N).float().to(dev)
    assert torch.equal(codec.encoder(x, lengths=[N] * B), codec.encoder(x))
    e1, c1, _ = codec(x, return_encoded=True, lengths=[N] * B)
    e2, c2, _ = codec(x, return_encoded=True)
    assert torch.equal(e1, e2) and torch.equal(c1, c2)
    # a partial frame past the last whole one is dropped, not curtailed from the left
    longer = torch.cat([x, torch.full((B, 123), NAN, device=dev)], dim=1)
    e3, c3, _ = codec(longer, return_encoded=True, curtail_from_left=True, lengths=[N] * B)
    assert torch.equal(e3, e2) and torch.equal(c3, c2)


# -------------------------------------------------------------------------------------------------------------------
# training
# -------------------------------------------------------------------------------------------------------------------
LENS = [48, 7, 23, 40]
N = 48
B = len(LENS)
PROMPT_LENS, NP = [7, 12, 9, 12], 12
TEXT_LENS, T, NUM_TOKENS = [10, 3, 7, 10], 10, 40


def _latents_alone(codec, x, lens, n_frames=N):
    """Alone-encoded latents and codes, zero-padded to n_frames (codes padded with 0: the lengths mask them)."""
    emb = torch.zeros(len(lens), n_frames, 128, device=dev)
    codes = torch.zeros(len(lens), n_frames, codec.num_quantizers, dtype=torch.int64, device=dev)
    for b, n in enumerate(lens):
        e, c, _ = codec(x[b:b + 1, :320 * n], return_encoded=True)
        emb[b, :n], codes[b, :n] = e[0], c[0]
    return emb, codes


def _grads(params):
    out = [None if p.grad is None else p.grad.detach().clone() for p in params]
    for p in params:
        p.grad = None
    return out


def _same_grads(got, want):
    exact = 0
    for i, (a, w) in enumerate(zip(got, want)):
        assert (a is None) == (w is None), i
        if a is None:
            continue
        assert bool(torch.isfinite(a).all()), i
        err = (a.double() - w.double()).norm().item()
        ref = w.double().norm().item()
        assert err <= RTOL * ref, (i, err, ref)
        exact += bool(torch.equal(a, w))
    print(f"{exact} of {len(got)} parameter gradients bit-identical")


def _uncond(codec, ce_weight):
    from naturalspeech2_pytorch_b200 import Model, NaturalSpeech2
    torch.manual_seed(0)
    model = Model(dim=128, depth=1, heads=2, wavenet_layers=2, wavenet_stacks=1).to(dev).train()
    return NaturalSpeech2(model, codec=codec, timesteps=2, rvq_cross_entropy_loss_weight=ce_weight)


def _draws():
    g = torch.Generator(device=dev).manual_seed(2)
    return torch.rand(B, device=dev, generator=g), torch.randn(B, N, 128, device=dev, generator=g)


@pytest.mark.parametrize("ce_weight", [0.0, 0.5])
def test_raw_audio_training_equals_alone_encoded_latents(codec, ce_weight):
    ns = _uncond(codec, ce_weight)
    params = list(ns.model.parameters())
    times, noise = _draws()
    x = _padded(B, N, LENS)
    loss_raw = ns(x, times=times, noise=noise, latent_lens=LENS)
    loss_raw.backward()
    g_raw = _grads(params)
    lat, codes = _latents_alone(codec, x, LENS)
    loss_lat = ns(lat, codes=codes, times=times, noise=noise, latent_lens=LENS)
    loss_lat.backward()
    assert bool(torch.isfinite(loss_raw)) and torch.equal(loss_raw.detach(), loss_lat.detach())
    _same_grads(g_raw, _grads(params))


def test_conditional_raw_audio_and_raw_prompt_equal_alone_encoded(codec):
    from naturalspeech2_pytorch_b200 import Model, NaturalSpeech2
    from naturalspeech2_pytorch_b200.encoders import Conditioner
    torch.manual_seed(0)
    cn = Conditioner(dim_codebook=128, num_phoneme_tokens=NUM_TOKENS).to(dev).train()
    model = Model(dim=128, depth=1, heads=2, wavenet_layers=2, wavenet_stacks=1, dim_prompt=512,
                  condition_on_prompt=True, cond_drop_prob=0.0).to(dev).train()
    ns = NaturalSpeech2(model, codec=codec, timesteps=2, conditioner=cn, rvq_cross_entropy_loss_weight=0.5)
    params = list(model.parameters()) + list(cn.parameters())
    g = torch.Generator().manual_seed(4)
    text = torch.randint(0, NUM_TOKENS, (B, T), generator=g).to(dev)
    duration = torch.randint(1, 3, (B, T), generator=g)
    for b, t in enumerate(TEXT_LENS):
        duration[b, t:] = 0
        assert int(duration[b].sum()) <= LENS[b]
    duration = duration.to(dev)
    pitch = (torch.rand(B, N, generator=g) * 300.0).to(dev)
    times, noise = _draws()
    x = _padded(B, N, LENS)
    prompt = _padded(B, NP, PROMPT_LENS)
    common = dict(text=text, duration=duration, pitch=pitch, times=times, noise=noise, prompt_lens=PROMPT_LENS,
                  phoneme_lens=TEXT_LENS, latent_lens=LENS)
    loss_raw = ns(x, prompt=prompt, **common)
    loss_raw.backward()
    g_raw = _grads(params)
    lat, codes = _latents_alone(codec, x, LENS)
    prompt_lat, _ = _latents_alone(codec, prompt, PROMPT_LENS, NP)
    loss_lat = ns(lat, codes=codes, prompt=prompt_lat, **common)
    loss_lat.backward()
    assert bool(torch.isfinite(loss_raw)) and torch.equal(loss_raw.detach(), loss_lat.detach())
    _same_grads(g_raw, _grads(params))


def test_cross_entropy_term_is_rq_with_ignored_targets(codec, monkeypatch):
    from naturalspeech2_pytorch_b200 import ops
    calls = []
    rvq_ce = ops.rvq_ce

    def spy(frames, cbs, cn2, own, tgt):
        loss = rvq_ce(frames, cbs, cn2, own, tgt)
        calls.append((frames.clone(), own.clone(), tgt.clone(), loss.clone()))
        return loss
    monkeypatch.setattr(ops, "rvq_ce", spy)
    times, noise = _draws()
    x = _padded(B, N, LENS)
    lat, codes = _latents_alone(codec, x, LENS)
    lat_nan = lat.clone()
    for b, n in enumerate(LENS):
        lat_nan[b, n:] = NAN   # padding that is not finite reaches neither x_start nor the own codes
    loss = _uncond(codec, 0.5)(lat_nan, codes=codes, times=times, noise=noise, latent_lens=LENS)
    mse = _uncond(codec, 0.0)(lat_nan, times=times, noise=noise, latent_lens=LENS)
    frames, own, tgt, ce = calls[-1]
    assert torch.equal(loss.detach(), mse.detach() + 0.5 * ce)
    valid = torch.zeros(B, N, dtype=torch.bool, device=dev)
    for b, n in enumerate(LENS):
        valid[b, :n] = True
    valid = valid.view(-1)
    assert torch.equal(tgt[valid], codes.view(-1, codes.shape[-1])[valid]) and bool((tgt[~valid] == -1).all())
    assert int((frames[~valid] != 0).sum()) == 0 and bool(torch.isfinite(frames).all())
    monkeypatch.setattr(ops, "rvq_ce", rvq_ce)
    _, ce_rq = codec.rq(frames.view(B, N, 128), tgt.view(B, N, -1))   # the existing path, -1 targets
    assert torch.equal(ce_rq, ce)
    _check_ce_bounds(codec, frames[valid], own[valid], tgt[valid], float(ce), B * N)


def _ce_entries(x, cb, own, tgt, dtype):
    """(F, Q) CE of every frame and stage in `dtype` (the expanded-distance formula on the own-code residual chain)."""
    cbd = cb.to(dtype)
    cn2 = (cbd * cbd).sum(-1)
    r = x.to(dtype)
    out = torch.zeros(own.shape, dtype=dtype, device=x.device)
    for q in range(own.shape[1]):
        lg = -((r * r).sum(-1, keepdim=True) - 2.0 * (r @ cbd[q].t()) + cn2[q][None]).clamp_min(0.0).sqrt()
        out[:, q] = lg.logsumexp(-1) - lg.gather(1, tgt[:, q:q + 1])[:, 0]
        r = r - cbd[q][own[:, q]]
    return out


def _check_ce_bounds(codec, x, own, tgt, loss, frames_reduced):
    """The valid frames' CE entries (ns2_rvq_ce's scratch, on those frames alone) and the batch's loss, a reduction
    over `frames_reduced` frames, against float64."""
    from naturalspeech2_pytorch_b200 import _lib, ops
    cb = codec.codebooks
    F, Q = own.shape
    scratch = torch.empty(F * Q, device=dev)
    out = torch.empty((), device=dev)
    _lib.check(_lib.load().ns2_rvq_ce(x.data_ptr(), F, 128, cb.data_ptr(), codec._prep()[1].data_ptr(), Q,
                                      cb.shape[1], own.data_ptr(), tgt.data_ptr(), scratch.data_ptr(), out.data_ptr(),
                                      torch.cuda.current_stream().cuda_stream), "ns2_rvq_ce")
    got = scratch.view(F, Q)
    ce64 = _ce_entries(x, cb, own, tgt, torch.float64)
    ce32 = _ce_entries(x, cb, own, tgt, torch.float32).double()
    err32 = float((ce32 - ce64).abs().max())
    assert_close(got, ce64, ERR_MULT * err32 + FLOOR * float(ce64.abs().max()),
                 ERR_MULT * float((ce32 - ce64).norm() / ce64.norm()) + 1e-6, "valid frames' CE entries")
    _, loss64, _ = residual_vq_ce(x.double(), cb.double(), tgt, own=own)
    loss64 = float(loss64)
    reduce_err = sum(acc_eps(frames_reduced) * float(ce64[:, q].abs().sum()) / F for q in range(Q))
    lbound = ERR_MULT * abs(float(ce32.mean(0).sum()) - loss64) + FLOOR * abs(loss64) + reduce_err
    assert abs(loss - loss64) <= lbound, (loss, loss64, lbound)
    print(f"CE with latent_lens: loss {abs(loss - loss64) / lbound:.0%} of its bound")


def test_d_pred_past_the_lengths_is_exactly_zero(codec):
    from naturalspeech2_pytorch_b200 import ops
    from naturalspeech2_pytorch_b200.diffusion import XStartCrossEntropyFunction, gamma_to_alpha_sigma, \
        sigmoid_schedule
    x = _padded(B, N, LENS)
    lat, codes = _latents_alone(codec, x, LENS)
    g = torch.Generator(device=dev).manual_seed(6)
    pred = torch.randn(B, N, 128, device=dev, generator=g)
    audio_in = lat.clone()
    for b, n in enumerate(LENS):
        pred[b, n:] = NAN
        audio_in[b, n:] = NAN
    pred.requires_grad_(True)
    alpha, sigma = gamma_to_alpha_sigma(sigmoid_schedule(torch.rand(B, device=dev, generator=g)))
    lens = ops.lengths(LENS, B, N, device=dev)
    from naturalspeech2_pytorch_b200.codec import codes_past_lengths
    tgt = codes_past_lengths(codes, LENS)
    loss = XStartCrossEntropyFunction.apply(pred, audio_in, alpha.contiguous(), sigma.contiguous(), codec, tgt, "v",
                                            lens)
    (d_pred,) = torch.autograd.grad(loss, [pred])
    assert bool(torch.isfinite(loss)) and bool(torch.isfinite(d_pred).all())
    for b, n in enumerate(LENS):
        assert bool((d_pred[b, n:].view(torch.int32) == 0).all()), b   # +0.0, bit for bit
        assert int((d_pred[b, :n] != 0).sum()) > 0, b


# -------------------------------------------------------------------------------------------------------------------
# sampling
# -------------------------------------------------------------------------------------------------------------------
def test_sampling_with_raw_prompt_equals_alone_encoded_prompt(codec):
    from naturalspeech2_pytorch_b200 import Model, NaturalSpeech2
    from naturalspeech2_pytorch_b200.encoders import Conditioner
    torch.manual_seed(0)
    cn = Conditioner(dim_codebook=128, num_phoneme_tokens=NUM_TOKENS)
    with torch.no_grad():   # durations of a few frames per phoneme, so every sample has a condition
        head = cn.duration_pitch.to_duration_pred.to_pred[0]
        head.weight.mul_(0.05)
        head.bias.fill_(2.5)
    model = Model(dim=128, depth=1, heads=2, wavenet_layers=2, wavenet_stacks=1, dim_prompt=512,
                  condition_on_prompt=True)
    ns = NaturalSpeech2(model.to(dev).eval(), codec=codec, timesteps=3, conditioner=cn.to(dev).eval())
    g = torch.Generator().manual_seed(7)
    text = torch.randint(0, NUM_TOKENS, (B, T), generator=g).to(dev)
    noise = torch.randn(B, N, 128, generator=g).to(dev)
    prompt = _padded(B, NP, PROMPT_LENS)
    prompt_lat, _ = _latents_alone(codec, prompt, PROMPT_LENS, NP)
    kw = dict(length=N, text=text, prompt_lens=PROMPT_LENS, phoneme_lens=TEXT_LENS, noise=noise)
    got = ns.sample(prompt=prompt, **kw)
    want = ns.sample(prompt=prompt_lat, **kw)
    assert bool(torch.isfinite(got).all()) and torch.equal(got, want)
