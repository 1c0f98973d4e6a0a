"""CPU: per-sample lengths of a padded waveform batch (`SEANetEncoder.forward(lengths=)`,
`EncodecRVQ.forward(lengths=)`, `EncodecRVQ.quantize(lengths=)`, and `NaturalSpeech2` taking raw audio and raw prompts
with lengths) are refused before any launch when malformed: wrong dtype, device or count, outside [7, N] frames, more
than 64 samples, or a waveform shorter than its lengths.  The minimum of 7 frames is derived here from the encoder's
own layer table.  Without an EncodecRVQ codec the refusals keep their wording."""
import pytest
import torch

from naturalspeech2_pytorch_b200 import _lib, build as _build
from naturalspeech2_pytorch_b200.seanet import MIN_FRAMES, _ResnetParams, _WNConv


@pytest.fixture(scope="module")
def lib():
    _build.build()
    return _lib.load()


def _codec():
    from naturalspeech2_pytorch_b200 import EncodecRVQ, SEANetEncoder
    return EncodecRVQ(torch.zeros(8, 1024, 128), encoder=SEANetEncoder())


def test_min_frames_follows_from_the_stage_paddings():
    """Each conv pads k - stride samples on the left at its input rate; Encodec reflects only inputs longer than the
    pad, so n frames must give every conv more than `pad` input rows: n * rate > pad."""
    from naturalspeech2_pytorch_b200 import SEANetEncoder
    convs, rate = [], 320
    for layer in SEANetEncoder().layers:
        blocks = [layer] if isinstance(layer, _WNConv) else \
            [layer.block[1], layer.block[3], layer.shortcut] if isinstance(layer, _ResnetParams) else []
        for conv in blocks:
            k, s = conv.conv.kernel_size[0], conv.conv.stride[0]
            convs.append((k - s, rate))
        if isinstance(layer, _WNConv):
            rate //= layer.conv.stride[0]
    assert rate == 1
    need = max(pad // r + 1 for pad, r in convs)
    assert need == MIN_FRAMES == 7
    assert (6, 1) in convs   # the binding one: the last k7 conv at the frame rate


BAD_LENGTHS = [
    ("dtype", lambda B: torch.full((B,), 8.0), "integers"),
    ("device", lambda B: torch.full((B,), 8, dtype=torch.int32, device="meta"), "device"),
    ("count", lambda B: [8] * (B + 1), "one length per sample"),
    ("below 7", lambda B: [6] + [8] * (B - 1), ">= 7"),
    ("zero", lambda B: [0] * B, ">= 7"),
    ("past the waveform", lambda B: [11] + [8] * (B - 1), "fewer than the longest"),
    ("rank", lambda B: torch.full((B, 1), 8, dtype=torch.int32), "one-dimensional"),
]


@pytest.mark.parametrize("case", [c[0] for c in BAD_LENGTHS])
def test_encoder_and_codec_refuse_bad_lengths_before_any_launch(lib, case):
    from naturalspeech2_pytorch_b200 import SEANetEncoder
    _, make, match = next(c for c in BAD_LENGTHS if c[0] == case)
    B, N = 3, 10
    audio = torch.zeros(B, 320 * N)
    codec = _codec()
    before = lib.ns2_launch_count()
    with pytest.raises(ValueError, match=match):
        SEANetEncoder()(audio, lengths=make(B))
    with pytest.raises(ValueError, match=match):
        codec(audio, return_encoded=True, lengths=make(B))
    with pytest.raises(ValueError, match=match):   # a partial last frame is dropped, never counted
        codec(torch.zeros(B, 320 * N + 319), lengths=make(B))
    assert lib.ns2_launch_count() == before


def test_quantize_refuses_bad_lengths_before_any_launch(lib):
    codec = _codec()
    frames = torch.zeros(2, 5, 128)
    before = lib.ns2_launch_count()
    for bad, match in (([0, 5], ">= 1"), ([5, 6], "fewer than the longest"), ([5], "one length per sample"),
                       (torch.tensor([1.0, 2.0]), "integers")):
        with pytest.raises(ValueError, match=match):
            codec.quantize(frames, lengths=bad)
    with pytest.raises(ValueError, match=r"\(B, N, 128\)"):
        codec.quantize(frames.view(10, 128), lengths=[1] * 10)
    assert lib.ns2_launch_count() == before


def test_more_than_64_samples_are_refused(lib):
    from naturalspeech2_pytorch_b200 import SEANetEncoder
    codec = _codec()
    before = lib.ns2_launch_count()
    with pytest.raises(ValueError, match="at most 64 samples"):
        SEANetEncoder()(torch.zeros(65, 320 * 7), lengths=[7] * 65)
    with pytest.raises(ValueError, match="at most 64 samples"):
        codec(torch.zeros(65, 320 * 7), lengths=[7] * 65)
    with pytest.raises(ValueError, match="at most 64 samples"):
        codec.quantize(torch.zeros(65, 7, 128), lengths=[7] * 65)
    assert lib.ns2_launch_count() == before


def test_natural_speech2_refuses_bad_raw_lengths_before_any_launch(lib):
    from naturalspeech2_pytorch_b200 import Model, NaturalSpeech2
    from naturalspeech2_pytorch_b200.encoders import Conditioner
    before = lib.ns2_launch_count()
    ns = NaturalSpeech2(Model(dim=128, depth=1, heads=2, wavenet_layers=1, wavenet_stacks=1), codec=_codec(),
                        timesteps=3, rvq_cross_entropy_loss_weight=0.5)
    with pytest.raises(ValueError, match=">= 7"):
        ns(torch.zeros(2, 3200), latent_lens=[6, 10])
    with pytest.raises(ValueError, match="fewer than the longest"):
        ns(torch.zeros(2, 3200), latent_lens=[8, 11])
    model = Model(dim=128, depth=1, heads=2, wavenet_layers=2, wavenet_stacks=1, dim_prompt=512,
                  condition_on_prompt=True)
    cn = Conditioner(dim_codebook=128, num_phoneme_tokens=10)
    nc = NaturalSpeech2(model, codec=_codec(), timesteps=2, conditioner=cn)
    text = torch.zeros(1, 3, dtype=torch.long)
    with pytest.raises(ValueError, match=">= 7"):
        nc.sample(length=8, prompt=torch.zeros(1, 4800), text=text, prompt_lens=[5], phoneme_lens=[3])
    with pytest.raises(ValueError, match="fewer than the longest"):
        nc(torch.zeros(1, 8, 128), text=text, prompt=torch.zeros(1, 4800), pitch=torch.ones(1, 8),
           duration=torch.ones(1, 3), prompt_lens=[16], phoneme_lens=[3])
    assert lib.ns2_launch_count() == before


def test_refusals_without_an_encodec_codec_keep_their_wording(lib):
    from naturalspeech2_pytorch_b200 import Model, NaturalSpeech2
    from naturalspeech2_pytorch_b200.encoders import Conditioner
    before = lib.ns2_launch_count()
    model = Model(dim=128, depth=1, heads=2, wavenet_layers=1, wavenet_stacks=1)
    for codec in (None, _OtherCodec()):
        kw = dict(codec=codec) if codec is not None else dict(target_sample_hz=24000)
        ns = NaturalSpeech2(model, timesteps=3, **kw)
        with pytest.raises(ValueError, match="encoded latents"):
            ns(torch.zeros(2, 3200), latent_lens=[8, 10])
        ns.rvq_cross_entropy_loss_weight = 0.5
        with pytest.raises(NotImplementedError, match="cross-entropy"):
            ns(torch.zeros(2, 10, 128), codes=torch.zeros(2, 10, 8, dtype=torch.long), latent_lens=[8, 10])
    cmodel = Model(dim=128, depth=1, heads=2, wavenet_layers=2, wavenet_stacks=1, dim_prompt=512,
                   condition_on_prompt=True)
    nc = NaturalSpeech2(cmodel, target_sample_hz=24000, timesteps=2,
                        conditioner=Conditioner(dim_codebook=128, num_phoneme_tokens=10))
    with pytest.raises(ValueError, match="encoded latents"):
        nc.sample(length=8, prompt=torch.zeros(1, 4800), text=torch.zeros(1, 3, dtype=torch.long), prompt_lens=[8])
    # an EncodecRVQ without an encoder takes no raw audio either
    from naturalspeech2_pytorch_b200 import EncodecRVQ
    ne = NaturalSpeech2(model, codec=EncodecRVQ(torch.zeros(8, 1024, 128)), timesteps=3)
    with pytest.raises(ValueError, match="encoded latents"):
        ne(torch.zeros(2, 3200), latent_lens=[8, 10])
    assert lib.ns2_launch_count() == before


class _OtherCodec:
    """A codec with EncodecWrapper's attributes that is not an EncodecRVQ."""
    target_sample_hz, seq_len_multiple_of, codebook_dim = 24000, 320, 128
