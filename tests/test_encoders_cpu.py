"""CPU: conditioning-encoder oracle against the reference goldens; drop-in surface (state_dict keys / shapes)."""
import numpy as np
import pytest
import torch

from helpers import DPP_CASES, ENCODER_CASES, build_encoder, dpp_case, encoder_case


@pytest.mark.parametrize("name", ENCODER_CASES)
def test_encoder_oracle_matches_reference_fp64(name):
    from oracle import encoders_oracle
    cls, kwargs, x, ref64, _, _ = encoder_case(name)
    enc = build_encoder(cls, kwargs)
    P = {k: v.double() for k, v in enc.state_dict().items()}
    if cls == "PhonemeEncoder":
        out = encoders_oracle.phoneme_encoder(P, x, heads=kwargs.get("heads", 8))
    else:
        out = encoders_oracle.speech_prompt_encoder(P, x.double(), heads=kwargs.get("heads", 8))
    assert np.abs(out.numpy() - ref64).max() < 1e-9


@pytest.mark.parametrize("name", ENCODER_CASES)
def test_encoder_state_dict_matches_reference(name):
    """Same keys, order and shapes as the reference module (recorded by make_golden.py from the reference itself)."""
    cls, kwargs, _, _, _, keys = encoder_case(name)
    enc = build_encoder(cls, kwargs)
    assert [(k, tuple(v.shape)) for k, v in enc.state_dict().items()] == [(k, tuple(s)) for k, s in keys]


def test_encoders_reject_cpu_inputs_and_masks():
    cls, kwargs, x, *_ = encoder_case("phon_small")
    enc = build_encoder(cls, kwargs)
    with pytest.raises(ValueError):
        enc(x)
    with pytest.raises(NotImplementedError):
        enc(x, mask=torch.ones_like(x, dtype=torch.bool))
    cls, kwargs, x, *_ = encoder_case("spe_small")
    with pytest.raises(ValueError):
        build_encoder(cls, kwargs)(x)


@pytest.mark.parametrize("name", DPP_CASES)
def test_duration_pitch_oracle_and_state_dict(name):
    from oracle import encoders_oracle
    kwargs, x, prompts, ref64, _, keys = dpp_case(name)
    enc = build_encoder("DurationPitchPredictor", kwargs)
    assert [(k, tuple(v.shape)) for k, v in enc.state_dict().items()] == [(k, tuple(s)) for k, s in keys]
    P = {k: v.double() for k, v in enc.state_dict().items()}
    dur, pitch = encoders_oracle.duration_pitch_predictor(P, x.double(), prompts.double(), heads=kwargs.get("heads", 8))
    assert np.abs(torch.stack((dur, pitch)).numpy() - ref64).max() < 1e-9


def test_length_regulation_oracle_and_host_glue_match_reference():
    """generate_mask_from_repeats / f0_to_coarse / expand_encodings: oracle == reference golden (bit-exact), and the
    product's torch glue (frame -> text index, coarse pitch bins) reproduces the reference's hard alignment."""
    from helpers import GOLDEN
    from naturalspeech2_pytorch_b200.encoders import f0_to_coarse, frames_to_text_index
    from oracle import encoders_oracle
    z = np.load(GOLDEN / "encoders.npz")
    ph, dur, pitch, table = (torch.from_numpy(z[f"expand_{k}"]) for k in ("phon", "duration", "pitch", "table"))
    np.testing.assert_array_equal(encoders_oracle.expand_encodings(ph, dur, pitch, table).numpy(), z["expand_cond"])
    idx = frames_to_text_index(dur)
    mask = encoders_oracle.generate_mask_from_repeats(dur)
    assert torch.equal(mask, idx.unsqueeze(1) == torch.arange(dur.shape[1]).view(1, -1, 1))
    assert torch.equal(f0_to_coarse(pitch), encoders_oracle.f0_to_coarse(pitch))


# ---- the constructor knobs beyond the defaults (tests/golden/make_golden_encoder_configs.py) ----
def _config_case(name):
    import ast
    from golden.make_golden_encoder_configs import ENCODER_CONFIG_CASES, encoder_config_inputs
    from helpers import GOLDEN
    z = np.load(GOLDEN / "encoder_configs.npz")
    cls, kwargs, _ = ENCODER_CONFIG_CASES[name]
    return (cls, dict(kwargs), encoder_config_inputs(name), z[f"{name}_fp64"], ast.literal_eval(str(z[f"{name}_keys"])),
            float(z["head_bias"]))


def _config_names():
    from golden.make_golden_encoder_configs import ENCODER_CONFIG_CASES
    return list(ENCODER_CONFIG_CASES)


@pytest.mark.parametrize("name", _config_names())
def test_encoder_oracle_matches_reference_at_other_configs(name):
    """Kernel sizes 1 ... 12, 16 ... 128 channels per GroupNorm group, heads x 64 != dim, 1- and 3-Block ResnetBlocks:
    the fp64 oracle equals the reference modules' fp64 outputs, and the state_dict has the reference's keys and shapes."""
    from oracle import encoders_oracle as eo
    cls, kwargs, x, ref64, keys, head_bias = _config_case(name)
    enc = build_encoder(cls, kwargs)
    assert [(k, tuple(v.shape)) for k, v in enc.state_dict().items()] == [(k, tuple(s)) for k, s in keys]
    P = {k: v.double() for k, v in enc.state_dict().items()}
    heads = kwargs.get("heads", 8)
    if cls == "SpeechPromptEncoder":
        out = eo.speech_prompt_encoder(P, x.double(), heads=heads, padding=kwargs["padding"])
    elif cls == "PhonemeEncoder":
        out = eo.phoneme_encoder(P, x, heads=heads)
    else:
        x, prompts = x
        for t in ("to_duration_pred", "to_pitch_pred"):
            P[f"{t}.to_pred.0.bias"].fill_(head_bias)
        h = P["phoneme_token_emb.weight"][x] if x.dtype == torch.int64 else x.double()
        out = torch.stack(eo.duration_pitch_predictor(P, h, prompts.double(), heads=heads))
        assert float(out.min()) > 0          # every row on the linear side of the ReLU
    assert np.abs(out.numpy() - ref64).max() < 1e-9


def test_encoder_constructors_accept_the_swept_configs_and_reject_their_neighbours():
    """Every configuration of tests/test_encoder_configs_fp64_gpu.py constructs; the nearest unsupported ones raise
    NotImplementedError in the constructor, before any kernel could launch."""
    from naturalspeech2_pytorch_b200.encoders import DurationPitchPredictor, PhonemeEncoder, SpeechPromptEncoder
    from restatements import ENCODER_CONFIGS as CONFIGS
    from naturalspeech2_pytorch_b200 import encoders
    for cls, kw, _, _ in CONFIGS.values():
        getattr(encoders, cls)(**kw)
    spe = dict(dim_codebook=128, dims=(256,), depth=1, heads=4)
    phon = dict(num_tokens=30, dim=256, dim_hidden=256, depth=1, heads=2)
    dpp = dict(dim=256, dim_hidden=256, depth=1, heads=2)
    bad = [
        (SpeechPromptEncoder, dict(spe, kernel_size=13, padding=6)),        # more taps than NS2_GEMM_MAX_SEGS
        (PhonemeEncoder, dict(phon, kernel_size=13)),
        (DurationPitchPredictor, dict(dpp, kernel_size=13)),
        (DurationPitchPredictor, dict(dpp, kernel_size=4)),                 # even predictor kernel
        (SpeechPromptEncoder, dict(spe, kernel_size=3, padding=2)),         # 2 padding != k - 1
        (SpeechPromptEncoder, dict(spe, kernel_size=12, padding=5)),
        (SpeechPromptEncoder, dict(spe, dims=(96, 256))),                   # channels not a multiple of 64
        (SpeechPromptEncoder, dict(spe, dim_codebook=96)),
        (PhonemeEncoder, dict(phon, dim=96)),
        (SpeechPromptEncoder, dict(spe, dims=(192,))),                      # transformer width not a multiple of 128
        (PhonemeEncoder, dict(phon, dim_hidden=192)),
        (DurationPitchPredictor, dict(dpp, dim=192, dim_hidden=192)),
        (SpeechPromptEncoder, dict(spe, dims=(1152,))),                     # ... or above 1024
        (PhonemeEncoder, dict(phon, dim_hidden=1152)),
        (DurationPitchPredictor, dict(dpp, dim=1152, dim_hidden=1152)),
        (SpeechPromptEncoder, dict(spe, dim_head=32)),                      # dim_head != 64
        (PhonemeEncoder, dict(phon, dim_head=128)),
        (DurationPitchPredictor, dict(dpp, dim_head=32)),
    ]
    for cls, kw in bad:
        with pytest.raises(NotImplementedError):
            cls(**kw)
