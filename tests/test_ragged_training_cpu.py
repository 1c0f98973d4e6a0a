"""CPU: training with per-sample lengths refuses what it does not support before any launch: the key-padding attention
backward entry point with NULL arguments or together with dropout, lengths with the encoders' dropout or with the
duration / pitch predictor, durations past a sample's phonemes, and a raw-audio prompt with lengths."""
import ctypes
import re
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent


@pytest.fixture(scope="module")
def lib():
    from naturalspeech2_pytorch_b200 import _lib, build
    build.build()
    return _lib.load()


def test_attn_bwd_args_carry_kv_lens(lib):
    from naturalspeech2_pytorch_b200 import _lib
    header = (ROOT / "include" / "ns2_b200.h").read_text()
    fields = re.search(r"typedef struct ns2_attn_bwd_args \{([^}]*)\} ns2_attn_bwd_args;", header).group(1)
    assert re.search(r"\bconst int32_t\* kv_lens;", fields)
    assert "kv_lens" in dict(_lib.AttnBwdArgs._fields_)
    assert re.search(r"int ns2_attn_bwd\(const ns2_attn_bwd_args\* args, ns2_stream_t stream\);", header)
    assert _lib.SIGNATURES["ns2_attn_bwd"][1][0] is ctypes.POINTER(_lib.AttnBwdArgs)
    assert hasattr(lib, "ns2_attn_bwd")


def test_attn_bwd_with_kv_lens_rejects_null_arguments(lib):
    from naturalspeech2_pytorch_b200._lib import AttnBwdArgs
    before = lib.ns2_launch_count()
    assert lib.ns2_attn_bwd(None, None) < 0
    assert b"NULL" in lib.ns2_last_error()
    assert lib.ns2_attn_bwd(ctypes.byref(AttnBwdArgs(kv_lens=16)), None) < 0      # NULL q / k / v / ...
    assert b"NULL" in lib.ns2_last_error()
    assert lib.ns2_attn_bwd(ctypes.byref(AttnBwdArgs()), None) < 0                # without kv_lens
    assert lib.ns2_launch_count() == before


def test_attn_bwd_refuses_kv_lens_with_dropout(lib):
    from naturalspeech2_pytorch_b200 import ops
    from naturalspeech2_pytorch_b200._lib import AttnBwdArgs, Dropout
    before = lib.ns2_launch_count()
    d = Dropout(1, 0, 0.5)
    assert lib.ns2_attn_bwd(ctypes.byref(AttnBwdArgs(dropout=ctypes.pointer(d), kv_lens=16)), None) < 0
    assert b"kv_lens" in lib.ns2_last_error()
    B, N = 2, 8
    q = torch.zeros(B, N, 64, dtype=torch.bfloat16)
    kv = torch.zeros(B, 5, 64, dtype=torch.bfloat16)
    with pytest.raises(ValueError, match="kv_lens"):
        ops.attention_bwd(q, kv, kv.clone(), q.clone(), q.clone(), torch.zeros(B, 1, N), torch.zeros(B, N, 64),
                          kv.clone(), kv.clone(), heads=1, dropout=(1, 0, 0.5), kv_lens=torch.ones(B, dtype=torch.int32))
    assert lib.ns2_launch_count() == before


def _conditioner(**kw):
    from naturalspeech2_pytorch_b200.encoders import Conditioner
    return Conditioner(dim_codebook=128, num_phoneme_tokens=10, **kw)


def _train_call(cn, **kw):
    B, Np, T, L = 2, 6, 4, 12
    duration = torch.tensor([[2, 1, 1, 0], [3, 3, 0, 0]])
    args = dict(prompt=torch.zeros(B, Np, 128), text=torch.zeros(B, T, dtype=torch.long), mode="train",
                pitch=torch.ones(B, L), duration=duration, prompt_lens=[6, 3], phoneme_lens=[3, 2])
    args.update(kw)
    return cn(**args)


def test_conditioner_refusals(lib):
    before = lib.ns2_launch_count()
    cn = _conditioner()
    with pytest.raises(ValueError, match="phoneme_lens"):   # sample 0 has frames at phoneme 3 >= phoneme_lens[0]
        _train_call(cn, duration=torch.tensor([[2, 1, 1, 1], [3, 3, 0, 0]]))
    with pytest.raises(ValueError):                        # a length out of [1, T]
        _train_call(cn, phoneme_lens=[5, 2])
    with pytest.raises(NotImplementedError, match="train_duration_pitch"):
        _train_call(_conditioner(train_duration_pitch=True))
    with pytest.raises(NotImplementedError, match="train_dropout"):
        _train_call(_conditioner(train_dropout=True))
    with pytest.raises(NotImplementedError, match="train_dropout"):
        _train_call(_conditioner(train_dropout=True), phoneme_lens=None)
    with pytest.raises(NotImplementedError, match="duration"):   # the existing checks come first
        _train_call(cn, duration=None)
    assert lib.ns2_launch_count() == before


def test_natural_speech2_forward_refusals(lib):
    from naturalspeech2_pytorch_b200 import Model, NaturalSpeech2
    before = lib.ns2_launch_count()
    model = Model(dim=128, depth=1, heads=2, wavenet_layers=2, wavenet_stacks=1, dim_prompt=512,
                  condition_on_prompt=True)
    ns = NaturalSpeech2(model, target_sample_hz=24000, timesteps=2, conditioner=_conditioner())
    audio = torch.zeros(1, 8, 128)
    text = torch.zeros(1, 3, dtype=torch.long)
    with pytest.raises(ValueError, match="encoded latents"):
        ns(audio, text=text, prompt=torch.zeros(1, 4800), pitch=torch.ones(1, 8), duration=torch.ones(1, 3),
           prompt_lens=[1], phoneme_lens=[3])
    with pytest.raises(ValueError, match="phoneme_lens"):
        ns(audio, prompt_enc=torch.zeros(1, 4, 512), cond=torch.zeros(1, 512, 8), phoneme_lens=[3])
    uncond = NaturalSpeech2(Model(dim=128, depth=1, heads=2, wavenet_layers=2, wavenet_stacks=1),
                            target_sample_hz=24000, timesteps=2)
    with pytest.raises(ValueError, match="conditional"):
        uncond(audio, prompt_lens=[1])
    assert lib.ns2_launch_count() == before
