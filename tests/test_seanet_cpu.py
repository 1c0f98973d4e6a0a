"""CPU: the SEANet decoder's torch oracle against the committed transformers goldens, the module's state_dict layout,
configuration checks, and host-side argument validation of the decoder's C-ABI entry points."""
import ctypes

import numpy as np
import pytest
import torch

from golden.make_golden_seanet import CASES, filled_state_dict, latents
import seanet_oracle


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(golden_dir / "seanet_decoder.npz")


@pytest.fixture(scope="module")
def keys_shapes(golden):
    return [(k, tuple(int(v) for v in s.split(","))) for k, s in zip(golden["keys"], golden["shapes"])]


@pytest.mark.parametrize("case", sorted(CASES))
def test_oracle_matches_transformers_fp64(golden, keys_shapes, case):
    B, N = CASES[case]
    sd = filled_state_dict(keys_shapes)
    y = seanet_oracle.decode(sd, latents(B, N), dtype=torch.float64)
    assert tuple(y.shape) == (B, 1, 320 * N)
    ref = torch.from_numpy(golden[f"{case}_f64s"])
    got = y[..., ::int(golden["stride"])]
    assert float((got - ref).abs().max()) <= 1e-9 * max(1.0, float(ref.abs().max()))


def test_oracle_bf16_emulation_error_is_the_autocast_scale(golden, keys_shapes):
    """The bf16-operand emulation lands at the same error scale as transformers under CPU autocast (within 2x)."""
    sd = filled_state_dict(keys_shapes)
    y64 = seanet_oracle.decode(sd, latents(2, 75))
    yem = seanet_oracle.decode(sd, latents(2, 75), emulate_bf16=True)
    rel = float((yem - y64).norm() / y64.norm())
    auto = float(golden["b2n75_err"][2])
    assert auto / 2 < rel < 2 * auto, (rel, auto)


def test_state_dict_layout_matches_transformers(keys_shapes):
    from naturalspeech2_pytorch_b200 import SEANetDecoder
    dec = SEANetDecoder()
    mine = [(k, tuple(v.shape)) for k, v in dec.state_dict().items()]
    assert sorted(mine) == sorted(keys_shapes)
    assert len(mine) == 62 and sum(int(np.prod(s)) for _, s in mine) == 7426018
    dec.load_state_dict({k: v.float() for k, v in filled_state_dict(keys_shapes).items()})


def test_encodec_key_mapping_round_trip(keys_shapes):
    """Meta encodec names -> transformers names, on names built from the upstream module layout."""
    from naturalspeech2_pytorch_b200 import SEANetDecoder
    sd = {k: v.float() for k, v in filled_state_dict(keys_shapes).items()}
    meta = {}
    for k, v in sd.items():
        k = k.replace("parametrizations.weight.original0", "weight_g").replace("parametrizations.weight.original1",
                                                                             "weight_v")
        i = int(k.split(".")[1])
        rest = k.split(".", 2)[2]
        if i in (3, 6, 9, 12):
            rest = rest.replace("conv.", "convtr.convtr.", 1)
        elif rest.startswith("conv."):
            rest = "conv." + rest
        elif rest.startswith(("block.", "shortcut.")):
            rest = rest.replace(".conv.", ".conv.conv.", 1)
        meta[f"decoder.model.{i}.{rest}"] = v
    dec = SEANetDecoder()
    dec.load_encodec_state_dict(meta)
    for k, v in dec.state_dict().items():
        assert torch.equal(v, sd[k]), k


@pytest.mark.parametrize("field,value", [("audio_channels", 2), ("upsampling_ratios", (8, 5, 4, 4)),
                                         ("use_causal_conv", False), ("norm_type", "time_group_norm"),
                                         ("pad_mode", "constant"), ("num_residual_layers", 2), ("compress", 4),
                                         ("num_lstm_layers", 1), ("hidden_size", 64), ("use_conv_shortcut", False)])
def test_unsupported_configuration_is_rejected(field, value):
    from naturalspeech2_pytorch_b200 import SEANetDecoder
    with pytest.raises(ValueError, match=field):
        SEANetDecoder(**{field: value})


def test_from_config_takes_the_24khz_defaults():
    from types import SimpleNamespace
    from naturalspeech2_pytorch_b200 import SEANetDecoder
    from naturalspeech2_pytorch_b200.seanet import SUPPORTED
    SEANetDecoder.from_config(SimpleNamespace(**SUPPORTED))
    with pytest.raises(ValueError):
        SEANetDecoder.from_config(SimpleNamespace(**{**SUPPORTED, "upsampling_ratios": [8, 6, 4, 2]}))


def test_lstm_gate_permutation_is_a_permutation():
    from naturalspeech2_pytorch_b200.seanet import lstm_gate_perm
    p = lstm_gate_perm()
    assert sorted(p.tolist()) == list(range(2048))
    # CTA 1, first warp, unit 0: gates i, f, g, o of hidden unit 32
    assert [int(p[128 + r]) for r in (0, 8, 64, 72)] == [32, 512 + 32, 1024 + 32, 1536 + 32]


@pytest.fixture(scope="module")
def lib():
    from naturalspeech2_pytorch_b200 import _lib, build
    build.build()
    return _lib.load()


def test_new_entry_points_reject_bad_sizes_before_launch(lib):
    """Dummy non-NULL pointers are never dereferenced: every check is host-side and no kernel is launched."""
    before = lib.ns2_launch_count()
    # LSTM: hidden must be 512, xproj rows must hold 4 * hidden values, w_hh 16-byte aligned, an output required
    assert lib.ns2_lstm_seq(256, 2048, 2048 * 4, 256, 2, 4, 256, None, 0, 0, 1024, 512, 2048, None, 0, 0, None) < 0
    assert b"hidden=256" in lib.ns2_last_error()
    assert lib.ns2_lstm_seq(256, 1024, 2048 * 4, 256, 2, 4, 512, None, 0, 0, 1024, 512, 2048, None, 0, 0, None) < 0
    assert b"row stride" in lib.ns2_last_error()
    assert lib.ns2_lstm_seq(256, 2048, 2048 * 4, 258, 2, 4, 512, None, 0, 0, 1024, 512, 2048, None, 0, 0, None) < 0
    assert lib.ns2_lstm_seq(256, 2048, 2048 * 4, 256, 2, 4, 512, None, 0, 0, None, 0, 0, None, 0, 0, None) < 0
    assert lib.ns2_lstm_seq(None, 0, 0, None, 0, 4, 512, None, 0, 0, None, 0, 0, None, 0, 0, None) == 0  # empty
    # elu_pad: channels % 4, unknown flags, misaligned strides
    assert lib.ns2_elu_pad(256, 30, 300, 2, 10, 30, 6, 1, 512, 32, 512, None) < 0
    assert b"channels=30" in lib.ns2_last_error()
    assert lib.ns2_elu_pad(256, 32, 320, 2, 10, 32, 6, 4, 512, 32, 512, None) < 0
    assert b"flags" in lib.ns2_last_error()
    assert lib.ns2_elu_pad(256, 34, 340, 2, 10, 32, 6, 1, 512, 32, 512, None) < 0
    assert lib.ns2_elu_pad(256, 32, 320, 2, 10, 32, 6, 1, 514, 32, 512, None) < 0
    # tail: 32-channel rows, aligned parameters
    assert lib.ns2_seanet_tail(256, 16, 160, 2, 10, 256, 512, 10, None) < 0
    assert lib.ns2_seanet_tail(256, 32, 320, 2, 10, 260, 512, 10, None) < 0
    assert lib.ns2_seanet_tail(256, 32, 320, 70000, 10, 256, 512, 10, None) < 0
    assert lib.ns2_launch_count() == before


def test_abi_constants_match_header():
    import re
    from pathlib import Path
    from naturalspeech2_pytorch_b200 import _lib
    h = (Path(__file__).resolve().parent.parent / "include" / "ns2_b200.h").read_text()
    for name in ("NS2_ELU_PAD_ELU", "NS2_ELU_PAD_RAW", "NS2_SEANET_TAIL_PARAMS", "NS2_ABI_VERSION"):
        assert int(re.search(rf"#define {name} (\d+)", h).group(1)) == getattr(_lib, name), name
    assert ctypes.sizeof(ctypes.c_int64) == 8
