"""CPU: the SEANet encoder's torch oracle against the committed transformers goldens, the module's state_dict layout,
configuration and input checks, `EncodecRVQ.from_state_dict`, and host-side argument validation of
`ns2_seanet_head`."""
import re
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from golden.make_golden_seanet_encoder import CASES, audio, filled_state_dict
import seanet_oracle


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(golden_dir / "seanet_encoder.npz")


@pytest.fixture(scope="module")
def keys_shapes(golden):
    return [(k, tuple(int(v) for v in s.split(","))) for k, s in zip(golden["keys"], golden["shapes"])]


@pytest.mark.parametrize("case", sorted(CASES))
def test_oracle_matches_transformers_fp64(golden, keys_shapes, case):
    B, N = CASES[case]
    f = seanet_oracle.encode(filled_state_dict(keys_shapes), audio(B, N), dtype=torch.float64)
    assert tuple(f.shape) == (B, N, 128)
    ref = torch.from_numpy(golden[f"{case}_f64"])
    assert float((f - ref).abs().max()) <= 1e-9 * max(1.0, float(ref.abs().max()))


def test_oracle_bf16_emulation_error_is_the_autocast_scale(golden, keys_shapes):
    """The bf16-operand emulation lands at the same error scale as transformers under CPU autocast (within 2x)."""
    sd = filled_state_dict(keys_shapes)
    f64 = seanet_oracle.encode(sd, audio(2, 75))
    fem = seanet_oracle.encode(sd, audio(2, 75), emulate_bf16=True)
    rel = float((fem - f64).norm() / f64.norm())
    auto = float(golden["b2n75_err"][2])
    assert auto / 2 < rel < 2 * auto, (rel, auto)


def test_state_dict_layout_matches_transformers(keys_shapes):
    from naturalspeech2_pytorch_b200 import SEANetEncoder
    enc = SEANetEncoder()
    mine = [(k, tuple(v.shape)) for k, v in enc.state_dict().items()]
    assert sorted(mine) == sorted(keys_shapes)
    assert len(mine) == 62 and sum(int(np.prod(s)) for _, s in mine) == 7425792
    enc.load_state_dict({k: v.float() for k, v in filled_state_dict(keys_shapes).items()})


def test_encodec_key_mapping_round_trip(keys_shapes):
    """Meta encodec names -> transformers names, on names built from the upstream module layout."""
    from naturalspeech2_pytorch_b200 import SEANetEncoder
    sd = {k: v.float() for k, v in filled_state_dict(keys_shapes).items()}
    meta = {}
    for k, v in sd.items():
        k = k.replace("parametrizations.weight.original0", "weight_g").replace("parametrizations.weight.original1",
                                                                             "weight_v")
        i = int(k.split(".")[1])
        rest = k.split(".", 2)[2]
        if rest.startswith("conv."):
            rest = "conv." + rest
        elif rest.startswith(("block.", "shortcut.")):
            rest = rest.replace(".conv.", ".conv.conv.", 1)
        meta[f"encoder.model.{i}.{rest}"] = v
    assert "encoder.model.3.conv.conv.weight_g" in meta and "encoder.model.13.lstm.weight_hh_l1" in meta
    enc = SEANetEncoder()
    enc.load_encodec_state_dict(meta)
    for k, v in enc.state_dict().items():
        assert torch.equal(v, sd[k]), k
    with pytest.raises(KeyError):
        SEANetEncoder().load_encodec_state_dict({"encoder.layers.0.conv.bias": torch.zeros(32)})


@pytest.mark.parametrize("field,value", [("audio_channels", 2), ("upsampling_ratios", (8, 5, 4, 4)),
                                         ("use_causal_conv", False), ("norm_type", "time_group_norm"),
                                         ("pad_mode", "constant"), ("num_residual_layers", 2), ("compress", 4),
                                         ("num_lstm_layers", 1), ("hidden_size", 64), ("use_conv_shortcut", False),
                                         ("num_filters", 64), ("kernel_size", 5)])
def test_unsupported_configuration_is_rejected(field, value):
    from naturalspeech2_pytorch_b200 import SEANetEncoder
    with pytest.raises(ValueError, match=field):
        SEANetEncoder(**{field: value})


def test_from_config_takes_the_24khz_defaults():
    from naturalspeech2_pytorch_b200 import SEANetEncoder
    from naturalspeech2_pytorch_b200.seanet import SUPPORTED
    enc = SEANetEncoder.from_config(SimpleNamespace(**SUPPORTED, sampling_rate=24000, codebook_size=1024))
    assert isinstance(enc, SEANetEncoder)
    with pytest.raises(ValueError):
        SEANetEncoder.from_config(SimpleNamespace(**{**SUPPORTED, "upsampling_ratios": [8, 6, 4, 2]}))


def test_from_state_dict_takes_the_encodec_model_layout(golden, keys_shapes):
    """Every EncodecModel key under encoder. / decoder. is one of the SEANet modules' keys, and the codebooks come from
    quantizer.layers.{q}.codebook.embed for the first num_quantizers stages."""
    from naturalspeech2_pytorch_b200 import EncodecRVQ, SEANetDecoder, SEANetEncoder
    model_keys = [str(k) for k in golden["model_keys"]]
    enc_sd = {k: v.float() for k, v in filled_state_dict(keys_shapes).items()}
    dec_shapes = {k: v.shape for k, v in SEANetDecoder().state_dict().items()}
    assert sorted(k[len("encoder."):] for k in model_keys if k.startswith("encoder.")) == sorted(enc_sd)
    assert sorted(k[len("decoder."):] for k in model_keys if k.startswith("decoder.")) == sorted(dec_shapes)
    sd = {}
    for k in model_keys:
        if k.startswith("encoder."):
            sd[k] = enc_sd[k[len("encoder."):]]
        elif k.startswith("decoder."):
            sd[k] = torch.randn(dec_shapes[k[len("decoder."):]])
        elif k.endswith(".codebook.embed"):
            sd[k] = torch.full((1024, 128), float(int(k.split(".")[2])))
        else:
            sd[k] = torch.zeros(1)
    for nq in (8, 4):
        codec = EncodecRVQ.from_state_dict(sd, num_quantizers=nq)
        assert isinstance(codec.encoder, SEANetEncoder) and isinstance(codec.decoder, SEANetDecoder)
        assert codec.num_quantizers == nq and tuple(codec.codebooks.shape) == (nq, 1024, 128)
        assert [float(codec.codebooks[q, 0, 0]) for q in range(nq)] == [float(q) for q in range(nq)]
    for k, v in codec.encoder.state_dict().items():
        assert torch.equal(v, enc_sd[k]), k
    for k, v in codec.decoder.state_dict().items():
        assert torch.equal(v, sd["decoder." + k]), k


@pytest.mark.parametrize("shape", [(2, 321), (2, 160), (1, 1, 330), (2, 2, 320), (320,), (1, 1, 1, 320)])
def test_bad_lengths_and_ranks_are_rejected(shape):
    from naturalspeech2_pytorch_b200 import SEANetEncoder
    with pytest.raises(ValueError):
        SEANetEncoder()(torch.zeros(shape))


def test_empty_input_returns_empty_frames_without_a_launch():
    from naturalspeech2_pytorch_b200 import SEANetEncoder
    enc = SEANetEncoder()
    assert tuple(enc(torch.zeros(0, 640)).shape) == (0, 2, 128)
    assert tuple(enc(torch.zeros(3, 1, 0)).shape) == (3, 0, 128)


@pytest.fixture(scope="module")
def lib():
    from naturalspeech2_pytorch_b200 import _lib, build
    build.build()
    return _lib.load()


def test_seanet_head_rejects_bad_arguments_before_launch(lib):
    """Dummy non-NULL pointers are never dereferenced: every check is host-side and no kernel is launched.
    Arguments: x, x_batch_stride, batch, length, params, out, out_row_stride, out_batch_stride, stream."""
    before = lib.ns2_launch_count()
    assert lib.ns2_seanet_head(256, 1000, -1, 1000, 256, 512, 32, 32 * 1002, None) < 0      # negative batch
    assert b"negative" in lib.ns2_last_error()
    assert lib.ns2_seanet_head(256, 1000, 70000, 1000, 256, 512, 32, 32 * 1002, None) < 0   # batch above 65535
    assert lib.ns2_seanet_head(None, 1000, 2, 1000, 256, 512, 32, 32 * 1002, None) < 0      # NULL x
    assert lib.ns2_seanet_head(256, 999, 2, 1000, 256, 512, 32, 32 * 1002, None) < 0        # x rows overlap
    assert b"batch stride" in lib.ns2_last_error()
    assert lib.ns2_seanet_head(258, 1000, 2, 1000, 256, 512, 32, 32 * 1002, None) < 0       # x misaligned
    assert lib.ns2_seanet_head(256, 1000, 2, 1000, 260, 512, 32, 32 * 1002, None) < 0       # params misaligned
    assert lib.ns2_seanet_head(256, 1000, 2, 1000, 256, 520, 32, 32 * 1002, None) < 0       # out misaligned
    assert lib.ns2_seanet_head(256, 1000, 2, 1000, 256, 512, 16, 16 * 1002, None) < 0       # fewer than 32 channels
    assert lib.ns2_seanet_head(256, 1000, 2, 1000, 256, 512, 36, 36 * 1002, None) < 0       # row stride % 8
    assert lib.ns2_seanet_head(256, 1000, 2, 1000, 256, 512, 32, 32 * 1002 + 4, None) < 0   # batch stride % 8
    assert lib.ns2_seanet_head(256, 1000, 2, 1000, 256, 512, 32, 32 * 1001, None) < 0       # out rows overlap
    assert lib.ns2_seanet_head(None, 0, 0, 1000, None, None, 0, 0, None) == 0               # empty: nothing to do
    assert lib.ns2_seanet_head(None, 0, 2, 0, None, None, 0, 0, None) == 0
    assert lib.ns2_launch_count() == before


def test_head_params_constant_matches_header():
    from naturalspeech2_pytorch_b200 import _lib
    h = (Path(__file__).resolve().parent.parent / "include" / "ns2_b200.h").read_text()
    assert int(re.search(r"#define NS2_SEANET_HEAD_PARAMS (\d+)", h).group(1)) == _lib.NS2_SEANET_HEAD_PARAMS
    assert _lib.NS2_SEANET_HEAD_PARAMS == 7 * 32 + 32 + 3 * 32 * 16 + 16 + 32 * 32 + 16 * 32 + 32


def test_pack_head_layout():
    """pack_head's blocks at the offsets the kernel reads (include/ns2_b200.h section 10)."""
    from naturalspeech2_pytorch_b200.seanet import pack_head
    g = torch.Generator().manual_seed(3)
    w0, b0 = torch.randn(32, 1, 7, generator=g), torch.randn(32, generator=g)
    w3, b3 = torch.randn(16, 32, 3, generator=g), torch.randn(16, generator=g)
    w1, b1 = torch.randn(32, 16, 1, generator=g), torch.randn(32, generator=g)
    ws, bs = torch.randn(32, 32, 1, generator=g), torch.randn(32, generator=g)
    p = pack_head(w0, b0, w3, b3, w1, b1, ws, bs)
    assert float(p[5 * 32 + 7]) == float(w0[7, 0, 5])                       # w0 [tap][out]
    assert float(p[224 + 3]) == float(b0[3])
    assert float(p[256 + (2 * 32 + 9) * 16 + 4]) == float(w3[4, 9, 2])      # w3 [tap][in][out]
    assert float(p[1792 + 15]) == float(b3[15])
    assert float(p[1808 + 6 * 32 + 30]) == float(ws[30, 6, 0])              # wsc [in][out]
    assert float(p[2832 + 11 * 32 + 1]) == float(w1[1, 11, 0])              # wc1 [in][out]
    assert float(p[3344 + 8]) == float(bs[8] + b1[8])
