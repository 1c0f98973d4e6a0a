"""The packed-weight cache shared by the denoiser and the encoders (`model._PackedCache`), on CPU: when `packed()` and
`packed_transposed()` are rebuilt, and the layout of the transposed conv packs the backward's dgrad GEMMs read."""
import pytest
import torch

from naturalspeech2_pytorch_b200 import Model
from naturalspeech2_pytorch_b200.encoders import PhonemeEncoder, SpeechPromptEncoder

MODULES = {
    "model_uncond": lambda: Model(dim=128, depth=1, heads=2, wavenet_layers=2, wavenet_stacks=1),
    "model_cond": lambda: Model(dim=128, depth=1, heads=2, wavenet_layers=2, wavenet_stacks=1, dim_prompt=192,
                                condition_on_prompt=True, resampler_depth=1),
    "prompt_encoder": lambda: SpeechPromptEncoder(dim_codebook=64, dims=(128, 128), depth=1, heads=2),
    "phoneme_encoder": lambda: PhonemeEncoder(num_tokens=10, dim=64, dim_hidden=128, depth=1, heads=2),
}


def _conv_packs(m):
    """(forward pack key, Conv1d weight (O, I, k)) of every conv whose transposed pack `_transpose_conv` builds."""
    if isinstance(m, Model):
        return [("wn_init_w", m.wavenet.init_conv.weight)] + [
            (f"l{l}_ff_wc", layer[5][2][1].weight) for l, layer in enumerate(m.transformer.layers)]
    if isinstance(m, SpeechPromptEncoder):
        return [(f"c{i}_w", c.weight) for i, c in enumerate(m._convs()) if i > 0]
    return [("c_w", m.conv[1].weight)]


@pytest.fixture(params=sorted(MODULES))
def module(request):
    torch.manual_seed(0)
    return MODULES[request.param]()


def _rebuilt(m, P, T):
    """Whether packed() was rebuilt since (P, T), checking that packed_transposed() was rebuilt exactly with it."""
    P2, T2 = m.packed(), m.packed_transposed()
    assert (P2 is P) == (T2 is T)
    return P2 is not P, P2, T2


def test_cached_while_parameters_are_unchanged(module):
    P, T = module.packed(), module.packed_transposed()
    assert module.packed() is P and module.packed_transposed() is T
    assert not _rebuilt(module, P, T)[0]


def test_rebuilt_after_in_place_update(module):
    P, T = module.packed(), module.packed_transposed()
    key, w = _conv_packs(module)[0]
    with torch.no_grad():
        w.add_(1.0)   # bumps the version counter, like an optimizer step
    rebuilt, P2, _ = _rebuilt(module, P, T)
    assert rebuilt
    assert not torch.equal(P[key], P2[key])


def test_rebuilt_after_load_state_dict(module):
    P, T = module.packed(), module.packed_transposed()
    module.load_state_dict(module.state_dict())
    assert _rebuilt(module, P, T)[0]


@pytest.mark.parametrize("convert", [lambda m: m.float(), lambda m: m.to("cpu")], ids=["float", "to"])
def test_rebuilt_after_module_conversion(module, convert):
    P, T = module.packed(), module.packed_transposed()
    assert convert(module) is module
    assert _rebuilt(module, P, T)[0]


def test_invalidate_packed(module):
    P, T = module.packed(), module.packed_transposed()
    module.invalidate_packed()
    assert _rebuilt(module, P, T)[0]


def test_freeze_packed_skips_the_version_check():
    torch.manual_seed(0)
    m = MODULES["model_uncond"]()
    m.freeze_packed = True
    P, T = m.packed(), m.packed_transposed()
    with torch.no_grad():
        next(m.parameters()).add_(1.0)
    assert not _rebuilt(m, P, T)[0]
    m.freeze_packed = False
    assert _rebuilt(m, P, T)[0]


def test_transposed_conv_packs_are_in_tap_out(module):
    P, T = module.packed(), module.packed_transposed()
    packs = _conv_packs(module)
    assert packs
    for key, w in packs:
        O, I, k = w.shape
        fwd, tr = P[key], T[key]
        o_pad, i_pad = fwd.shape[0], fwd.shape[1] // k
        # forward pack: tap t of w at columns [t*i_pad, t*i_pad + I), zero padding elsewhere
        ref = torch.zeros(o_pad, k, i_pad)
        ref[:O, :, :I] = w.detach().permute(0, 2, 1)
        assert torch.equal(fwd, ref.reshape(o_pad, k * i_pad).bfloat16()), key
        # transposed pack: [in][tap][out]
        assert tr.shape == (i_pad, k * o_pad), key
        assert torch.equal(tr.view(i_pad, k, o_pad), fwd.view(o_pad, k, i_pad).permute(2, 1, 0)), key
