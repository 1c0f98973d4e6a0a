"""GPU: the whole SEANet decoder against float64 references - the committed transformers goldens, the fp64 oracle at
(4, 1024) where the LSTM's 2 x 1024 recurrent steps accumulate error - and through `NaturalSpeech2.sample()`."""
import numpy as np
import pytest
import torch

from golden.make_golden_seanet import CASES, filled_state_dict, latents
import seanet_oracle

pytestmark = pytest.mark.gpu

REL_MARGIN = 2e-3


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(golden_dir / "seanet_decoder.npz")


@pytest.fixture(scope="module")
def sd64(golden):
    keys_shapes = [(k, tuple(int(v) for v in s.split(","))) for k, s in zip(golden["keys"], golden["shapes"])]
    return filled_state_dict(keys_shapes)


@pytest.fixture(scope="module")
def dec(sd64):
    from naturalspeech2_pytorch_b200 import SEANetDecoder
    d = SEANetDecoder()
    d.load_state_dict({k: v.float() for k, v in sd64.items()})
    return d.cuda().eval()


def _err(got, ref):
    got, ref = got.double(), ref.double()
    return float((got - ref).norm() / ref.norm()), float((got - ref).abs().max())


@pytest.mark.parametrize("case", sorted(CASES))
def test_decoder_against_transformers_goldens(golden, dec, case):
    B, N = CASES[case]
    y = dec(latents(B, N).float().cuda())
    assert tuple(y.shape) == (B, 1, 320 * N) and y.dtype == torch.float32
    rel, mx = _err(y.cpu(), torch.from_numpy(golden[f"{case}_ref32"]))
    auto_rel, auto_max = (float(v) for v in golden[f"{case}_err"][2:4])
    assert rel <= auto_rel + REL_MARGIN, (rel, auto_rel)
    assert mx <= 2 * auto_max, (mx, auto_max)


def test_decoder_against_fp64_oracle_long_sequence(golden, sd64, dec):
    B, N = 4, 1024
    emb = latents(B, N).cuda()
    sdc = {k: v.cuda() for k, v in sd64.items()}
    y64 = seanet_oracle.decode(sdc, emb, dtype=torch.float64)
    yem = seanet_oracle.decode(sdc, emb, dtype=torch.float64, emulate_bf16=True)
    y = dec(emb.float())
    rel, mx = _err(y, y64)
    em_rel, em_max = _err(yem, y64)
    auto_rel, auto_max = (float(v) for v in golden["b2n130_err"][2:4])
    print(f"(4, 1024): rel-L2 {rel:.3e} max-abs {mx:.3e}; bf16 emulation {em_rel:.3e} / {em_max:.3e}")
    assert rel <= auto_rel + REL_MARGIN, (rel, auto_rel)
    assert rel <= 1.5 * em_rel, (rel, em_rel)
    assert mx <= 2 * max(em_max, auto_max), (mx, em_max, auto_max)


def test_sample_returns_decoded_waveforms(dec):
    from naturalspeech2_pytorch_b200 import EncodecRVQ, Model, NaturalSpeech2
    torch.manual_seed(0)
    model = Model(dim=128, depth=1, heads=2, wavenet_layers=2, wavenet_stacks=1).cuda().eval()
    cb = torch.randn(4, 1024, 128)
    ns = NaturalSpeech2(model, codec=EncodecRVQ(cb, decoder=dec).cuda(), timesteps=2)
    B, N = 2, 40
    noise = torch.randn(B, N, 128, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    audio = ns.sample(length=N, batch_size=B, noise=noise)
    assert tuple(audio.shape) == (B, 320 * N)
    lat = ns.ddim_sample((B, N, 128), noise=noise)
    assert torch.equal(audio, dec(lat)[:, 0])


def test_decoder_is_deterministic(dec):
    emb = latents(3, 200).float().cuda()
    assert torch.equal(dec(emb), dec(emb))
