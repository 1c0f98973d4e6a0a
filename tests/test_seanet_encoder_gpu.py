"""GPU: the whole SEANet encoder against float64 references - the committed transformers goldens (frames and
EncodecModel's codes), the fp64 oracle at (4, 1024 frames) where the LSTM's 2 x 1024 recurrent steps accumulate
error - and the raw-audio paths it opens: `EncodecRVQ(encoder=...)`, `NaturalSpeech2.forward(raw_audio)`,
`process_prompt(raw_prompt)` and the decoder round trip."""
import numpy as np
import pytest
import torch

from golden.make_golden_seanet_encoder import CASES, audio, codebooks, filled_state_dict
import seanet_oracle

pytestmark = pytest.mark.gpu

REL_MARGIN = 2e-3


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(golden_dir / "seanet_encoder.npz")


@pytest.fixture(scope="module")
def sd64(golden):
    keys_shapes = [(k, tuple(int(v) for v in s.split(","))) for k, s in zip(golden["keys"], golden["shapes"])]
    return filled_state_dict(keys_shapes)


@pytest.fixture(scope="module")
def enc(sd64):
    from naturalspeech2_pytorch_b200 import SEANetEncoder
    e = SEANetEncoder()
    e.load_state_dict({k: v.float() for k, v in sd64.items()})
    return e.cuda().eval()


@pytest.fixture(scope="module")
def cb(golden):
    return codebooks(golden["cb_scale"])           # (8, 1024, 128) float64, fp32-representable


def _err(got, ref):
    got, ref = got.double(), ref.double()
    return float((got - ref).norm() / ref.norm()), float((got - ref).abs().max())


@pytest.mark.parametrize("case", sorted(CASES))
def test_encoder_against_transformers_goldens(golden, enc, case):
    B, N = CASES[case]
    f = enc(audio(B, N).float().cuda())
    assert tuple(f.shape) == (B, N, 128) and f.dtype == torch.float32
    rel, mx = _err(f.cpu(), torch.from_numpy(golden[f"{case}_f64"]))
    auto_rel, auto_max = (float(v) for v in golden[f"{case}_err"][2:4])
    print(f"{case}: rel-L2 {rel:.3e} max-abs {mx:.3e}; autocast-bf16 {auto_rel:.3e} / {auto_max:.3e}")
    assert rel <= auto_rel + REL_MARGIN, (rel, auto_rel)
    assert mx <= 2 * auto_max, (mx, auto_max)


def test_encoder_against_fp64_oracle_long_sequence(sd64, enc):
    B, N = 4, 1024
    x = audio(B, N).cuda()
    sdc = {k: v.cuda() for k, v in sd64.items()}
    f64 = seanet_oracle.encode(sdc, x, dtype=torch.float64)
    fem = seanet_oracle.encode(sdc, x, dtype=torch.float64, emulate_bf16=True)
    f = enc(x.float())
    rel, mx = _err(f, f64)
    em_rel, em_max = _err(fem, f64)
    print(f"(4, 1024): rel-L2 {rel:.3e} max-abs {mx:.3e}; bf16 emulation {em_rel:.3e} / {em_max:.3e}")
    assert rel <= 1.5 * em_rel, (rel, em_rel)


@pytest.mark.parametrize("case", sorted(CASES))
def test_codes_are_nearest_within_the_frame_error(golden, enc, cb, case):
    """RVQ encode is exact, so wherever the GPU's codes agree with EncodecModel's fp64 codes on stages < q, the
    triangle inequality bounds stage q: ||r64 - cb[c_gpu]|| <= ||r64 - cb[c_ref]|| + 2 ||f_gpu - f64||, with r64 the
    fp64 residual.  No tuned threshold; the agreement fraction is reported, not asserted."""
    from naturalspeech2_pytorch_b200 import EncodecRVQ
    B, N = CASES[case]
    codec = EncodecRVQ(cb.float(), encoder=enc).cuda()
    x = audio(B, N).float().cuda()
    _, codes, _ = codec(x, return_encoded=True)
    f = enc(x).double().cpu().reshape(-1, 128)
    f64 = torch.from_numpy(golden[f"{case}_f64"]).reshape(-1, 128)
    ref = torch.from_numpy(golden[f"{case}_codes"].astype(np.int64)).reshape(-1, 8)
    got = codes.cpu().reshape(-1, 8)
    delta = (f - f64).norm(dim=-1)
    r = f64.clone()
    agree = torch.ones(r.shape[0], dtype=torch.bool)
    checked = 0
    for q in range(8):
        d_gpu = (r - cb[q][got[:, q]]).norm(dim=-1)
        d_ref = (r - cb[q][ref[:, q]]).norm(dim=-1)
        ok = d_gpu <= d_ref * (1 + 1e-9) + 2 * delta
        assert bool(ok[agree].all()), f"stage {q}: {int((~ok & agree).sum())} frames outside the bound"
        checked += int(agree.sum())
        agree &= got[:, q] == ref[:, q]
        r = r - cb[q][ref[:, q]]
    print(f"{case}: codes equal to EncodecModel's on {float((got == ref).double().mean()):.4f} of entries; "
          f"{checked} (frame, stage) pairs checked")


def test_codec_composition_and_curtailing(enc, cb):
    from naturalspeech2_pytorch_b200 import EncodecRVQ
    codec = EncodecRVQ(cb.float(), encoder=enc).cuda()
    x = audio(3, 40).float().cuda()
    emb, codes, _ = codec(x, return_encoded=True)
    c2, e2 = codec.quantize(enc(x))
    assert torch.equal(codes, c2) and torch.equal(emb, e2)
    assert torch.equal(codec(x), codes)
    long = torch.cat([x, audio(3, 1).float().cuda()[:, :123]], dim=1)   # T = 320 * 40 + 123
    for left, part in ((False, long[:, :12800]), (True, long[:, -12800:])):
        emb_l, codes_l, _ = codec(long, return_encoded=True, curtail_from_left=left)
        c3, e3 = codec.quantize(enc(part))
        assert torch.equal(codes_l, c3) and torch.equal(emb_l, e3)
    assert torch.equal(codec(long), codes)


@pytest.fixture(scope="module")
def small_model():
    from naturalspeech2_pytorch_b200 import Model
    torch.manual_seed(0)
    return Model(dim=128, depth=1, heads=2, wavenet_layers=2, wavenet_stacks=1).cuda()


@pytest.mark.parametrize("ce_weight", [0.0, 0.5])
def test_raw_audio_training_loss_equals_preencoded(enc, cb, small_model, ce_weight):
    from naturalspeech2_pytorch_b200 import EncodecRVQ, NaturalSpeech2
    codec = EncodecRVQ(cb.float(), encoder=enc).cuda()
    ns = NaturalSpeech2(small_model, codec=codec, timesteps=2, rvq_cross_entropy_loss_weight=ce_weight)
    B, N = 2, 24
    x = audio(B, N).float().cuda()
    times = torch.tensor([0.3, 0.8], device="cuda")
    noise = torch.randn(B, N, 128, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))
    loss_raw = ns(x, times=times, noise=noise)
    emb, codes, _ = codec(x, return_encoded=True)
    loss_lat = ns(emb, codes=codes, times=times, noise=noise)
    assert torch.isfinite(loss_raw) and torch.equal(loss_raw.detach(), loss_lat.detach())
    loss_raw.backward()   # the raw-audio loss trains the denoiser like the pre-encoded one


def test_raw_prompt_is_left_curtailed_encoding(enc, cb):
    from naturalspeech2_pytorch_b200 import EncodecRVQ, Model, NaturalSpeech2
    model = Model(dim=128, depth=1, heads=2, wavenet_layers=2, wavenet_stacks=1, dim_prompt=128,
                  condition_on_prompt=True).cuda()
    codec = EncodecRVQ(cb.float(), encoder=enc).cuda()
    ns = NaturalSpeech2(model, codec=codec, timesteps=2)
    prompt = audio(2, 10).float().cuda()[:, :3000]               # 9 frames + 120 samples
    got = ns.process_prompt(prompt)
    _, ref_emb = codec.quantize(enc(prompt[:, -2880:]))
    assert tuple(got.shape) == (2, 9, 128) and torch.equal(got, ref_emb)


def test_round_trip_returns_audio_shape(enc):
    from naturalspeech2_pytorch_b200 import SEANetDecoder
    dec = SEANetDecoder().cuda().eval()
    x = audio(2, 12).float().cuda()
    y = dec(enc(x))
    assert tuple(y.shape) == (2, 1, 320 * 12) and bool(torch.isfinite(y).all())
    y3 = dec(enc(x[:, None]))
    assert torch.equal(y, y3)


def test_encoder_is_deterministic_and_returns_owned_tensors(enc):
    x = audio(3, 200).float().cuda()
    a = enc(x)
    b = enc(x)
    assert torch.equal(a, b)
    assert a.data_ptr() != b.data_ptr()   # a new tensor per call, never a cached workspace
