"""GPU: SpeechPromptEncoder / PhonemeEncoder (SURVEY f3) through the C ABI against the reference's fp64 goldens.
Tolerance protocol of the denoiser (DESIGN.md, SURVEY H1): our max-abs and rms error must not exceed the error of the
reference's own autocast-bf16 run on the same inputs, plus an absolute bound at output std ~ 1."""
import numpy as np
import pytest
import torch

from helpers import DPP_CASES, ENCODER_CASES, build_encoder, dpp_case, encoder_case, err_stats

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", ENCODER_CASES)
def test_encoder_matches_reference_golden(name):
    cls, kwargs, x, ref64, ref_bf16, _ = encoder_case(name)
    enc = build_encoder(cls, kwargs, device="cuda")
    out = enc(x.cuda())
    assert out.dtype == torch.float32 and tuple(out.shape) == ref64.shape
    got = out.cpu().numpy()
    assert np.isfinite(got).all()
    emax, erms = err_stats(got, ref64)
    bmax, brms = err_stats(ref_bf16, ref64)
    print(f"{name}: ours max {emax:.3e} rms {erms:.3e} | reference bf16-autocast max {bmax:.3e} rms {brms:.3e}")
    assert emax <= max(bmax, 1e-3) and erms <= max(brms, 1e-4), (emax, erms, bmax, brms)
    assert emax < 8e-2 and erms < 1.5e-2
    # second call (packed weights cached) returns the same values in a fresh tensor
    out2 = enc(x.cuda())
    assert out2.data_ptr() != out.data_ptr() and torch.equal(out, out2)


def test_silu_conv_gemm_matches_torch():
    """The k=9 'same' convolution + SiLU as a nine-segment GEMM, both kernel families (<=128 rows: single CTA,
    >128 rows: CTA pair), bf16 and fp32 outputs, against torch fp32 conv1d on the bf16-rounded operands."""
    import torch.nn.functional as F
    from naturalspeech2_pytorch_b200 import _lib, ops
    from naturalspeech2_pytorch_b200.encoders import _conv_segs
    from naturalspeech2_pytorch_b200.model import _pack_conv
    g = torch.Generator().manual_seed(3)
    for rows, c_in, c_out in ((103, 128, 256), (300, 256, 512), (1024, 64, 128)):
        x = torch.randn(2, rows, c_in, generator=g).bfloat16()
        w = (torch.randn(c_out, c_in, 9, generator=g) / (9 * c_in) ** 0.5)
        b = torch.randn(c_out, generator=g) * 0.1
        ref = F.silu(F.conv1d(x.float().transpose(1, 2), w.bfloat16().float(), b, padding=4)).transpose(1, 2)
        causal = F.silu(F.conv1d(F.pad(x.float().transpose(1, 2), (8, 0)), w.bfloat16().float(), b)).transpose(1, 2)
        for dt, epi in ((torch.bfloat16, ops.EPI_BF16), (torch.float32, ops.EPI_F32)):
            for want, first in ((ref, 4), (causal, 8)):
                out = torch.empty(2, rows, c_out, device="cuda", dtype=dt)
                ops.gemm(x.cuda(), _pack_conv(w).cuda(), out, n=c_out, epilogue=epi, segs=_conv_segs(c_in, 9, first),
                         bias=b.cuda(), flags=_lib.NS2_GEMM_FLAG_SILU)
                err = (out.float().cpu() - want).abs().max().item()
                assert err < (2e-2 if dt == torch.bfloat16 else 2e-3), (rows, c_in, c_out, dt, first, err)


def test_embedding_bf16():
    from naturalspeech2_pytorch_b200 import ops
    g = torch.Generator().manual_seed(4)
    table = torch.randn(51, 128, generator=g)
    ids = torch.randint(0, 50, (3, 17), generator=g)
    ids[2, 10:] = -1
    out = ops.embedding_bf16(ids.cuda(), table.cuda(), torch.empty(3, 17, 128, device="cuda", dtype=torch.bfloat16), 50)
    want = table[ids.masked_fill(ids < 0, 50)].bfloat16()
    assert torch.equal(out.cpu(), want)


@pytest.mark.parametrize("name", DPP_CASES)
def test_duration_pitch_predictor_matches_reference_golden(name):
    kwargs, x, prompts, ref64, ref_bf16, _ = dpp_case(name)
    enc = build_encoder("DurationPitchPredictor", kwargs, device="cuda")
    dur, pitch = enc(x.cuda(), prompts.cuda())
    got = torch.stack((dur, pitch)).cpu().numpy()
    assert got.shape == ref64.shape and np.isfinite(got).all() and (got >= 0).all()
    emax, erms = err_stats(got, ref64)
    bmax, brms = err_stats(ref_bf16, ref64)
    print(f"{name}: ours max {emax:.3e} rms {erms:.3e} | reference bf16-autocast max {bmax:.3e} rms {brms:.3e}")
    assert emax <= max(bmax, 1e-3) and erms <= max(brms, 1e-4), (emax, erms, bmax, brms)
    assert emax < 5e-2 and erms < 1e-2


def test_groupnorm_silu_and_rowdot_match_torch():
    import torch.nn.functional as F
    from naturalspeech2_pytorch_b200 import ops
    g = torch.Generator().manual_seed(6)
    for B, N, Cn, G in ((2, 37, 128, 8), (3, 100, 512, 8), (1, 5, 64, 4)):
        x = torch.randn(B, N, Cn, generator=g) * 2 + 0.5
        w, b = torch.randn(Cn, generator=g), torch.randn(Cn, generator=g)
        r = torch.randn(B, N, Cn, generator=g)
        want = F.silu(F.group_norm(x.double().transpose(1, 2), G, w.double(), b.double(), 1e-5)).transpose(1, 2)
        o32 = torch.empty(B, N, Cn, device="cuda")
        obf = torch.empty(B, N, Cn, device="cuda", dtype=torch.bfloat16)
        ops.groupnorm_silu(x.cuda(), w.cuda(), b.cuda(), G, out_f32=o32, out_bf16=obf)
        assert (o32.cpu().double() - want).abs().max() < 2e-5
        assert (obf.cpu().double() - want).abs().max() < 4e-2
        xr = r.clone().cuda()                                     # in-place residual: out aliases resid
        ops.groupnorm_silu(x.cuda(), w.cuda(), b.cuda(), G, resid=xr, out_f32=xr)
        assert (xr.cpu().double() - (want + r.double())).abs().max() < 2e-5
        wv, bias = torch.randn(Cn, generator=g), torch.randn(1, generator=g)
        out = ops.rowdot(x.cuda(), wv.cuda(), bias.cuda(), torch.empty(B, N, device="cuda"), relu=True)
        assert (out.cpu().double() - F.relu(x.double() @ wv.double() + bias.double())).abs().max() < 1e-4


def test_expand_encodings_bit_exact():
    from helpers import GOLDEN
    from naturalspeech2_pytorch_b200.encoders import expand_encodings
    z = np.load(GOLDEN / "encoders.npz")
    ph, dur, pitch, table = (torch.from_numpy(z[f"expand_{k}"]).cuda() for k in ("phon", "duration", "pitch", "table"))
    cond = expand_encodings(ph, dur, pitch, table)
    np.testing.assert_array_equal(cond.cpu().numpy(), z["expand_cond"])


def test_conditioner_drives_conditional_sampling():
    """prompt latents + phoneme ids -> (prompt_enc, cond) -> NaturalSpeech2.sample (the flow of ns2.py:1472-1493)."""
    from naturalspeech2_pytorch_b200 import Model, NaturalSpeech2
    from naturalspeech2_pytorch_b200.encoders import Conditioner, expand_encodings
    torch.manual_seed(0)
    cond_net = Conditioner(dim_codebook=128, num_phoneme_tokens=50).cuda().eval()
    with torch.no_grad():
        for trunk in (cond_net.duration_pitch.to_duration_pred, cond_net.duration_pitch.to_pitch_pred):
            trunk.to_pred[0].bias.fill_(3.0)     # random-init heads predict ~0 frames per phoneme otherwise
    g = torch.Generator().manual_seed(1)
    prompt = torch.randn(2, 103, 128, generator=g).cuda()
    text = torch.randint(0, 50, (2, 23), generator=g).cuda()
    prompt_enc, cond = cond_net(prompt=prompt, text=text, mode="sample")
    assert prompt_enc.shape == (2, 103, 512) and cond.shape[:2] == (2, 512) and cond.shape[2] > 0
    assert torch.isfinite(prompt_enc).all() and torch.isfinite(cond).all()
    # the composite equals its parts
    ph = cond_net.phoneme_enc(text)
    dur, pitch = cond_net.duration_pitch(ph, prompt_enc)
    assert torch.equal(cond, expand_encodings(ph, dur, pitch, cond_net.pitch_emb.weight))
    model = Model(dim=128, depth=1, heads=2, wavenet_layers=2, wavenet_stacks=1, dim_prompt=512,
                  condition_on_prompt=True).cuda().eval()
    ns = NaturalSpeech2(model, target_sample_hz=24000, timesteps=2, conditioner=cond_net)
    out = ns.sample(length=64, prompt=prompt, text=text)
    assert out.shape == (2, 64, 128) and torch.isfinite(out).all()
    with pytest.raises(NotImplementedError):
        cond_net(prompt=prompt, text=text, mode="train")
