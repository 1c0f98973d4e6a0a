"""CPU: the duration / pitch predictor's restatement (`oracle.encoders_oracle.duration_pitch_predictor`, with the token
table gathered in front) under fp64 autograd through the weighted L1 losses reproduces the reference module's own
gradients (tests/golden/grads_dpp_train.npz, make_golden_dpp_train.py).  This pins the oracle that
tests/test_duration_pitch_backward_fp64_gpu.py differentiates, and checks the fixture's sign margins."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from golden.make_golden_dpp_train import DPP_TRAIN_CASES, dpp_train_inputs
from fp64_check import rel_l2
from helpers import GOLDEN, build_encoder

Z = np.load(GOLDEN / "grads_dpp_train.npz")


@pytest.mark.parametrize("name", list(DPP_TRAIN_CASES))
def test_oracle_fp64_autograd_matches_the_reference_golden(name):
    from oracle import encoders_oracle as eo
    kwargs, *_ = DPP_TRAIN_CASES[name]
    enc = build_encoder("DurationPitchPredictor", kwargs)
    names = [str(n) for n in Z[f"{name}::names"]]
    assert [n for n, _ in enc.named_parameters()] == names
    P = {n: p.detach().double().requires_grad_(True) for n, p in enc.named_parameters()}
    with torch.no_grad():
        for h, b in zip(("to_duration_pred", "to_pitch_pred"), Z[f"{name}::biases"]):
            P[f"{h}.to_pred.0.bias"].fill_(float(b))
    x, prompts = dpp_train_inputs(name)
    table = x.dtype == torch.int64
    x = P["phoneme_token_emb.weight"][x] if table else x.double().requires_grad_(True)
    prompts = prompts.double().requires_grad_(True)
    dur, pitch = eo.duration_pitch_predictor(P, x, prompts, heads=kwargs.get("heads", 8))
    tgt = torch.from_numpy(Z[f"{name}::targets"])
    margin = float(Z["margin"])
    # the fixture decides every ReLU and |.| branch by at least `margin`
    for p, t in zip((dur, pitch), tgt):
        assert float(p.min()) >= margin * (1 - 1e-9) and float((p - t).abs().min()) >= margin * (1 - 1e-9)
    np.testing.assert_allclose(torch.stack((dur, pitch)).detach().numpy(), Z[f"{name}::preds"], rtol=1e-9, atol=1e-9)
    w_d, w_p = (float(v) for v in Z["weights"])
    l_dur, l_pitch = F.l1_loss(tgt[0], dur), F.l1_loss(tgt[1], pitch)
    loss = w_d * l_dur + w_p * l_pitch
    np.testing.assert_allclose([l_dur.item(), l_pitch.item(), loss.item()], Z[f"{name}::losses"], rtol=1e-9)
    loss.backward()
    norms = np.array([P[n].grad.norm().item() for n in names])
    np.testing.assert_allclose(norms, Z[f"{name}::norms"], rtol=1e-9, atol=1e-12)
    d_in = P["phoneme_token_emb.weight"].grad if table else x.grad
    assert rel_l2(d_in, Z[f"{name}::d_table" if table else f"{name}::d_x"]) < 1e-6       # stored as fp32
    assert rel_l2(prompts.grad, Z[f"{name}::d_prompts"]) < 1e-6
