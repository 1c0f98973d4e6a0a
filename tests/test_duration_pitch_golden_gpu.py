"""GPU: the duration / pitch predictor's hand-written backward against the REFERENCE module's own fp64 autograd through
the weighted L1 losses (tests/golden/grads_dpp_train.npz, make_golden_dpp_train.py), in the style of
tests/test_conditional_training_gpu.py: losses, every parameter's gradient norm, and d x (or the token table's
gradient) and d prompts whole.  The parameters are the fixture's fp32 weights (not bf16-rounded), so the comparison
includes our bf16 operands.  The fixture keeps every head pre-activation and every |prediction - target| at least its
margin from 0; the test asserts that our forward error is under 1/20 of it, so no branch can differ."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from golden.make_golden_dpp_train import DPP_TRAIN_CASES, dpp_train_inputs
from helpers import GOLDEN, build_encoder

pytestmark = pytest.mark.gpu
Z = np.load(GOLDEN / "grads_dpp_train.npz")


def _rel_cos(got, ref):
    got, ref = got.detach().double().cpu().flatten(), torch.as_tensor(ref).double().flatten()
    return float((got - ref).norm() / ref.norm()), float(F.cosine_similarity(got, ref, dim=0))


@pytest.mark.parametrize("name", list(DPP_TRAIN_CASES))
def test_backward_matches_the_reference_golden(name):
    kwargs, *_ = DPP_TRAIN_CASES[name]
    enc = build_encoder("DurationPitchPredictor", kwargs, device="cuda")
    with torch.no_grad():
        for h, b in zip(("to_duration_pred", "to_pitch_pred"), Z[f"{name}::biases"]):
            getattr(enc, h).to_pred[0].bias.fill_(float(b))
    enc.train()
    x, prompts = dpp_train_inputs(name)
    table = x.dtype == torch.int64
    x = x.cuda() if table else x.cuda().requires_grad_(True)
    prompts = prompts.cuda().requires_grad_(True)
    dur, pitch = enc(x, prompts)
    tgt = torch.from_numpy(Z[f"{name}::targets"]).float().cuda()
    fwd_err = float((torch.stack((dur, pitch)).detach().double().cpu() - torch.from_numpy(Z[f"{name}::preds"])).abs().max())
    print(f"{name}: forward max-abs {fwd_err:.3e}, margin {float(Z['margin'])}")
    assert 20 * fwd_err <= float(Z["margin"]), "a ReLU or L1 branch could differ from the fixture's"
    w_d, w_p = (float(v) for v in Z["weights"])
    l_dur, l_pitch = F.l1_loss(tgt[0], dur), F.l1_loss(tgt[1], pitch)
    loss = w_d * l_dur + w_p * l_pitch
    np.testing.assert_allclose([l_dur.item(), l_pitch.item(), loss.item()], Z[f"{name}::losses"], rtol=2e-3)
    loss.backward()
    worst = ("", 0.0)
    for n, ref in zip((str(v) for v in Z[f"{name}::names"]), Z[f"{name}::norms"]):
        g = dict(enc.named_parameters())[n].grad
        assert g is not None and bool(torch.isfinite(g).all()), n
        if float(ref) == 0.0:   # dpp_512's duration bias: as many rows above as below target, +-w/T cancel exactly
            assert float(g.norm()) < 1e-5, (n, float(g.norm()))      # fp32 sums of those terms: rounding only
            continue
        rel = abs(float(g.norm()) - float(ref)) / float(ref)
        worst = max(worst, (n, rel), key=lambda t: t[1])
    print(f"{name}: worst gradient-norm deviation {worst[0]} {worst[1]:.3%}")
    assert worst[1] < 0.02, worst
    wholes = [("d prompts", prompts.grad, Z[f"{name}::d_prompts"])]
    wholes.append(("d table", enc.phoneme_token_emb.weight.grad, Z[f"{name}::d_table"]) if table else
                  ("d x", x.grad, Z[f"{name}::d_x"]))
    for what, got, ref in wholes:
        rel, cos = _rel_cos(got, ref)
        print(f"{name} {what}: rel-L2 {rel:.3%} cos {cos:.6f}")
        assert rel < 0.03 and cos > 0.9995, (what, rel, cos)   # the bounds of test_conditional_training_gpu.py
