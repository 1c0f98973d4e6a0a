"""GPU: the duration / pitch predictor trained jointly with the conditional model: `Conditioner(train_duration_pitch=
True)` returns the reference's L1 losses (ns2.py:1579-1590) and `NaturalSpeech2.forward` adds them, weighted
(ns2.py:1600-1602, 1684); their gradients reach the predictor and, through its inputs, both encoders."""
import pytest
import torch
import torch.nn.functional as F

from param_fill import fill_module
from restatements import DPP_TRAIN_SHAPE, dpp_train_inputs, dpp_train_loss

pytestmark = pytest.mark.gpu
B, T_TEXT, NP, L = DPP_TRAIN_SHAPE
W_DUR, W_PITCH = 0.7, 0.3


def _setup(flag=True):
    from naturalspeech2_pytorch_b200 import Model, NaturalSpeech2
    from naturalspeech2_pytorch_b200.encoders import Conditioner
    torch.manual_seed(0)
    cond_net = Conditioner(dim_codebook=128, num_phoneme_tokens=50, train_duration_pitch=flag)
    fill_module(cond_net, 77)
    with torch.no_grad():
        for trunk, bias in ((cond_net.duration_pitch.to_duration_pred, 10.0), (cond_net.duration_pitch.to_pitch_pred, 3.0)):
            trunk.to_pred[0].weight.mul_(0.01)   # keep the ReLU heads alive at random init: pre ~ the bias, away
            trunk.to_pred[0].bias.fill_(bias)    # from the targets (1-5 frames, 100-300 Hz)
    model = Model(dim=128, depth=1, heads=2, wavenet_layers=2, wavenet_stacks=1, dim_prompt=512,
                  condition_on_prompt=True)
    fill_module(model, 78)
    cond_net.cuda().train()
    model.cuda().train()
    ns = NaturalSpeech2(model, target_sample_hz=24000, timesteps=4, conditioner=cond_net,
                        duration_loss_weight=W_DUR, pitch_loss_weight=W_PITCH)
    return ns, cond_net, model


def _capture(cond_net):
    """Hook that keeps the predictor's outputs."""
    seen = {}

    def hook(module, args, out):
        seen["pred"] = tuple(o.detach() for o in out)
    return seen, cond_net.duration_pitch.register_forward_hook(hook)


def test_loss_adds_the_weighted_duration_and_pitch_losses():
    from naturalspeech2_pytorch_b200.encoders import average_over_durations
    inp = dpp_train_inputs()
    ns, cond_net, _ = _setup(flag=False)
    loss_off = dpp_train_loss(ns, inp)
    cond_net.train_duration_pitch = True
    seen, h = _capture(cond_net)
    loss_on = dpp_train_loss(ns, inp)
    h.remove()
    dur_pred, pitch_pred = seen["pred"]
    ph_pitch = average_over_durations(inp["pitch"][:, None].float(), inp["duration"])[:, 0]
    want = loss_off + (W_DUR * F.l1_loss(inp["duration"].float(), dur_pred) + W_PITCH * F.l1_loss(ph_pitch, pitch_pred))
    assert torch.equal(loss_on.detach(), want.detach()), (float(loss_on), float(want))
    assert loss_on.requires_grad and float(loss_on - loss_off) > 0


def test_encoder_outputs_receive_the_predictors_input_gradients():
    """With the flag, the gradient reaching each encoder's output is the flag-off one plus that of the weighted L1
    losses through the predictor's node (its d x / d prompts), and every predictor parameter gets a gradient."""
    inp = dpp_train_inputs()
    ns, cond_net, _ = _setup(flag=False)
    params = dict(cond_net.named_parameters())
    encs = ("phoneme_enc", "prompt_enc")

    def outputs():
        outs = {}
        hooks = [getattr(cond_net, n).register_forward_hook(lambda m, a, out, n=n: outs.__setitem__(n, out))
                 for n in encs]
        return outs, hooks

    def total_grads():
        outs, hooks = outputs()
        got = {}
        cond_net.zero_grad(set_to_none=True)
        loss = dpp_train_loss(ns, inp)
        for n in encs:
            outs[n].register_hook(lambda g, n=n: got.__setitem__(n, g.clone()))
        loss.backward()
        for h in hooks:
            h.remove()
        return got

    off = total_grads()
    assert all(p.grad is None for n, p in params.items() if n.startswith("duration_pitch."))
    cond_net.train_duration_pitch = True
    on = total_grads()
    pred_grads = {n: p.grad for n, p in params.items() if n.startswith("duration_pitch.")}
    missing = [n for n, g in pred_grads.items() if g is None or not bool(torch.isfinite(g).all())]
    zero = [n for n, g in pred_grads.items() if g is not None and float(g.norm()) == 0]
    assert not missing and not zero, (missing, zero)
    # the predictor's share alone: d (w_d L_d + w_p L_p) / d encoder outputs
    outs, hooks = outputs()
    _, _, l_dur, l_pitch = cond_net(prompt=ns.process_prompt(inp["prompt"]), text=inp["text"], mode="train",
                                    pitch=inp["pitch"], duration=inp["duration"])
    for h in hooks:
        h.remove()
    share = dict(zip(encs, torch.autograd.grad(W_DUR * l_dur + W_PITCH * l_pitch, [outs[n] for n in encs])))
    for n in encs:
        assert float(share[n].norm()) > 0
        want = off[n] + share[n]           # the pitch table's scatter adds with atomics: last-bit differences
        assert torch.allclose(on[n], want, rtol=1e-5, atol=1e-6 * float(want.abs().max())), n


def test_two_identical_steps_give_bit_identical_gradients():
    inp = dpp_train_inputs()
    ns, cond_net, model = _setup()
    runs = []
    for _ in range(2):
        cond_net.zero_grad(set_to_none=True)
        model.zero_grad(set_to_none=True)
        dpp_train_loss(ns, inp).backward()
        runs.append({n: p.grad.clone() for n, p in cond_net.named_parameters() if n.startswith("duration_pitch.")})
    assert runs[0].keys() == runs[1].keys() and len(runs[0]) > 0
    assert all(torch.equal(runs[0][n], runs[1][n]) for n in runs[0])


def test_adamw_steps_lower_both_losses():
    from naturalspeech2_pytorch_b200.encoders import average_over_durations
    inp = dpp_train_inputs()
    ns, cond_net, model = _setup()
    opt = torch.optim.AdamW(list(cond_net.parameters()) + list(model.parameters()), lr=1e-5)
    hist = []
    for _ in range(5):
        seen, h = _capture(cond_net)
        opt.zero_grad(set_to_none=True)
        dpp_train_loss(ns, inp).backward()
        h.remove()
        ph_pitch = average_over_durations(inp["pitch"][:, None].float(), inp["duration"])[:, 0]
        hist.append((float(F.l1_loss(inp["duration"].float(), seen["pred"][0])),
                     float(F.l1_loss(ph_pitch, seen["pred"][1]))))
        opt.step()
    assert hist[-1][0] < hist[0][0] and hist[-1][1] < hist[0][1], hist
