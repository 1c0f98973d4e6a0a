"""GPU: the conditioning encoders trained with the reference's dropout (`train_dropout=True`): output and every
parameter gradient against float64 autograd of the masked restatement (tests/dropout_oracle.py) given the masks of the
seed the call drew; the seed's draw, eval() and conditional training with dropout."""
import numpy as np
import pytest
import torch

import dropout_oracle as do
from helpers import build_encoder, encoder_case
from restatements import drawn_seed, e2e_front_end, e2e_inputs, e2e_loss

pytestmark = pytest.mark.gpu


def _rel_cos(got, ref):
    got, ref = got.detach().double().cpu().flatten(), ref.detach().double().cpu().flatten()
    rel = float((got - ref).norm() / ref.norm().clamp_min(1e-12))
    cos = float(torch.nn.functional.cosine_similarity(got, ref, dim=0))
    return rel, cos


def _assert_tensor(got, ref, what):
    rel, cos = _rel_cos(got, ref)
    assert rel < 0.03 and cos > 0.9995, (what, rel, cos)   # the bounds of test_conditional_training_gpu.py


def _encoder(name, p, train_dropout=True):
    cls, kwargs, x, *_ = encoder_case(name)
    kw = dict(kwargs)
    if cls == "SpeechPromptEncoder":
        kw["dropout"] = p
    else:
        kw.update(conv_dropout=p, attn_dropout=p)
    enc = build_encoder(cls, kw, device="cuda").train()
    enc.train_dropout = train_dropout
    return cls, kwargs, enc, x


def _fp64(cls, kwargs, enc, x, w, seed, p):
    """Output and parameter gradients of fp64 autograd of the restatement, with the masks of `seed` (None: no dropout)."""
    P = {k: v.detach().double().cpu().requires_grad_(True) for k, v in enc.state_dict().items()}
    H, depth = kwargs.get("heads", 8), kwargs["depth"]
    B, N = x.shape[:2]
    masks = conv = None
    if seed is not None:
        masks = [do.mask_tensor(do.attention_mask(seed, 1 + l, p, B, H, N, N), p) for l in range(depth)]
        if cls == "PhonemeEncoder":
            D = kwargs["dim_hidden"]
            conv = do.mask_tensor(do.elementwise_mask(seed, 0, p, B * N * D).reshape(B, N, D), p)
    if cls == "SpeechPromptEncoder":
        ref = do.speech_prompt_encoder(P, x.double(), heads=H, attn_masks=masks)
    else:
        ref = do.phoneme_encoder(P, x, heads=H, conv_mask=conv, attn_masks=masks)
    (ref * w).sum().backward()
    return ref.detach(), {n: P[n].grad for n, _ in enc.named_parameters()}


def _gpu(enc, x, w):
    for prm in enc.parameters():
        prm.grad = None
    out = enc(x.cuda())
    out.backward(w.float().cuda())
    return out.detach(), {n: prm.grad.clone() for n, prm in enc.named_parameters()}


@pytest.mark.parametrize("p", [0.2, 0.5])
@pytest.mark.parametrize("name", ["spe_small", "spe_long", "phon_small"])
def test_encoder_dropout_matches_fp64_autograd(name, p):
    """Output and every parameter gradient with dropout against fp64 autograd given the masks of the drawn seed:
    gradient norms within 2 %; whole tensors < 3 % rel-L2 and cos > 0.9995, or - for the few gradients whose bf16
    error is already larger without dropout (attention's to_q, through dS = P (dP - D)) - no worse than twice the
    error of the same gradient in the same training step without dropout."""
    cls, kwargs, enc, x = _encoder(name, p)
    torch_seed = 1000 + int(p * 10)
    w = torch.randn(enc(x.cuda()).shape, generator=torch.Generator().manual_seed(5), dtype=torch.float64)
    enc.train_dropout = False
    plain_out, plain_g = _gpu(enc, x, w)
    plain_ref, plain_rg = _fp64(cls, kwargs, enc, x, w, None, p)
    enc.train_dropout = True
    torch.manual_seed(torch_seed)
    out, g = _gpu(enc, x, w)
    seed = drawn_seed(torch_seed)
    ref, rg = _fp64(cls, kwargs, enc, x, w, seed, p)
    _assert_tensor(out, ref, f"{name} p{p} output")
    assert _rel_cos(out, plain_ref)[0] > 0.05, "the output must differ from the undropped encoder's"
    for n in g:
        assert bool(torch.isfinite(g[n]).all()), n
        assert abs(float(g[n].norm()) - float(rg[n].norm())) < 0.02 * float(rg[n].norm()), (n, float(g[n].norm()),
                                                                                           float(rg[n].norm()))
        rel, cos = _rel_cos(g[n], rg[n])
        rel0, cos0 = _rel_cos(plain_g[n], plain_rg[n])
        print(f"{name} p{p} {n}: rel-L2 {rel:.3%} cos {cos:.6f} (without dropout {rel0:.3%} {cos0:.6f})")
        assert rel < max(0.03, 2 * rel0) and cos > min(0.9995, 1 - 2 * (1 - cos0)), (n, rel, cos, rel0, cos0)


@pytest.mark.parametrize("name", ["spe_small", "phon_small"])
def test_seed_draw_eval_and_no_grad(name):
    _, _, enc, x = _encoder(name, 0.2)
    x = x.cuda()
    with torch.no_grad():
        torch.manual_seed(7)
        a = enc(x)
        b = enc(x)                        # the next call draws another seed: other masks
        torch.manual_seed(7)
        a2 = enc(x)                       # torch.manual_seed reproduces the draw
    assert not torch.equal(a, b) and torch.equal(a, a2)
    torch.manual_seed(7)
    g = enc(x)                            # the autograd path draws the same masks as train mode under no_grad
    assert g.grad_fn is not None and torch.equal(g.detach(), a)
    enc.eval()
    state = torch.get_rng_state()
    with torch.no_grad():
        e = enc(x)
    assert torch.equal(torch.get_rng_state(), state), "eval() draws nothing"
    enc.train_dropout = False
    enc.train()
    state = torch.get_rng_state()
    with torch.no_grad():
        t = enc(x)
    assert torch.equal(torch.get_rng_state(), state), "train_dropout=False draws nothing"
    assert torch.equal(e, t), "eval() with train_dropout is the inference forward"
    assert not torch.equal(e, a)


def test_conditional_training_with_dropout_lowers_the_loss():
    """AdamW steps over the denoiser and the front end with the encoders' dropout on lower the (dropout-free) loss on
    a fixed batch."""
    from naturalspeech2_pytorch_b200 import NaturalSpeech2
    mods, cond_net = e2e_front_end("e2e_small")
    for enc in (cond_net.prompt_enc, cond_net.phoneme_enc):
        enc.train_dropout = True
        assert enc.attn_dropout > 0 or enc.conv_dropout > 0
    ns = NaturalSpeech2(mods["model"], target_sample_hz=24000, timesteps=4, conditioner=cond_net)
    inp = e2e_inputs("e2e_small")

    def eval_loss():
        for m in mods.values():
            m.eval()
        with torch.no_grad():
            v = float(e2e_loss(ns, inp))
        for m in mods.values():
            m.train()
        return v

    params = [p for m in mods.values() for p in m.parameters()]
    opt = torch.optim.AdamW(params, lr=2e-4)
    before = eval_loss()
    torch.manual_seed(11)
    losses = []
    for _ in range(8):
        opt.zero_grad(set_to_none=True)
        loss = e2e_loss(ns, inp)
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
    assert all(np.isfinite(losses)), losses
    assert eval_loss() < before, (before, losses)
