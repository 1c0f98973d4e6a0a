"""GPU: training on a batch of latents of different lengths, each padded at its end (`Model.forward(lengths=)`,
`NaturalSpeech2.forward(latent_lens=)`).

The contract, in the manner of test_ragged_training_gpu.py, with sample b = x[b, :L_b]:
  * forward: the training forward's prediction rows [0, L_b) are bit-identical to the alone call (and to the inference
    forward's), rows past L_b are exact zeros; each masked MSE row is bit-identical to the alone one;
  * backward of sum_b w_b mse_b: every parameter gradient equals sum_b w_b g_b (g_b: the gradient of the alone call's
    MSE) within a relative L2 of RTOL = 2^-19, the bound of test_ragged_training_gpu.py (fp32 summation order of the
    weight gradients differs between a batch and an alone call).  The lengths stay within one 128-key attention tile:
    past it the attention backward adds dQ of several key tiles with atomics in a varying order, and batch and alone
    can then differ by more than 2^-19 (see test_ragged_training_fp64_gpu.py);
  * padding: d cond and d x rows past L_b and d prompt rows past prompt_lens are exact zeros; NaN in the padded x rows
    reaches no output and no gradient;
  * lengths all equal to N reproduce the call without lengths: the forward bit for bit, the gradients within RTOL.
Unconditional and conditional (with prompt_lens) Models at small dims; NaturalSpeech2.forward with the conditioner.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu
dev = "cuda"
N, D, DP, NP = 100, 128, 128, 24
LENS = [1, 37, 64, 100, 77]
PROMPT_LENS = [3, 24, 10, 24, 1]
B = len(LENS)
RTOL = 2.0 ** -19


def _model(cond):
    from naturalspeech2_pytorch_b200 import Model
    torch.manual_seed(0)
    kw = dict(dim_prompt=DP, condition_on_prompt=True, cond_drop_prob=0.0) if cond else {}
    return Model(dim=D, depth=2, heads=2, wavenet_layers=3, wavenet_stacks=2, **kw).to(dev).train()


def _close(got, want, what):
    if want is None:
        assert got is None or int((got != 0).sum()) == 0, what
        return
    got, want = got.double(), want.double()
    assert bool(torch.isfinite(got).all()), what
    err = (got - want).norm().item()
    rel = err / want.norm().item() if err > 0 else 0.0
    assert rel <= RTOL, (what, rel)


def _inputs(cond):
    g = torch.Generator(device=dev).manual_seed(1)
    x = torch.randn(B, N, D, device=dev, generator=g)
    target = torch.randn(B, N, D, device=dev, generator=g)
    times = torch.rand(B, device=dev, generator=g)
    w = torch.rand(B, device=dev, generator=g) + 0.5
    prompt = cnd = None
    if cond:
        prompt = torch.randn(B, NP, DP, device=dev, generator=g)
        cnd = torch.randn(B, DP, N, device=dev, generator=g)
    return x, target, times, w, prompt, cnd


def _nan_past(t, lens, dim=1):
    t = t.clone()
    for b, n in enumerate(lens):
        t[b].narrow(dim - 1, n, t.shape[dim] - n).fill_(float("nan"))
    return t


def _loss(model, x, target, times, w, prompt, cnd, lens=None, prompt_lens=None, wrt=()):
    from naturalspeech2_pytorch_b200 import training
    kw = {}
    if prompt is not None:
        kw = dict(prompt=prompt, cond=cnd)
        if prompt_lens is not None:
            kw["prompt_lens"] = prompt_lens
    lt = None if lens is None else torch.tensor(lens, dtype=torch.int32, device=dev)
    if lt is not None:
        kw["lengths"] = lt
    pred = model(x, times, **kw)
    rows = training.MseRowsFunction.apply(pred, target, lt)
    params = list(model.parameters())
    grads = torch.autograd.grad((rows * w).sum(), params + list(wrt), allow_unused=True)
    return pred.detach(), rows.detach(), grads[:len(params)], grads[len(params):]


@pytest.mark.parametrize("cond", [False, True], ids=["uncond", "cond_prompt_lens"])
def test_model_training_matches_each_sample_alone(cond):
    model = _model(cond)
    x, target, times, w, prompt, cnd = _inputs(cond)
    plens = PROMPT_LENS if cond else None
    wrt = ()
    xp = _nan_past(x, LENS).requires_grad_(True)
    if cond:
        prompt_in = _nan_past(prompt, PROMPT_LENS).requires_grad_(True)
        cnd_in = cnd.clone().requires_grad_(True)
        wrt = (prompt_in, cnd_in)
    else:
        prompt_in = cnd_in = None
    pred, rows, grads, dins = _loss(model, xp, target, times, w, prompt_in, cnd_in, LENS, plens, wrt)
    assert bool(torch.isfinite(pred).all())
    want = [None if g is None else torch.zeros_like(g, dtype=torch.float64) for g in grads]
    for b, n in enumerate(LENS):
        pa = None if not cond else prompt[b:b + 1, :PROMPT_LENS[b]].clone()
        ca = None if not cond else cnd[b:b + 1, :, :n].clone()
        p_b, r_b, g_b, _ = _loss(model, x[b:b + 1, :n].clone().requires_grad_(True), target[b:b + 1, :n].contiguous(),
                                 times[b:b + 1], w[b:b + 1], pa, ca)
        assert torch.equal(pred[b, :n], p_b[0]), b
        assert int((pred[b, n:] != 0).sum()) == 0, b
        assert torch.equal(rows[b], r_b[0]), b
        for k, g in enumerate(g_b):
            if g is not None:
                want[k] += g.double()
    for k, (name, _) in enumerate(model.named_parameters()):
        _close(grads[k], want[k] if grads[k] is not None or want[k] is not None else None, name)
    if cond:
        d_prompt, d_cond = dins
        for b, (n, m) in enumerate(zip(LENS, PROMPT_LENS)):
            assert int((d_prompt[b, m:] != 0).sum()) == 0, ("d prompt padding", b)
            assert int((d_cond[b, :, n:] != 0).sum()) == 0, ("d cond padding", b)
    with torch.no_grad():   # the training forward's valid rows are the inference forward's
        model.eval()
        kw = dict(prompt=prompt, cond=cnd, prompt_lens=plens) if cond else {}
        inf = model(x, times, lengths=LENS, **kw)
        model.train()
    for b, n in enumerate(LENS):
        assert torch.equal(inf[b, :n], pred[b, :n]), b


@pytest.mark.parametrize("cond", [False, True], ids=["uncond", "cond"])
def test_full_lengths_reproduce_the_call_without_lengths(cond):
    model = _model(cond)
    x, target, times, w, prompt, cnd = _inputs(cond)
    p_full, r_full, g_full, _ = _loss(model, x, target, times, w, prompt, cnd, [N] * B)
    p_none, r_none, g_none, _ = _loss(model, x, target, times, w, prompt, cnd)
    assert torch.equal(p_full, p_none) and torch.equal(r_full, r_none)
    for (name, _), a, c in zip(model.named_parameters(), g_full, g_none):
        _close(a, c, name)


def test_natural_speech2_forward_latent_lens(monkeypatch):
    """Each MSE row of NaturalSpeech2.forward(latent_lens=, prompt_lens=) is bit-identical to its alone run; the loss is
    mean(mse) * mean(weight) (ns2.py:1651-1666); gradients are finite and reach no padded prompt row."""
    from naturalspeech2_pytorch_b200 import NaturalSpeech2, training
    from naturalspeech2_pytorch_b200.diffusion import gamma_to_alpha_sigma
    model = _model(True)
    ns = NaturalSpeech2(model, target_sample_hz=24000, timesteps=3)
    rows = []
    mse_apply = training.MseRowsFunction.apply

    def spy(pred, target, lens=None):
        r = mse_apply(pred, target, lens)
        rows.append(r.detach().clone())
        return r
    monkeypatch.setattr(training.MseRowsFunction, "apply", spy)
    x, _, times, _, prompt, cnd = _inputs(True)
    noise = torch.randn(B, N, D, device=dev, generator=torch.Generator(device=dev).manual_seed(3))
    pe = _nan_past(prompt, PROMPT_LENS).requires_grad_(True)
    loss = ns(_nan_past(x, LENS), prompt_enc=pe, cond=cnd, times=times, noise=noise, latent_lens=LENS,
              prompt_lens=PROMPT_LENS)
    batch_rows = rows[-1]
    (d_pe,) = torch.autograd.grad(loss, [pe])
    for b, (n, m) in enumerate(zip(LENS, PROMPT_LENS)):
        ns(x[b:b + 1, :n], prompt_enc=prompt[b:b + 1, :m], cond=cnd[b:b + 1, :, :n], times=times[b:b + 1],
           noise=noise[b:b + 1, :n].contiguous())
        assert torch.equal(batch_rows[b], rows[-1][0]), b
        assert int((d_pe[b, m:] != 0).sum()) == 0, b
    assert bool(torch.isfinite(d_pe).all())
    alpha, sigma = gamma_to_alpha_sigma(ns.gamma_schedule(times), ns.scale)
    snr = (alpha * alpha) / (sigma * sigma)
    weight = snr.clamp(max=ns.min_snr_gamma) / (snr + 1) if ns.min_snr_loss_weight else snr / (snr + 1)
    want = batch_rows.double().mean() * weight.double().mean()
    assert abs(loss.item() - want.item()) <= 1e-5 * abs(want.item())


def test_natural_speech2_forward_refusals():
    from naturalspeech2_pytorch_b200 import NaturalSpeech2
    from naturalspeech2_pytorch_b200.encoders import Conditioner
    model = _model(True)
    x = torch.zeros(2, 16, D, device=dev)
    ns = NaturalSpeech2(model, target_sample_hz=24000, timesteps=3)
    with pytest.raises(ValueError, match="encoded latents"):
        ns(torch.zeros(2, 3200, device=dev), latent_lens=[8, 16])
    ns.rvq_cross_entropy_loss_weight = 0.5
    with pytest.raises(NotImplementedError, match="cross-entropy"):
        ns(x, codes=torch.zeros(2, 16, 8, dtype=torch.long, device=dev), latent_lens=[8, 16])
    for kw in (dict(train_duration_pitch=True), dict(train_dropout=True)):
        cn = Conditioner(dim_codebook=128, num_phoneme_tokens=40, **kw).to(dev).train()
        ns2 = NaturalSpeech2(model, target_sample_hz=24000, timesteps=3, conditioner=cn)
        with pytest.raises(NotImplementedError, match="latent_lens"):
            ns2(x, latent_lens=[8, 16])
