"""CPU: the denoiser feed-forward's folded conv pack (`model._fold_conv_linear`).  The causal k=3 conv and the output
projection after it (ns2.py:1019-1024) run as one conv whose tap t is W2 @ Wc[:, :, t] and whose bias is W2 @ bc + b2.
Checked against the float64 products of the module's own parameters: values, the exactly-zero padding columns, the
transposed twin the backward's dgrad reads, and that the folded conv computes the unfolded pair, first rows included."""
import pytest
import torch

from naturalspeech2_pytorch_b200 import Model
from naturalspeech2_pytorch_b200.model import _round_up


@pytest.fixture(scope="module")
def model():
    torch.manual_seed(0)
    return Model(dim=128, depth=2, heads=2, wavenet_layers=2, wavenet_stacks=1)


def _fold64(ff):
    """float64 (taps (3, D, Di), bias (D,)) of FeedForward Sequential `ff` = [lin1, GEGLU, conv, lin2]."""
    wc, w2 = ff[2][1].weight.detach().double(), ff[-1].weight.detach().double()
    taps = torch.stack([w2 @ wc[:, :, t] for t in range(3)])
    return taps, w2 @ ff[2][1].bias.detach().double() + ff[-1].bias.detach().double()


def test_folded_pack_and_bias_match_the_float64_product(model):
    P, D, Di = model.packed(), model.dim, model.ff_inner
    Dp = _round_up(Di, 128)
    for l, layer in enumerate(model.transformer.layers):
        taps, bias = _fold64(layer[5])
        wo, bo = P[f"l{l}_ff_wo"], P[f"l{l}_ff_bo"]
        assert wo.dtype == torch.bfloat16 and wo.shape == (D, 3 * Dp)
        assert bo.dtype == torch.float32 and bo.shape == (D,)
        for t in range(3):
            got = wo[:, t * Dp:t * Dp + Di].double()
            # rounded to bf16 once: within half an ulp (<= 2^-8 |w|; fp32's half ulp on the way is 2^-16 of that)
            assert bool(((got - taps[t]).abs() <= 2.0 ** -8 * (1 + 2.0 ** -15) * taps[t].abs()).all()), (l, t)
            assert (got == taps[t].float().bfloat16().double()).float().mean() > 0.999, (l, t)
            assert not wo[:, t * Dp + Di:(t + 1) * Dp].any(), f"layer {l} tap {t}: padding columns must be exactly 0"
        assert bool(((bo.double() - bias).abs() <= 2.0 ** -24 * bias.abs()).all()), l


def test_folded_pack_keeps_the_unfolded_packs(model):
    P = model.packed()
    for l in range(model.depth):
        for k in ("wc", "bc", "w2", "b2"):   # the backward's W2 / conv gradients read them
            assert f"l{l}_ff_{k}" in P


def test_folded_transposed_twin_is_in_tap_out(model):
    P, T, D = model.packed(), model.packed_transposed(), model.dim
    Dp = _round_up(model.ff_inner, 128)
    for l in range(model.depth):
        fwd, tr = P[f"l{l}_ff_wo"], T[f"l{l}_ff_wo"]
        assert tr.shape == (Dp, 3 * D)
        assert torch.equal(tr.view(Dp, 3, D), fwd.view(D, 3, Dp).permute(2, 1, 0))


def test_folded_conv_computes_conv_then_linear_on_every_row(model):
    """y[n] = sum_t W'_t g[n - 2 + t] + b' equals W2 (conv(g) + bc) + b2 with the causal zero padding, rows 0 and 1
    (whose first taps read the padding) included; evaluated in float64 on the bf16 pack."""
    P, D, Di = model.packed(), model.dim, model.ff_inner
    Dp = _round_up(Di, 128)
    ff = model.transformer.layers[0][5]
    g = torch.randn(2, 5, Di, dtype=torch.float64)
    gp = torch.nn.functional.pad(g.transpose(1, 2), (2, 0))                        # causal padding (ns2.py:583-595)
    c = torch.nn.functional.conv1d(gp, ff[2][1].weight.double(), ff[2][1].bias.double()).transpose(1, 2)
    ref = c @ ff[-1].weight.double().T + ff[-1].bias.double()
    wo = P["l0_ff_wo"].double().view(D, 3, Dp)[:, :, :Di]
    gz = torch.cat((torch.zeros(2, 2, Di, dtype=torch.float64), g), dim=1)
    got = sum(gz[:, t:t + 5] @ wo[:, t].T for t in range(3)) + P["l0_ff_bo"].double()
    mag = sum(gz[:, t:t + 5].abs() @ wo[:, t].abs().T for t in range(3)) + P["l0_ff_bo"].double().abs()
    assert bool(((got - ref).abs() <= 2.0 ** -8 * mag).all())


def test_fold_follows_a_parameter_update(model):
    P = model.packed()
    wo, bo = P["l1_ff_wo"], P["l1_ff_bo"]
    with torch.no_grad():
        model.transformer.layers[1][5][2][1].bias.add_(1.0)   # an optimizer step bumps the version counter
    P2 = model.packed()
    assert torch.equal(P2["l1_ff_wo"], wo)
    taps, bias = _fold64(model.transformer.layers[1][5])
    assert not torch.equal(P2["l1_ff_bo"], bo)
    assert bool(((P2["l1_ff_bo"].double() - bias).abs() <= 2.0 ** -24 * bias.abs()).all())
