"""GPU: the denoiser's hand-written backward (`training.train_backward` and its building blocks) against float64
autograd of the torch port (`oracle.denoiser_torch_port.model_forward_autograd`, pinned to the reference's own fp64
gradients by tests/test_oracle_cpu.py) at the benchmarked dims: dim 512, all 8 Wavenet dilations (1 ... 128) in 8
groups, 4 stacks, depth 2.

Both sides see the same operands: every parameter, x, prompt, cond and d out are bf16-representable values (the packs
hold exactly the parameters; `train_backward` casts d out to bf16), so what is left is the rounding of activations and
gradients inside the kernels.  Every parameter gradient and d prompt / d cond is compared whole, with the denoiser's
family of tests/fp64_check.py:
  (i)  rel-L2 <= C x the rel-L2 of the same port in fp32 under torch.autocast("cuda", bfloat16) (the reference's own
       reduced-precision mode, same rounded operands) + floor;
  (ii) rel-L2 <= ceiling;
and elements whose fp64 gradient is exactly zero (null parameters at p = 0, conv taps that only ever read the causal
padding, curtailed cond frames) must be exactly zero.  Three deliberately wrong references (one dilation off, one tile
of d out rows missing, one drop flag flipped) must be rejected by the same bounds.

Measured on an H100 80GB HBM3 (700 W power limit), worst tensor per case, rel-L2 ours / autocast-bf16 of the same
tensor:
  A  uncond, B 2, N 1024                       transformer.layers.0.1.to_q.weight       8.9e-3 / 1.5e-2
  B  cond, p = 0.5 mixed masks, B 4, N 1024     transformer.layers.0.1.to_q.weight       9.9e-3 / 1.6e-2
  C  cond, heads 6, dim_prompt 320, Lc 900      perceiver_resampler.layers.0.0.to_q.weight 9.6e-3 / 1.3e-2
  C' same, Lc 700 (zero-padded frames)          transformer.layers.1.3.to_q.weight       9.4e-3 / 1.5e-2
  D  uncond, B 3, N 100                         transformer.layers.1.1.to_q.weight       1.1e-2 / 1.9e-2
On every tensor of every case ours / autocast-bf16 <= 0.81.  Against the bounds below the tightest tensor uses 73 %
of its bound (D's to_q, at the ceiling).  The wrong references sit at rel-L2 1.2 (dilation), 0.18 (row tile) and
0.54-0.79 (drop flag).  The whole module takes ~35 s.
"""
import time

import pytest
import torch

from fp64_check import DENOISER, assert_rejected, bf, bound, compare, over, round_params
from helpers import build_model
from restatements import drop_masks, port_grads

pytestmark = pytest.mark.gpu

WN = dict(depth=2, wavenet_layers=8, wavenet_stacks=4)
CASES = {
    # name: (model kwargs, B, N, prompt length, cond frames, cond_drop_prob)
    "A_uncond": (dict(dim=512, heads=8, **WN), 2, 1024, None, None, 0.),
    "B_cond_mixed_drop": (dict(dim=512, heads=8, dim_prompt=512, condition_on_prompt=True, **WN), 4, 1024, 103, 1024, .5),
    "C_cond_proj_curtailed": (dict(dim=512, heads=6, dim_prompt=320, condition_on_prompt=True, **WN), 3, 777, 45, 900, 0.),
    "C_cond_proj_padded": (dict(dim=512, heads=6, dim_prompt=320, condition_on_prompt=True, **WN), 3, 777, 45, 700, 0.),
    "D_short": (dict(dim=512, heads=8, **WN), 3, 100, None, None, 0.),
}
# gradients kept after a case for the sensitivity tests
KEEP = ("wavenet.stacks.3.blocks.7.conv.weight", "wavenet.stacks.3.blocks.0.conv.weight", "transformer.to_pred.1.weight",
        "transformer.layers.1.5.3.weight", "null_prompt_tokens", "null_prompt_cond", "perceiver_resampler.latents")


_CACHE = {}


def _case(name):
    """Run one case once: our backward, the fp64 reference and the autocast-bf16 run of the port; per-tensor statistics
    and the kept gradients."""
    if name in _CACHE:
        return _CACHE[name]
    kwargs, B, N, Np, Lc, p = CASES[name]
    t0 = time.perf_counter()
    model = build_model(kwargs, 1234, device="cuda").train()
    round_params(model)
    D = kwargs["dim"]
    g = torch.Generator().manual_seed(20)
    inp = {"x": bf(g, B, N, D), "times": torch.rand(B, generator=g).cuda()}
    if Np is not None:
        inp["prompt"], inp["cond"] = bf(g, B, Np, kwargs["dim_prompt"]), bf(g, B, kwargs["dim_prompt"], Lc)
    d_out = bf(g, B, N, D)
    seed, dp, dc = drop_masks(B, p)
    drop = (dp, dc) if Np is not None else (None, None)

    # ours: loss.backward() through DenoiserFunction, d prompt / d cond requested
    X = {k: inp[k].clone().requires_grad_(True) for k in ("prompt", "cond") if k in inp}
    if seed is not None:
        torch.manual_seed(seed)
    out = model(inp["x"], inp["times"], **X, **({"cond_drop_prob": p} if X else {}))
    out.backward(d_out)
    ours = {n: prm.grad for n, prm in model.named_parameters()}
    ours.update({f"d {k}": v.grad for k, v in X.items()})
    params = {n: prm.detach() for n, prm in model.named_parameters()}
    del out, X

    ref = port_grads(params, kwargs, inp, drop, d_out)
    ac = port_grads(params, kwargs, inp, drop, d_out, autocast=True)
    assert set(ref) == set(ours)
    stats, fails = {}, []
    for n, r in ref.items():
        assert ours[n] is not None, n
        s = compare(ours[n], r, ac[n], max_abs=True)
        if isinstance(s, str):
            fails.append((n, s))
        elif s is not None:
            stats[n] = s
    res = dict(kwargs=kwargs, params=params, inp=inp, d_out=d_out, drop=drop, stats=stats, fails=fails,
               ours={n: ours[n].clone() for n in KEEP if n in ours},
               zeros={n: (ours[n].clone(), ref[n].clone()) for n in ("d cond",) if n in ours},
               conv_taps={n: (ours[n].clone(), ref[n].clone()) for n in ours if n.endswith(".conv.weight")}
               if N < 256 else {}, seconds=time.perf_counter() - t0)
    model.zero_grad(set_to_none=True)
    del ours, ref, ac, model
    torch.cuda.empty_cache()
    _CACHE[name] = res
    return res


@pytest.mark.parametrize("name", list(CASES))
def test_backward_matches_fp64_autograd(name):
    r = _case(name)
    stats = r["stats"]
    ranked = sorted(stats.items(), key=lambda kv: kv[1].rel / bound(DENOISER, kv[1].rel_ac), reverse=True)
    worst_rel = max(stats.items(), key=lambda kv: kv[1].rel)
    ratio = max(s.rel / s.rel_ac for s in stats.values())
    print(f"\n{name}: {len(stats)} tensors compared in {r['seconds']:.1f} s; worst rel-L2 {worst_rel[0]}: "
          f"ours {worst_rel[1].rel:.3e} autocast-bf16 {worst_rel[1].rel_ac:.3e}; max ratio ours / autocast-bf16 {ratio:.2f}")
    for n, s in ranked[:8]:
        print(f"  {n}: rel-L2 ours {s.rel:.3e} / autocast-bf16 {s.rel_ac:.3e} (bound {bound(DENOISER, s.rel_ac):.3e}); "
              f"max-abs ours {s.max_abs:.3e} / autocast-bf16 {s.max_abs_ac:.3e} (max |ref| {s.max_ref:.3e})")
    assert not r["fails"], f"non-finite, or non-zero where the fp64 gradient is exactly zero: {r['fails'][:8]}"
    bad = [(n, s.rel, s.rel_ac) for n, s in ranked if over(DENOISER, s)]
    assert not bad, f"{len(bad)} tensors over the bound (name, rel-L2, autocast rel-L2): {bad[:8]}"


def test_short_sequence_conv_taps_beyond_n_are_exact_zeros():
    """N = 100: the taps of the dilation-64 / -128 convs whose shift (2 - t) 2^g >= N only read the causal padding."""
    r = _case("D_short")
    N = CASES["D_short"][2]
    checked = 0
    for n, (o, ref) in r["conv_taps"].items():
        g = int(n.split(".")[4])
        for t in range(3):
            if (2 - t) * 2 ** g >= N:
                o_t = o.reshape(ref.shape)[:, :, t]
                assert float(ref[:, :, t].abs().max()) == 0.0, (n, t)
                assert int((o_t != 0).sum()) == 0, (n, t, float(o_t.abs().max()))
                checked += 1
    assert checked == 4 * 3   # stacks x (one tap at dilation 64, two at 128)


def test_curtailed_cond_frames_get_exact_zero_gradient():
    r = _case("C_cond_proj_curtailed")
    N = CASES["C_cond_proj_curtailed"][2]
    o, ref = r["zeros"]["d cond"]
    assert o.shape == ref.shape and o.shape[-1] > N
    assert int((o[:, :, N:] != 0).sum()) == 0
    assert float(ref[:, :, N:].abs().max()) == 0.0 and float(ref[:, :, :N].abs().max()) > 0


def _assert_rejected(r, wrong, names):
    assert_rejected(r["ours"], wrong, r["stats"], names, DENOISER)


def test_rejects_reference_with_one_dilation_off():
    """Block 7 of the last stack at dilation 64 instead of 128."""
    r = _case("A_uncond")
    kw = r["kwargs"]
    dil = [[2 ** i for i in range(kw["wavenet_layers"])] for _ in range(kw["wavenet_stacks"])]
    dil[-1][-1] = 64
    name = "wavenet.stacks.3.blocks.7.conv.weight"
    wrong = port_grads(r["params"], kw, r["inp"], r["drop"], r["d_out"], dilations=dil, only=[name])
    _assert_rejected(r, wrong, [name])


def test_rejects_reference_with_one_row_tile_missing():
    """d out with the last 64 rows of sample 0 zeroed."""
    r = _case("A_uncond")
    d_out = r["d_out"].clone()
    d_out[0, -64:] = 0
    names = ["transformer.to_pred.1.weight", "transformer.layers.1.5.3.weight", "wavenet.stacks.3.blocks.0.conv.weight"]
    wrong = port_grads(r["params"], r["kwargs"], r["inp"], r["drop"], d_out, only=names)
    _assert_rejected(r, wrong, names)


def test_rejects_reference_with_one_drop_flag_flipped():
    """Case B with one sample's prompt-drop flag flipped."""
    r = _case("B_cond_mixed_drop")
    dp, dc = r["drop"]
    dp = dp.clone()
    dp[0] = ~dp[0]
    names = ["null_prompt_tokens", "null_prompt_cond", "perceiver_resampler.latents"]
    wrong = port_grads(r["params"], r["kwargs"], r["inp"], (dp, dc), r["d_out"], only=names)
    _assert_rejected(r, wrong, names)
