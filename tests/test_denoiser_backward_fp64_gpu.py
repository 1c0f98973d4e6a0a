"""GPU: the denoiser's hand-written backward (`training.train_backward` and its building blocks) against float64
autograd of the torch port (`oracle.denoiser_torch_port.model_forward_autograd`, pinned to the reference's own fp64
gradients by tests/test_oracle_cpu.py) at the benchmarked dims: dim 512, all 8 Wavenet dilations (1 ... 128) in 8
groups, 4 stacks, depth 2.

Both sides see the same operands: every parameter, x, prompt, cond and d out are bf16-representable values (the packs
hold exactly the parameters; `train_backward` casts d out to bf16), so what is left is the rounding of activations and
gradients inside the kernels.  Every parameter gradient and d prompt / d cond is compared whole:
  (i)  rel-L2 <= C_AUTOCAST x the rel-L2 of the same port in fp32 under torch.autocast("cuda", bfloat16) (the
       reference's own reduced-precision mode, same rounded operands) + REL_FLOOR;
  (ii) rel-L2 <= REL_CEILING;
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

from helpers import build_model, oracle_config
from oracle import denoiser_torch_port as tp

pytestmark = pytest.mark.gpu

C_AUTOCAST = 1.0     # measured ratio ours / autocast-bf16 <= 0.81 on every tensor of every case
REL_FLOOR = 2e-3
REL_CEILING = 1.5e-2  # measured worst 1.1e-2 (case D)

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


def _rel(got, ref):
    return float((got.double() - ref).norm() / ref.norm())


def _drop_masks(B, p):
    """(seed, prompt-drop mask, cond-drop mask) as Model.forward draws them after torch.manual_seed(seed): prompt first,
    cond second (`model._prob_mask_like`); for 0 < p < 1 the first seed where each mask drops some samples and keeps
    others."""
    if p == 0:
        zeros = torch.zeros(B, dtype=torch.bool, device="cuda")
        return None, zeros, zeros
    for seed in range(100):
        torch.manual_seed(seed)
        dp = torch.zeros((B,), device="cuda").float().uniform_(0, 1) < p
        dc = torch.zeros((B,), device="cuda").float().uniform_(0, 1) < p
        if 0 < int(dp.sum()) < B and 0 < int(dc.sum()) < B:
            return seed, dp, dc
    raise AssertionError("no seed gives mixed drop masks")


def _port_grads(params, kwargs, inp, drop, d_out, dtype=torch.float64, autocast=False, dilations=None, only=None):
    """{name: d out-weighted gradient} of the torch port on `params` (the model's rounded fp32 values) in `dtype`,
    optionally under bf16 autocast; names are the parameters' and "d prompt" / "d cond"."""
    P = {n: p.detach().to(dtype).requires_grad_(True) for n, p in params.items()}
    X = {k: inp[k].to(dtype).requires_grad_(True) for k in ("prompt", "cond") if k in inp}
    leaves = dict(P, **{f"d {k}": v for k, v in X.items()})
    names = list(leaves) if only is None else list(only)
    with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
        out = tp.model_forward_autograd(P, oracle_config(kwargs), inp["x"].to(dtype), inp["times"].to(dtype),
                                        X.get("prompt"), X.get("cond"), drop_prompt=drop[0], drop_cond=drop[1],
                                        dilations=dilations)
    g = torch.autograd.grad(out, [leaves[n] for n in names], d_out.to(out.dtype), allow_unused=True)
    return {n: torch.zeros_like(leaves[n]) if gi is None else gi.detach() for n, gi in zip(names, g)}


_CACHE = {}


def _case(name):
    """Run one case once: our backward, the fp64 reference and the autocast-bf16 run of the port; per-tensor statistics
    and the kept gradients."""
    if name in _CACHE:
        return _CACHE[name]
    kwargs, B, N, Np, Lc, p = CASES[name]
    t0 = time.perf_counter()
    model = build_model(kwargs, 1234, device="cuda").train()
    with torch.no_grad():
        for prm in model.parameters():
            prm.copy_(prm.bfloat16().float())        # the packs hold exactly these values
    D = kwargs["dim"]
    g = torch.Generator().manual_seed(20)
    bf = lambda *s: torch.randn(*s, generator=g).bfloat16().float().cuda()  # noqa: E731
    inp = {"x": bf(B, N, D), "times": torch.rand(B, generator=g).cuda()}
    if Np is not None:
        inp["prompt"], inp["cond"] = bf(B, Np, kwargs["dim_prompt"]), bf(B, kwargs["dim_prompt"], Lc)
    d_out = bf(B, N, D)
    seed, dp, dc = _drop_masks(B, p)
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

    ref = _port_grads(params, kwargs, inp, drop, d_out)
    ac = _port_grads(params, kwargs, inp, drop, d_out, dtype=torch.float32, autocast=True)
    assert set(ref) == set(ours)
    stats, zero_fail, nonfinite = {}, [], []
    for n, r in ref.items():
        o = ours[n]
        assert o is not None, n
        o = o.reshape(r.shape)
        if not bool(torch.isfinite(o).all()):
            nonfinite.append(n)
            continue
        zero = r == 0
        if bool(zero.any()) and bool((o[zero] != 0).any()):
            zero_fail.append((n, int((o[zero] != 0).sum()), int(zero.sum())))
        if bool(zero.all()):
            continue
        stats[n] = (_rel(o, r), _rel(ac[n], r), float((o.double() - r).abs().max()),
                    float((ac[n].double() - r).abs().max()), float(r.abs().max()))
    res = dict(kwargs=kwargs, params=params, inp=inp, d_out=d_out, drop=drop, stats=stats, zero_fail=zero_fail,
               nonfinite=nonfinite, ours={n: ours[n].clone() for n in KEEP if n in ours},
               zeros={n: (ours[n].clone(), ref[n].clone()) for n in ("d cond",) if n in ours},
               conv_taps={n: (ours[n].clone(), ref[n].clone()) for n in ours if n.endswith(".conv.weight")}
               if N < 256 else {}, seconds=time.perf_counter() - t0)
    model.zero_grad(set_to_none=True)
    del ours, ref, ac, model
    torch.cuda.empty_cache()
    _CACHE[name] = res
    return res


def _bound(rel_ac):
    return min(C_AUTOCAST * rel_ac + REL_FLOOR, REL_CEILING)


def _fails(got, ref, rel_ac):
    rel = _rel(got, ref)
    return rel > _bound(rel_ac), rel


@pytest.mark.parametrize("name", list(CASES))
def test_backward_matches_fp64_autograd(name):
    r = _case(name)
    stats = r["stats"]
    assert not r["nonfinite"], r["nonfinite"][:8]
    ranked = sorted(stats.items(), key=lambda kv: kv[1][0] / _bound(kv[1][1]), reverse=True)
    worst_rel = max(stats.items(), key=lambda kv: kv[1][0])
    ratio = max(s[0] / s[1] for s in stats.values())
    print(f"\n{name}: {len(stats)} tensors compared in {r['seconds']:.1f} s; worst rel-L2 {worst_rel[0]}: "
          f"ours {worst_rel[1][0]:.3e} autocast-bf16 {worst_rel[1][1]:.3e}; max ratio ours / autocast-bf16 {ratio:.2f}")
    for n, (rel, rel_ac, mx, mx_ac, rmax) in ranked[:8]:
        print(f"  {n}: rel-L2 ours {rel:.3e} / autocast-bf16 {rel_ac:.3e} (bound {_bound(rel_ac):.3e}); "
              f"max-abs ours {mx:.3e} / autocast-bf16 {mx_ac:.3e} (max |ref| {rmax:.3e})")
    assert not r["zero_fail"], f"non-zero where the fp64 gradient is exactly zero: {r['zero_fail'][:8]}"
    bad = [(n, s[0], s[1]) for n, s in ranked if s[0] > _bound(s[1])]
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
    for n in names:
        fails, rel = _fails(r["ours"][n].reshape(wrong[n].shape), wrong[n], r["stats"][n][1])
        print(f"  {n}: rel-L2 vs the wrong reference {rel:.3e} (bound {_bound(r['stats'][n][1]):.3e})")
        assert fails, f"{n}: the bound accepts a wrong reference (rel-L2 {rel:.3e})"


def test_rejects_reference_with_one_dilation_off():
    """Block 7 of the last stack at dilation 64 instead of 128."""
    r = _case("A_uncond")
    kw = r["kwargs"]
    dil = [[2 ** i for i in range(kw["wavenet_layers"])] for _ in range(kw["wavenet_stacks"])]
    dil[-1][-1] = 64
    name = "wavenet.stacks.3.blocks.7.conv.weight"
    wrong = _port_grads(r["params"], kw, r["inp"], r["drop"], r["d_out"], dilations=dil, only=[name])
    _assert_rejected(r, wrong, [name])


def test_rejects_reference_with_one_row_tile_missing():
    """d out with the last 64 rows of sample 0 zeroed."""
    r = _case("A_uncond")
    d_out = r["d_out"].clone()
    d_out[0, -64:] = 0
    names = ["transformer.to_pred.1.weight", "transformer.layers.1.5.3.weight", "wavenet.stacks.3.blocks.0.conv.weight"]
    wrong = _port_grads(r["params"], r["kwargs"], r["inp"], r["drop"], d_out, only=names)
    _assert_rejected(r, wrong, names)


def test_rejects_reference_with_one_drop_flag_flipped():
    """Case B with one sample's prompt-drop flag flipped."""
    r = _case("B_cond_mixed_drop")
    dp, dc = r["drop"]
    dp = dp.clone()
    dp[0] = ~dp[0]
    names = ["null_prompt_tokens", "null_prompt_cond", "perceiver_resampler.latents"]
    wrong = _port_grads(r["params"], r["kwargs"], r["inp"], (dp, dc), r["d_out"], only=names)
    _assert_rejected(r, wrong, names)
