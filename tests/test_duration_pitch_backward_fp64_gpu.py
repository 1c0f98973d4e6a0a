"""GPU: the duration / pitch predictor's hand-written backward (`DurationPitchPredictor` through `encoders.
_EncoderFunction`) against float64 autograd on the GPU at the reference's default dims: dim 512, depth 10, 8 heads,
3 ResnetBlocks x 2 k=3 convs per layer, both trunks.

The reference is `oracle.encoders_oracle.duration_pitch_predictor`, pinned to the reference module by
tests/test_encoders_cpu.py (and, with a token table, the table gathered in front of it).  Both sides see the same
operands: every parameter is rounded to bf16 in place, inputs, prompts and upstream gradients are bf16-representable.
The fp64 reference runs with cuDNN off, so conv taps that only read the zero padding get exactly zero gradients.
Every parameter gradient, d x (or the token table's gradient) and d prompts are compared whole, with the predictor's
family of tests/fp64_check.py (the encoders' numbers): rel-L2 <= C x the rel-L2 of the same restatement under bf16
autocast + floor, and <= ceiling; exact zeros where fp64 is zero; nothing non-finite.  to_q needs no bound of
its own here: the conditioning test bounds it relative to the fused q / kv gradient because nearly flat self-attention
leaves its exact gradient below the rounding of D = rowsum(dO * O); with the prompts among the keys the predictor's
attention is not that flat, and to_q meets the common bound (ours at most 1.1 x its autocast twin).  Its error as a
share of the q / kv gradient is printed for comparison (measured worst 4.9e-3).

ReLU heads: a row whose head pre-activation lies within the forward error of 0 could take the other branch in fp64.
Each case sets the two head biases (bf16 values) from the fp64 pre-activations so that every |pre| is at least
MARGIN x the measured max-abs error of our predictions, and asserts it: in most cases every row is alive; where the
sorted pre-activations leave a wide enough gap (the short cases) the bias puts the threshold in it, so some rows are
dead and their gradient must be exactly zero.

Wrong references that the same bounds must reject: one conv's taps reversed, GroupNorm with 4 groups instead of 8,
keys without the queries (cross_attn_include_queries off), and the two trunks' upstream gradients swapped.

Measured on an H100 80GB HBM3 (700 W power limit).  Worst tensor per case, rel-L2 ours / autocast-bf16 of the same
tensor; the largest ours / autocast ratio; our forward's max-abs error and the smallest |pre-activation| (>= 20x it):
  main      B 4, T 100, Np 103   to_duration_pred.layers.9.0.2.blocks.0.norm.weight   1.10e-2 / 1.42e-2   1.01   3.6e-2 / 3.8
  short     B 3, T 5, Np 3       to_duration_pred.layers.4.1.gamma                    1.10e-2 / 9.9e-3    1.11   2.9e-2 / 2.8
  one       B 2, T 1, Np 7       to_pitch_pred.layers.0.0.2.blocks.0.norm.weight      9.5e-3 / 1.19e-2    1.28   2.1e-2 / 1.3
  table     token table, T 50    to_duration_pred.layers.7.0.0.blocks.0.proj.weight   1.28e-2 / 1.82e-2   0.99   5.2e-2 / 2.3
  dur_only  only duration_pred   to_duration_pred.layers.0.2.to_q.weight              7.0e-3 / 1.07e-2    0.90   3.5e-2 / 2.5
The tightest tensor uses 71 % of its bound (one: a to_q, at 1.28 x its twin); "one" has 2 ReLU-dead rows.  Each case
takes about 5 s.
"""
import time

import pytest
import torch

from fp64_check import MARGIN, PREDICTOR, assert_rejected, autograd, bf, bound, compare, over, round_params
from oracle import encoders_oracle as eo
from param_fill import fill_module
from restatements import DPP_DEPTH as DEPTH
from restatements import DPP_DIM as DIM
from restatements import DPP_HEADS as HEADS
from restatements import TRUNKS, predictor_fwd, set_head_biases

pytestmark = pytest.mark.gpu

NUM_TOKENS = 100
CASES = {
    # name: (B, T, Np, token table, which predictions get a gradient)
    "main": (4, 100, 103, False, "both"),
    "short": (3, 5, 3, False, "both"),
    "one": (2, 1, 7, False, "both"),
    "table": (2, 50, 40, True, "both"),
    "dur_only": (2, 40, 30, False, "duration"),
}


def _is_q(name):
    return name.endswith(".2.to_q.weight")


def _predictor(table):
    from naturalspeech2_pytorch_b200.encoders import DurationPitchPredictor
    m = DurationPitchPredictor(dim=DIM, num_phoneme_tokens=NUM_TOKENS if table else None)
    fill_module(m, 4321)
    m.cuda()
    round_params(m)
    assert (m.heads, len(m.to_duration_pred.layers), len(m.to_duration_pred.layers[0][0])) == (HEADS, DEPTH, 3)
    return m


def _trunk_without_query_keys(P, pre, x, prompts, heads, groups=8, eps=1e-5):
    """A wrong reference: eo._trunk restated with keys / values from the prompts alone (cross_attn_include_queries
    off, ns2.py:1060-1061)."""
    import torch.nn.functional as F
    for l in range(DEPTH):
        lp = f"{pre}layers.{l}."
        for r in range(3):
            h = x.transpose(1, 2)
            for c in range(2):
                bp = f"{lp}0.{r}.blocks.{c}."
                h = F.conv1d(h, P[bp + "proj.weight"], P[bp + "proj.bias"], padding=1)
                h = F.silu(F.group_norm(h, groups, P[bp + "norm.weight"], P[bp + "norm.bias"], eps))
            x = h.transpose(1, 2) + x
        nx = eo._rmsnorm(x, P[lp + "1.gamma"])
        q = nx @ P[lp + "2.to_q.weight"].T
        k, v = (prompts @ P[lp + "2.to_kv.weight"].T).chunk(2, dim=-1)
        b, n, _ = q.shape
        q, k, v = (t.view(b, t.shape[1], heads, -1).transpose(1, 2) for t in (q, k, v))
        sim = torch.einsum("bhid,bhjd->bhij", q, k) * (q.shape[-1] ** -0.5)
        o = torch.einsum("bhij,bhjd->bhid", sim.softmax(dim=-1), v).transpose(1, 2).reshape(b, n, -1)
        x = o @ P[lp + "2.to_out.weight"].T + x
    return F.relu(x @ P[pre + "to_pred.0.weight"].T + P[pre + "to_pred.0.bias"]).squeeze(-1)


_CACHE = {}


def _case(name):
    if name in _CACHE:
        return _CACHE[name]
    t0 = time.perf_counter()
    B, T, Np, table, which = CASES[name]
    m = _predictor(table)
    g = torch.Generator().manual_seed(7 + list(CASES).index(name))
    x = torch.randint(0, NUM_TOKENS, (B, T), generator=g).cuda() if table else bf(g, B, T, DIM)
    prompts = bf(g, B, Np, DIM)
    biases = set_head_biases(m, x, prompts, table)
    d_outs = {"duration": bf(g, B, T, scale=0.05), "pitch": bf(g, B, T, scale=0.05) if which == "both" else None}

    # ours
    m.train()
    x_in = x if table else x.clone().requires_grad_(True)
    p_in = prompts.clone().requires_grad_(True)
    dur, pitch = m(x_in, p_in)
    outs = [(dur, d_outs["duration"])] + ([(pitch, d_outs["pitch"])] if which == "both" else [])
    torch.autograd.backward([o for o, _ in outs], [d for _, d in outs])
    ours = {n: p.grad for n, p in m.named_parameters()}
    if not table:
        ours["x"] = x_in.grad
    ours["prompts"] = p_in.grad
    ours.update({"out duration": dur.detach(), "out pitch": pitch.detach()})
    m.eval()
    with torch.no_grad():
        ev = m(x, prompts)
    train_equals_eval = torch.equal(ev[0], dur.detach()) and torch.equal(ev[1], pitch.detach())

    params = {n: p.detach() for n, p in m.named_parameters()}
    inputs = {"prompts": prompts} if table else {"x": x, "prompts": prompts}
    fwd = predictor_fwd(x, prompts, table)
    # cuDNN off for both runs: conv taps that only read the zero padding get exact zeros
    ref = autograd(fwd, params, d_outs, inputs=inputs, cudnn=False, out_prefix="out ")
    ac = autograd(fwd, params, d_outs, autocast=True, inputs=inputs, cudnn=False, out_prefix="out ")

    # the ReLU margin: every fp64 pre-activation at least MARGIN x our forward's max-abs error away from 0
    fwd_err = max(float((ours["out " + k].double() - ref["out " + k]).abs().max()) for k in ("duration", "pitch"))
    P64 = {n: p.double() for n, p in params.items()}
    for t in TRUNKS:
        P64[t + "to_pred.0.bias"] = P64[t + "to_pred.0.bias"] + 1e3
    with torch.backends.cudnn.flags(enabled=False):
        pre = predictor_fwd(x, prompts, table)(P64, torch.float64)
    min_pre = min(float((pre[k] - 1e3).abs().min()) for k in ("duration", "pitch"))
    dead = sum(int((pre[k] - 1e3 < 0).sum()) for k in ("duration", "pitch"))

    stats, fails, none_ok = {}, [], True
    for n, r in ref.items():
        o = ours.get(n)
        if which == "duration" and n.startswith(TRUNKS[1]):
            none_ok &= o is None
            continue
        assert o is not None and o.shape == r.shape, n
        s = compare(o, r, ac[n], ref[n.replace("to_q", "to_kv")] if _is_q(n) else None)
        if isinstance(s, str):
            fails.append((n, s))
        elif s is not None and not n.startswith("out "):
            stats[n] = s
    res = dict(stats=stats, fails=fails, none_ok=none_ok, fwd_err=fwd_err,
               min_pre=min_pre, dead=dead, biases=biases, train_equals_eval=train_equals_eval, params=params,
               inputs=inputs, d_outs=d_outs, x=x, prompts=prompts, table=table,
               ours={n: ours[n].clone() for n in ("to_duration_pred.layers.0.0.0.blocks.0.proj.weight",
                                                  "to_duration_pred.layers.9.0.2.blocks.1.norm.weight",
                                                  "to_duration_pred.layers.9.2.to_kv.weight",
                                                  "to_pitch_pred.layers.9.0.0.blocks.0.proj.weight", "prompts")
                     if ours.get(n) is not None})
    del ours, ref, ac
    torch.cuda.empty_cache()
    res["seconds"] = time.perf_counter() - t0
    _CACHE[name] = res
    return res


@pytest.mark.parametrize("name", list(CASES))
def test_backward_matches_fp64_autograd(name):
    r = _case(name)
    stats = r["stats"]
    q = {n: s for n, s in stats.items() if _is_q(n)}
    worst = max(stats.items(), key=lambda kv: kv[1].rel)
    ratio = max(((n, s) for n, s in stats.items() if s.rel_ac > 0), key=lambda kv: kv[1].rel / kv[1].rel_ac)
    use = max(stats.items(), key=lambda kv: kv[1].rel / bound(PREDICTOR, kv[1].rel_ac))
    worst_q = max(q.items(), key=lambda kv: kv[1].share)
    print(f"\n{name}: {len(stats)} tensors in {r['seconds']:.1f} s; worst rel-L2 {worst[0]} ours {worst[1].rel:.3e} / "
          f"autocast {worst[1].rel_ac:.3e}; max ratio {ratio[1].rel / ratio[1].rel_ac:.2f} ({ratio[0]}); tightest "
          f"{use[0]} at {use[1].rel / bound(PREDICTOR, use[1].rel_ac):.0%} of its bound; worst to_q {worst_q[0]} "
          f"{worst_q[1].share:.3e}; forward max-abs {r['fwd_err']:.3e}, min |pre| {r['min_pre']:.3e}, dead rows "
          f"{r['dead']}, head biases {r['biases']}")
    assert r["min_pre"] >= MARGIN * r["fwd_err"], "fixture: a head pre-activation lies too close to 0"
    assert r["train_equals_eval"], "the training forward must be bit-identical to the inference forward"
    assert r["none_ok"], "a trunk without an upstream gradient must leave its parameters' .grad None"
    assert not r["fails"], f"non-finite, or non-zero where the fp64 value is exactly zero: {r['fails'][:8]}"
    bad = [(n, s) for n, s in stats.items() if over(PREDICTOR, s)]
    assert not bad, f"{len(bad)} tensors over the bound: {bad[:8]}"


def test_short_cases_cover_dead_rows_and_padding_taps():
    """T = 1: the k=3 taps 0 and 2 only read the zero padding, so their gradients are exactly zero (checked by the
    zero rule of the main test); its head biases leave ReLU-dead rows, whose gradients must be exactly zero too."""
    r = _case("one")
    assert r["dead"] > 0
    assert "to_duration_pred.layers.0.0.0.blocks.0.proj.weight" in r["stats"]


# ---- wrong references ----
def _assert_rejected(r, wrong, names):
    assert_rejected(r["ours"], wrong, r["stats"], names, PREDICTOR)


def _wrong(r, fwd, d_outs, names):
    return autograd(fwd, r["params"], d_outs, inputs=r["inputs"], only=names, cudnn=False)


def test_rejects_reversed_conv_taps():
    r = _case("main")
    key = "to_duration_pred.layers.0.0.0.blocks.0.proj.weight"
    base = predictor_fwd(r["x"], r["prompts"], r["table"])

    def fwd(P, dtype):
        return base(dict(P, **{key: P[key].flip(-1)}), dtype)
    _assert_rejected(r, _wrong(r, fwd, r["d_outs"], [key]), [key])


def test_rejects_wrong_group_count():
    r = _case("main")
    names = ["to_duration_pred.layers.9.0.2.blocks.1.norm.weight"]
    fwd = predictor_fwd(r["x"], r["prompts"], r["table"], groups=4)
    _assert_rejected(r, _wrong(r, fwd, r["d_outs"], names), names)


def test_rejects_keys_without_the_queries():
    r = _case("main")
    names = ["to_duration_pred.layers.9.2.to_kv.weight", "prompts"]
    fwd = predictor_fwd(r["x"], r["prompts"], r["table"], trunk=_trunk_without_query_keys)
    _assert_rejected(r, _wrong(r, fwd, r["d_outs"], names), names)


def test_rejects_swapped_trunks():
    r = _case("main")
    names = ["to_duration_pred.layers.0.0.0.blocks.0.proj.weight", "to_pitch_pred.layers.9.0.0.blocks.0.proj.weight"]
    d = r["d_outs"]
    fwd = predictor_fwd(r["x"], r["prompts"], r["table"])
    _assert_rejected(r, _wrong(r, fwd, {"duration": d["pitch"], "pitch": d["duration"]}, names), names)
