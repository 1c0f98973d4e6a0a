"""GPU: the diffusion wrapper (`NaturalSpeech2`) against float64 across the configurations its constructor accepts.

Rows (tests/golden/make_golden_diffusion_configs.DIFFUSION_CONFIGS, on make_golden's uncond_small weights, plus
cond_guided on cond_small): the sigmoid, linear and cosine schedules with their keyword arguments, scale < 1, the
min-SNR weight on and off with gamma 1, 3 and 5, the v / eps / x0 objectives, the RVQ cross-entropy term at weight 0.5,
classifier-free guidance at cond_scale 0, 1 and 3, and 1, 2, 3, 7 and 1000 sampling steps.  Per row:

(a) training loss and d pred.  The model output `pred` is captured inside `forward` and keeps its gradient; the
    reference is float64 autograd of `oracle.diffusion_oracle.diffusion_loss` (and, with the CE term, of
    tests/rvq_ce_restatement.py on the oracle's x_start) on the same audio, noise, times and pred, with the fp32
    alpha / sigma of the reference's formulas.  The batch holds the edge times t = 0, 1e-7, 0.5, 1 - 2^-24 and 1:
    where the same formula in torch fp32 gives inf or NaN ours must give the same non-finite values, and everywhere
    else ours is finite and within the bound.  A non-finite min-SNR weight makes the whole (B,1,B)-broadcast loss
    non-finite, so the batch is also run without the times whose fp32 sigma is 0 and compared the same way.
(b) sampler, step by step.  The eager loop (cuda_graphs=False) is recorded at every step (x_i, v_i); each x_{i+1} is
    checked against the oracle's float64 DDIM step from the same x_i, v_i and the wrapper's fp32 coefficients, which
    are bit-identical to the reference's per-step formulas evaluated on the GPU, and within one ulp of gamma of the
    coefficients the reference built on the CPU (CUDA's fp32 sqrt is correctly rounded where torch's CPU sqrt is not,
    and the two sigmoids differ in the last bit).  The last step lands on sigma_next = 0.
(c) graph path.  `sample()` with CUDA graphs is bit-identical to the eager loop, 1000 steps included, also with
    time_difference = 0.3 (a value the reference never reads in DDIM).  A second configuration swapped into the same
    wrapper reuses the captured graph and still matches its own eager loop: the coefficients come from the per-step
    copy, not from the capture.
(d) the whole 3-step trajectory against the float64 denoiser port (oracle.denoiser_torch_port) inside the oracle's
    sampler: rel-L2 <= C x the rel-L2 of the same trajectory through the port under bf16 autocast + floor, with the
    denoiser family's C and floor of tests/fp64_check.py and no ceiling.
    rel-L2 is relative to the whole sample, i.e. to its spread, which matters for eps: 1/alpha ~ 3e4 at t = 1.

Bound of (a) and (b), the protocol of the RVQ CE suites: max |ours - fp64| <= C x max |torch fp32 - fp64| +
2^-16 max |fp64|.  The DDIM kernel contracts into FMAs, so it is not bitwise equal to torch fp32.

(e) sensitivity: the same bounds reject a min-SNR weight paired per sample instead of the reference's (B,1,B)
broadcast, the previous step's coefficients, `scale` applied to sigma as well, the eps x_start clamped on sigma
instead of alpha, and the cosine schedule with tau ignored.

Measured on an H100 80GB HBM3 (700 W power limit).  Worst ratio of our error to torch fp32's, per row (batch without
sigma = 0; in the edge batch every ratio is <= 1.00, and in sig_x0_off, lin_eps_off and cos_kw_x0 its loss and d pred
are inf / NaN exactly where torch fp32's are):
  (a) loss / d pred        sig_v 1.00 / 0.96, sig_kw_eps 1.00 / 1.00, sig_x0_off 1.00 / 1.00, lin_v_half 1.00 / 1.00,
                           lin_eps_off 0.35 / 2.22 (CE term on), lin_x0_g1 1.00 / 1.00, cos_v 0.85 / 1.00,
                           cos_tau075 0.71 / 0.72 (CE term on, 17 % / 18 % of the bound, edge batch alike), cos_kw_x0
                           1.00 / 1.00, cond_guided 1.00 / 1.00; every other loss and d pred uses <= 3 % of its bound
  (b) DDIM steps           1.00 ... 1.13 at 7 steps, 1.82 (sig_v) and 1.08 (cos_tau075) at 1000; <= 1 % of the bound
hence C = 4.  (d) ours / autocast-bf16 rel-L2 0.52 ... 0.55 (sig_v 3.5e-3 / 6.3e-3, sig_x0_off 5.6e-3 / 1.1e-2,
cond_guided at cond_scale 3 5.2e-3 / 9.8e-3), hence the denoiser's C = 1.  The wrong references of (e) sit at 140 x
(pairing, lin_x0_g1 loss) to 2e6 x their bound.  The whole module takes ~33 s, the sig_v row (1, 2, 7 and 1000 steps,
eager and twice graphed, plus the module's warm-up) ~10 s of it.
"""
import time

import numpy as np
import pytest
import torch

from fp64_check import DENOISER, bound, rel_l2
from golden.make_golden_diffusion_configs import COEF_STEPS, DIFFUSION_CONFIGS, GOLDEN_CONFIGS
from helpers import GOLDEN, build_model, load_model_golden, oracle_config
from oracle import denoiser_torch_port as tp
from oracle import diffusion_oracle as do

pytestmark = pytest.mark.gpu

C = 4.0              # ours / torch-fp32 error ratio allowed in (a) and (b)
FLOOR = 2.0 ** -16

ROWS = dict(DIFFUSION_CONFIGS, cond_guided=dict())
STEPS = {"sig_v": (1, 2, 7, 1000), "cos_tau075": (7, 1000)}
CE_WEIGHT = 0.5
EDGE_TIMES = (0., 1e-7, 0.5, 1 - 2 ** -24, 1., 0.3)
N_LOSS, N_SAMPLE, B_SAMPLE = 32, 32, 2


def _cfg(name):
    kw = ROWS[name]
    return dict(objective=kw.get("objective", "v"), scale=kw.get("scale", 1.),
                schedule=kw.get("noise_schedule", "sigmoid"),
                schedule_kwargs=kw.get("schedule_kwargs"), min_snr_loss_weight=kw.get("min_snr_loss_weight", True),
                min_snr_gamma=kw.get("min_snr_gamma", 5), ce=kw.get("rvq_cross_entropy_loss_weight", 0.))


_MODELS = {}


def _model(case):
    """make_golden's weights, rounded to bf16 in place so that the float64 port sees what the packs hold."""
    if case not in _MODELS:
        z, kwargs, seed = load_model_golden(case)
        m = build_model(kwargs, seed, device="cuda")
        with torch.no_grad():
            for p in m.parameters():
                p.copy_(p.bfloat16().float())
        extra = {}
        if kwargs.get("condition_on_prompt"):
            extra = dict(prompt_enc=torch.from_numpy(z["in_prompt"]).cuda(), cond=torch.from_numpy(z["in_cond"]).cuda())
        _MODELS[case] = (m, kwargs, extra)
    return _MODELS[case]


def _wrapper(name, timesteps, model=None, codec=None, **extra):
    from naturalspeech2_pytorch_b200 import NaturalSpeech2
    m = model if model is not None else _model("cond_small" if name == "cond_guided" else "uncond_small")[0]
    kw = dict(ROWS[name], **extra)
    if codec is None:
        kw.pop("rvq_cross_entropy_loss_weight", None)
        return NaturalSpeech2(m, target_sample_hz=24000, timesteps=timesteps, **kw)
    return NaturalSpeech2(m, codec, timesteps=timesteps, **kw)


def _coefficients(cfg, times, tau=None, scale_sigma=False):
    """The reference's fp32 (alpha, sigma) at `times` (the wrapper's restatement of its formulas); optionally a wrong
    variant: another tau, or sigma scaled too."""
    from naturalspeech2_pytorch_b200 import diffusion
    skw = dict(cfg["schedule_kwargs"] or {})
    if tau is not None:
        skw["tau"] = tau
    sched = {"linear": diffusion.simple_linear_schedule, "cosine": diffusion.cosine_schedule,
             "sigmoid": diffusion.sigmoid_schedule}[cfg["schedule"]]
    a, s = diffusion.gamma_to_alpha_sigma(sched(times, **skw), cfg["scale"])
    return a, (s * cfg["scale"] if scale_sigma else s)


def _bound(err32, ref64):
    return C * err32 + FLOOR * ref64


def _excess(ours, ref64, err32):
    """max |ours - ref64| / bound (> 1 fails)."""
    d = float((ours.double() - ref64).abs().max())
    return d / _bound(err32, float(ref64.abs().max()))


# ---------------------------------------------------------------------------------------------------------------
# (a) training loss and d pred
# ---------------------------------------------------------------------------------------------------------------
def _loss_reference(cfg, pred, audio, noise, alpha, sigma, dtype, codec=None, codes=None, own=None, paired=False):
    """(loss, d pred, own codes) of the oracle's loss in `dtype` by autograd."""
    from rvq_ce_restatement import residual_vq_ce
    p = pred.detach().to(dtype).requires_grad_(True)
    A, X, a, s = audio.to(dtype), noise.to(dtype), alpha.to(dtype), sigma.to(dtype)
    loss, parts = do.diffusion_loss(p, A, X, a, s, cfg["objective"], cfg["min_snr_loss_weight"], cfg["min_snr_gamma"])
    if paired:
        loss = (parts["per_sample"] * parts["weight"]).mean()
    if codec is not None:
        x_start = do.x_start_from_pred(A, p, a, s, cfg["objective"])
        _, ce, own = residual_vq_ce(x_start, codec.codebooks.to(dtype), codes, own=own)
        loss = loss + CE_WEIGHT * ce
    loss.backward()
    return loss.detach(), p.grad, own


def _ours_loss(ns, model, audio, noise, times, extra, codes=None):
    model.train()
    model.zero_grad(set_to_none=True)
    preds = []

    def keep(module, args, out):
        out.retain_grad()
        preds.append(out)

    hook = model.register_forward_hook(keep)
    kw = dict(extra)
    if codes is not None:
        kw["codes"] = codes
    loss = ns(audio, times=times, noise=noise, **kw)
    hook.remove()
    loss.backward()
    model.eval()
    return loss.detach(), preds[0].detach(), preds[0].grad


def _against_fp32(ours, r32, r64):
    """Where torch fp32 gives inf or NaN ours gives the same value; everywhere else ours (and the fp64 reference) is
    finite.  -> (excess of ours over the bound on the finite part, ours / torch-fp32 error ratio there)."""
    ours, r32 = ours.reshape(r32.shape), r32.float()
    fin = torch.isfinite(r32)
    assert torch.equal(torch.isnan(ours), torch.isnan(r32)), "NaN where torch fp32 has none, or none where it has"
    inf = torch.isinf(r32)
    assert torch.equal(ours[inf], r32[inf]), "infinities differ from torch fp32"
    assert bool(torch.isfinite(ours[fin]).all()), "non-finite where torch fp32 is finite"
    assert bool(torch.isfinite(r64[fin]).all()), "fp64 non-finite where torch fp32 is finite"
    if not bool(fin.any()):
        return 0.0, 0.0
    o, a, b = ours[fin].double(), r32[fin].double(), r64[fin]
    err32 = float((a - b).abs().max())
    return _excess(o, b, err32), float((o - b).abs().max()) / max(err32, 1e-300)


def _run_loss(name):
    from golden.make_golden_rvq_ce import rvq_ce_inputs
    from naturalspeech2_pytorch_b200 import EncodecRVQ
    cfg = _cfg(name)
    model, kwargs, extra = _model("cond_small" if name == "cond_guided" else "uncond_small")
    B = len(EDGE_TIMES)
    N = 160 if extra else N_LOSS
    cb, latents, codes = rvq_ce_inputs(B, N, 128)
    if extra:
        extra = {k: v[:1].expand(B, *v.shape[1:]).contiguous() for k, v in extra.items()}
    codec = EncodecRVQ(cb).cuda() if cfg["ce"] else None
    ns = _wrapper(name, 4, model, codec)
    g = torch.Generator().manual_seed(30)
    audio, noise = latents.cuda(), torch.randn(B, N, 128, generator=g).cuda()
    times_all = torch.tensor(EDGE_TIMES, device="cuda")
    out = {}
    alpha_all, sigma_all = _coefficients(cfg, times_all)
    for batch in ("edge", "finite"):
        keep = torch.ones(B, dtype=torch.bool, device="cuda") if batch == "edge" else sigma_all > 0
        idx = keep.nonzero().flatten()
        if batch == "finite" and len(idx) == B and out["edge"]["finite"]:
            out["finite"] = out["edge"]
            continue
        sel = lambda t: t[idx].contiguous()  # noqa: E731
        a, n, t = sel(audio), sel(noise), sel(times_all)
        ex = {k: sel(v) for k, v in extra.items()}
        cd = sel(codes.cuda()) if codec is not None else None
        loss, pred, d_pred = _ours_loss(ns, model, a, n, t, ex, cd)
        alpha, sigma = _coefficients(cfg, t)
        l32, d32, own = _loss_reference(cfg, pred, a, n, alpha, sigma, torch.float32, codec, cd)
        l64, d64, _ = _loss_reference(cfg, pred, a, n, alpha, sigma, torch.float64, codec, cd, own)
        out[batch] = dict(loss=loss, d_pred=d_pred, pred=pred, audio=a, noise=n, times=t, codes=cd, codec=codec,
                          l32=l32, d32=d32, l64=l64, d64=d64, own=own,
                          finite=bool(torch.isfinite(l32)) and bool(torch.isfinite(d32).all()))
    return out


# ---------------------------------------------------------------------------------------------------------------
# (b), (c), (d) sampling
# ---------------------------------------------------------------------------------------------------------------
def _eager_trajectory(ns, noise, cond_scale, extra):
    """Every (x_i, v_i) of the eager loop and the final sample."""
    xs, vs = [], []
    model = ns.model
    real = type(model).forward_with_cond_scale

    def record(x, t, **kw):
        xs.append(x.clone())
        v = real(model, x, t, **kw)
        vs.append(v.clone())
        return v

    model.forward_with_cond_scale = record
    try:
        final = _sample(ns, noise, cond_scale, extra)
    finally:
        del model.forward_with_cond_scale
    return torch.stack(xs + [final]), torch.stack(vs)


def _sample(ns, noise, cond_scale, extra):
    kw = dict(prompt_enc=extra["prompt_enc"], cond=extra["cond"], cond_scale=cond_scale) if extra else {}
    return ns.sample(length=noise.shape[1], batch_size=noise.shape[0], noise=noise, **kw)


def _step_stats(cfg, xs, vs, coef, wrong=None):
    """Per step: (excess of ours over the bound, excess of the wrong reference or None, torch-fp32 error, our error)."""
    out = []
    for i in range(vs.shape[0]):
        c = [coef[i, k] for k in range(4)]
        ref64 = do.ddim_step_coef(xs[i].double(), vs[i].double(), *(v.double() for v in c), objective=cfg["objective"])
        ref32 = do.ddim_step_coef(xs[i], vs[i], *c, objective=cfg["objective"])
        err32 = float((ref32.double() - ref64).abs().max())
        ex = _excess(xs[i + 1], ref64, err32)
        exw = None
        if wrong is not None and wrong(i, xs[i], vs[i], coef) is not None:
            w = wrong(i, xs[i], vs[i], coef)
            exw = _excess(xs[i + 1], w, err32) if torch.isfinite(w).all() else float("inf")
        out.append((ex, exw, err32, float((xs[i + 1].double() - ref64).abs().max())))
    return out


def _port_trajectory(name, model, kwargs, extra, noise, coef, cond_scale, dtype, autocast):
    cfg = _cfg(name)
    P = {n: p.detach().to(dtype) for n, p in model.named_parameters()}
    pc = oracle_config(kwargs)
    x = noise.to(dtype)
    B = x.shape[0]
    T = coef.shape[0]
    times = torch.linspace(1., 0., T + 1, device="cuda")[:-1]
    X = {k: v.to(dtype) for k, v in extra.items()}
    for i in range(T):
        t = times[i].expand(B).to(dtype)
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
            if extra:
                keep = torch.zeros(B, dtype=torch.bool, device="cuda")
                c = tp.model_forward_autograd(P, pc, x, t, X["prompt_enc"], X["cond"], drop_prompt=keep, drop_cond=keep)
                if cond_scale != 1:
                    n = tp.model_forward_autograd(P, pc, x, t, X["prompt_enc"], X["cond"], drop_prompt=~keep,
                                                  drop_cond=~keep)
                    c = n.to(dtype) + cond_scale * (c.to(dtype) - n.to(dtype))
                v = c.to(dtype)
            else:
                v = tp.model_forward_autograd(P, pc, x, t).to(dtype)
        x = do.ddim_step_coef(x, v, *(coef[i, k].to(dtype) for k in range(4)), objective=cfg["objective"])
    return x


def _run_sampling(name):
    from naturalspeech2_pytorch_b200.diffusion import gamma_to_alpha_sigma
    cfg = _cfg(name)
    model, kwargs, extra = _model("cond_small" if name == "cond_guided" else "uncond_small")
    N = 160 if extra else N_SAMPLE
    scales = (0., 1., 3.) if extra else (1.,)
    g = torch.Generator().manual_seed(31)
    noise = torch.randn(B_SAMPLE, N, 128, generator=g).cuda()
    res = {"steps": {}, "graph": {}, "traj": {}}
    for T in STEPS.get(name, (7,)):
        for cs in scales:
            eager = _wrapper(name, T, model, cuda_graphs=False)
            xs, vs = _eager_trajectory(eager, noise, cs, extra)
            times, coef = eager._schedule_tables(B_SAMPLE, "cuda")
            per_step = torch.stack([torch.stack((*gamma_to_alpha_sigma(eager.gamma_schedule(t), eager.scale),
                                                 *gamma_to_alpha_sigma(eager.gamma_schedule(tn), eager.scale)))
                                    for t, tn in eager.get_sampling_timesteps(B_SAMPLE, device="cuda")])
            res["steps"][(T, cs)] = dict(xs=xs, vs=vs, coef=coef, tables_bit_identical=torch.equal(per_step, coef))
            graphed = _wrapper(name, T, model, cuda_graphs=True)
            shifted = _wrapper(name, T, model, cuda_graphs=True, time_difference=0.3)
            res["graph"][(T, cs)] = (torch.equal(_sample(graphed, noise, cs, extra), xs[-1]),
                                     torch.equal(_sample(shifted, noise, cs, extra), xs[-1]))
    for cs in scales:
        ns = _wrapper(name, 3, model, cuda_graphs=True)
        ours = _sample(ns, noise, cs, extra)
        _, coef = ns._schedule_tables(B_SAMPLE, "cuda")
        ref = _port_trajectory(name, model, kwargs, extra, noise, coef, cs, torch.float64, False)
        ac = _port_trajectory(name, model, kwargs, extra, noise, coef, cs, torch.float32, True)
        res["traj"][cs] = (rel_l2(ours, ref), rel_l2(ac, ref))
    return res


_CACHE = {}


def _row(name):
    if name not in _CACHE:
        t0 = time.perf_counter()
        loss = _run_loss(name)
        samp = _run_sampling(name)
        torch.cuda.synchronize()
        _CACHE[name] = dict(loss=loss, samp=samp, seconds=time.perf_counter() - t0)
    return _CACHE[name]


@pytest.mark.parametrize("name", list(ROWS))
def test_loss_and_d_pred_match_fp64(name):
    """Both batches: the edge batch (every edge time) and the batch without the times whose fp32 sigma is 0; the loss
    and d pred of each are finite and within the bound wherever torch fp32 is finite, and equal to its inf / NaN
    elsewhere."""
    r = _row(name)["loss"]
    line = [f"\n{name}:"]
    worst = []
    for batch in ("edge", "finite"):
        f = r[batch]
        el, rl = _against_fp32(f["loss"], f["l32"], f["l64"])
        ed, rd = _against_fp32(f["d_pred"], f["d32"], f["d64"])
        ts = [round(t, 8) for t in f["times"].tolist()]
        line.append(f"{batch} batch (t = {ts}, fp32 loss {float(f['l32']):.6g}): "
                    f"ours / fp32 error loss {rl:.2f} d pred {rd:.2f}, bound use loss {el:.0%} d pred {ed:.0%};")
        worst.append((batch, el, ed))
    print(" ".join(line))
    assert r["finite"]["finite"], name
    bad = [w for w in worst if w[1] > 1 or w[2] > 1]
    assert not bad, (name, bad)


@pytest.mark.parametrize("name", list(ROWS))
def test_sampler_steps_match_fp64(name):
    r = _row(name)
    cfg = _cfg(name)
    for (T, cs), s in r["samp"]["steps"].items():
        assert s["tables_bit_identical"], (name, T, "schedule tables differ from the per-step formulas")
        assert float(s["coef"][-1, 3].abs().max()) == 0.0
        stats = _step_stats(cfg, s["xs"], s["vs"], s["coef"])
        worst = max(st[0] for st in stats)
        ratio = max(st[3] / st[2] for st in stats if st[2] > 0)
        print(f"\n{name} T={T} cond_scale={cs}: worst step at {worst:.0%} of its bound; max ours / torch-fp32 error "
              f"{ratio:.2f}")
        assert worst <= 1, (name, T, cs, [round(st[0], 3) for st in stats][:10])
        if T == 1 and cfg["scale"] == 1.:   # sigma_next = 0, alpha_next = 1: the step returns x_start itself
            from naturalspeech2_pytorch_b200 import ops
            x0 = torch.empty_like(s["xs"][0])
            ops.x_start_from_pred(s["xs"][0], s["vs"][0], s["coef"][0, 0].contiguous(), s["coef"][0, 1].contiguous(),
                                  x0, objective=cfg["objective"])
            assert torch.equal(s["xs"][1], x0), name


@pytest.mark.parametrize("name", list(ROWS))
def test_graph_path_is_bit_identical_to_eager(name):
    r = _row(name)
    for key, (same, shifted) in r["samp"]["graph"].items():
        assert same, (name, key, "graph != eager")
        assert shifted, (name, key, "time_difference changed the sample")


@pytest.mark.parametrize("name", list(ROWS))
def test_trajectory_matches_fp64_port(name):
    r = _row(name)
    for cs, (rel, rel_ac) in r["samp"]["traj"].items():
        print(f"{name} cond_scale={cs}: 3-step trajectory rel-L2 ours {rel:.3e} / autocast-bf16 {rel_ac:.3e}; "
              f"row took {r['seconds']:.1f} s")
        assert rel <= bound(DENOISER.without_ceiling(), rel_ac), (name, cs, rel, rel_ac)


@pytest.mark.parametrize("name", GOLDEN_CONFIGS)
def test_gpu_schedule_tables_match_reference_coefficients(name):
    """`_schedule_tables` on the GPU against the coefficients the reference's own ddim_sample built on the CPU
    (tests/golden/diffusion_configs.npz).  The devices round differently, as the reference itself does when it runs on
    either: CUDA's fp32 sqrt is correctly rounded and torch's CPU sqrt is not on a few values (6 of the 1001 of the
    linear schedule at T = 1000), and the two sigmoids differ in the last bit (on ~500 of the 1000 sigmoid steps).
    So: every coefficient within one ulp of gamma of the reference's; the times equal the CPU's linspace; the linear
    coefficients equal the correctly rounded value of their formula bit for bit, so they differ from the reference's
    only where its CPU sqrt is not."""
    z = np.load(GOLDEN / "diffusion_configs.npz")
    kw = DIFFUSION_CONFIGS[name]
    for T in COEF_STEPS:
        ref = torch.from_numpy(z[f"{name}::coef{T}"]).cuda()
        times, coef = _wrapper(name, T, _model("uncond_small")[0])._schedule_tables(B_SAMPLE, "cuda")
        t_all = torch.cat((times[:, 0], times.new_zeros(1)))
        assert torch.equal(t_all.cpu(), torch.linspace(1., 0., T + 1)), (name, T)
        expected = None
        if kw.get("noise_schedule") == "linear":
            g = (1 - t_all).clamp(min=(kw.get("schedule_kwargs") or {}).get("clip_min", 1e-9))
            rn_sqrt = lambda x: x.double().sqrt().float()  # noqa: E731  (the fp32 square root, correctly rounded)
            a, sg = rn_sqrt(g) * kw.get("scale", 1.), rn_sqrt(1 - g)
            expected = torch.stack((a[:-1], sg[:-1], a[1:], sg[1:]), dim=1)
        for b in range(B_SAMPLE):
            c = coef[:, :, b]
            note = "" if expected is None else \
                f", {int((ref != expected).any(1).sum())} where its sqrt is not correctly rounded"
            print(f"{name} T={T}: {int((c != ref).any(1).sum())} of {T} steps differ from the reference's CPU "
                  f"coefficients{note}")
            assert bool(((c ** 2 - ref ** 2).abs() <= 2 ** -21).all()), (name, T)   # alpha^2, sigma^2: gamma
            if expected is not None:
                assert torch.equal(c, expected), (name, T)


def test_second_configuration_reuses_the_model_cached_graph():
    """Swap another schedule and scale (same objective and shape) into a wrapper whose graph is captured: the
    graph in the model's cache is reused and the sample equals the eager loop of that configuration."""
    model = _model("uncond_small")[0]
    model._graphs.clear()   # the module's models are shared: count this test's captures only
    noise = torch.randn(B_SAMPLE, N_SAMPLE, 128, generator=torch.Generator().manual_seed(32)).cuda()
    ns = _wrapper("sig_v", 7, model, cuda_graphs=True)
    first = _sample(ns, noise, 1., {})
    assert torch.equal(first, _sample(_wrapper("sig_v", 7, model, cuda_graphs=False), noise, 1., {}))
    for other in ("lin_v_half", "cos_v"):
        o = _wrapper(other, 7, model, cuda_graphs=False)
        ns.gamma_schedule, ns.scale = o.gamma_schedule, o.scale
        got = _sample(ns, noise, 1., {})
        assert len(model._graphs) == 1
        assert torch.equal(got, _sample(o, noise, 1., {})), other
        assert not torch.equal(got, first), other


# ---------------------------------------------------------------------------------------------------------------
# (e) sensitivity
# ---------------------------------------------------------------------------------------------------------------
def test_rejects_min_snr_weight_paired_per_sample():
    for name in ("sig_v", "lin_x0_g1"):
        f = _row(name)["loss"]["finite"]
        cfg = _cfg(name)
        alpha, sigma = _coefficients(cfg, f["times"])
        w64, dw64, _ = _loss_reference(cfg, f["pred"], f["audio"], f["noise"], alpha, sigma, torch.float64,
                                       f["codec"], f["codes"], f["own"], paired=True)
        el = _excess(f["loss"].reshape(1), w64.reshape(1), float((f["l32"].double() - f["l64"]).abs()))
        ed = _excess(f["d_pred"], dw64, float((f["d32"].double() - f["d64"]).abs().max()))
        print(f"{name}: per-sample pairing at {el:.3g} x (loss) and {ed:.3g} x (d pred) the bound")
        assert el > 1 and ed > 1, (name, el, ed)


def _assert_steps_reject(name, wrong, T=7, what=""):
    cfg = _cfg(name)
    s = _row(name)["samp"]["steps"][(T, 1.)]
    stats = _step_stats(cfg, s["xs"], s["vs"], s["coef"], wrong)
    rej = [st[1] for st in stats if st[1] is not None]
    print(f"{name} {what}: the wrong reference sits at {min(rej):.3g} ... {max(rej):.3g} x the bound")
    assert rej and min(rej) > 1, (name, what, rej)


def test_rejects_previous_step_coefficients():
    def wrong(i, x, v, coef):
        if i == 0:
            return None
        return do.ddim_step_coef(x.double(), v.double(), *(coef[i - 1, k].double() for k in range(4)), objective="v")
    _assert_steps_reject("sig_v", wrong, what="previous step's coefficients")


def test_rejects_scale_applied_to_sigma():
    cfg = _cfg("lin_v_half")

    def wrong(i, x, v, coef):
        c = [coef[i, k].double() for k in range(4)]
        return do.ddim_step_coef(x.double(), v.double(), c[0], c[1] * cfg["scale"], c[2], c[3] * cfg["scale"],
                                 objective="v")
    _assert_steps_reject("lin_v_half", wrong, what="scale on sigma")
    f = _row("lin_v_half")["loss"]["finite"]
    alpha, sigma = _coefficients(cfg, f["times"], scale_sigma=True)
    w64, dw64, _ = _loss_reference(cfg, f["pred"], f["audio"], f["noise"], alpha, sigma, torch.float64)
    el = _excess(f["loss"].reshape(1), w64.reshape(1), float((f["l32"].double() - f["l64"]).abs()))
    ed = _excess(f["d_pred"], dw64, float((f["d32"].double() - f["d64"]).abs().max()))
    print(f"lin_v_half scale on sigma: loss at {el:.3g} x and d pred at {ed:.3g} x the bound")
    assert el > 1 and ed > 1, (el, ed)


def test_rejects_eps_x_start_clamped_on_sigma():
    def wrong(i, x, v, coef):
        a, s, an, sn = (coef[i, k].double()[:, None, None] for k in range(4))
        x, v = x.double(), v.double()
        x0 = (x - s * v) / s.clamp(min=1e-10)
        eps = (x - a * x0) / s.clamp(min=1e-10)
        return x0 * an + eps * sn
    _assert_steps_reject("sig_kw_eps", wrong, what="x_start / sigma")


def test_rejects_cosine_without_tau():
    name = "cos_tau075"
    cfg = _cfg(name)
    t_all = torch.linspace(1., 0., 8, device="cuda")
    a, sg = _coefficients(cfg, t_all, tau=1)
    bad = torch.stack((a[:-1], sg[:-1], a[1:], sg[1:]), dim=1)[:, :, None].expand(-1, -1, B_SAMPLE)

    def wrong(i, x, v, coef):
        return do.ddim_step_coef(x.double(), v.double(), *(bad[i, k].double() for k in range(4)), objective="eps")
    _assert_steps_reject(name, wrong, what="tau ignored")
    f = _row(name)["loss"]["finite"]
    alpha, sigma = _coefficients(cfg, f["times"], tau=1)
    w64, _, _ = _loss_reference(cfg, f["pred"], f["audio"], f["noise"], alpha, sigma, torch.float64, f["codec"],
                                f["codes"], f["own"])
    assert _excess(f["loss"].reshape(1), w64.reshape(1), float((f["l32"].double() - f["l64"]).abs())) > 1
