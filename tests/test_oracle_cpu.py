"""CPU: the oracle (oracle/*.py) against every golden vector generated from the reference."""
import numpy as np
import pytest
import torch

from helpers import (BIG_MODEL_CASES, MODEL_CASES, GOLDEN, build_model, err_stats, golden_inputs, golden_rows,
                     load_model_golden, numpy_params, oracle_config)
from oracle import denoiser_oracle, diffusion_oracle, rvq_oracle
from param_fill import rvq_fixture_inputs


@pytest.mark.parametrize("name", MODEL_CASES)
def test_denoiser_oracle_matches_reference_fp64(name):
    z, kwargs, seed = load_model_golden(name)
    if name == "readme_uncond":
        pytest.skip("covered by the fp32 run below (kept out of the fp64 run for CPU time)")
    model = build_model(kwargs, seed)
    P = numpy_params(model)
    cfg = oracle_config(kwargs)
    extra = {}
    if kwargs.get("condition_on_prompt"):
        extra = dict(prompt=z["in_prompt"], cond=z["in_cond"])
    out = denoiser_oracle.model_forward(P, cfg, z["in_x"], z["in_times"], dtype=np.float64, **extra)
    emax, _ = err_stats(out, z["out_fp64"])
    # fp64 vs fp64 on fp32-born weights: only summation-order noise is allowed
    assert emax < 1e-9, f"oracle deviates from the reference fp64 output: {emax}"
    if kwargs.get("condition_on_prompt"):
        B = z["in_x"].shape[0]
        ones = np.ones(B, dtype=bool)
        null = denoiser_oracle.model_forward(P, cfg, z["in_x"], z["in_times"], dtype=np.float64,
                                             drop_prompt=ones, drop_cond=ones, **extra)
        assert err_stats(null, z["out_fp64_null"])[0] < 1e-9
        cfg3 = null + (out - null) * 3.0  # forward_with_cond_scale, ns2.py:927
        assert err_stats(cfg3, z["out_fp64_cfg3"])[0] < 1e-8


def test_denoiser_oracle_fp32_readme_config():
    z, kwargs, seed = load_model_golden("readme_uncond")
    model = build_model(kwargs, seed)
    out = denoiser_oracle.model_forward(numpy_params(model), oracle_config(kwargs), z["in_x"], z["in_times"],
                                        dtype=np.float32)
    emax, _ = err_stats(out, z["out_fp64"])
    ref32, _ = err_stats(z["out_fp32"], z["out_fp64"])
    assert emax < 5e-5, (emax, ref32)


def test_state_dict_keys_match_reference_fixture():
    """Appendix B of SURVEY.md: key names / shapes of the conditional model."""
    from naturalspeech2_pytorch_b200 import Model
    m = Model(dim=512, depth=1, dim_prompt=512, condition_on_prompt=True)
    sd = m.state_dict()
    expect = {
        "null_prompt_cond": (2048,), "null_prompt_tokens": (32, 512), "null_cond": (512, 1),
        "to_time_cond.0.weights": (256,), "to_time_cond.1.weight": (2048, 513),
        "to_prompt_cond.1.weight": (2048, 512), "perceiver_resampler.latents": (32, 512),
        "perceiver_resampler.layers.0.0.to_kv.weight": (1024, 512),
        "perceiver_resampler.layers.1.1.0.weight": (2730, 512),
        "perceiver_resampler.layers.1.1.2.weight": (512, 1365),
        "perceiver_resampler.norm.gamma": (512,), "cond_to_model_dim.weight": (512, 512, 1),
        "wavenet.init_conv.weight": (512, 512, 3),
        "wavenet.stacks.0.blocks.7.to_time_cond.weight": (1024, 4096),
        "wavenet.stacks.3.blocks.0.skip_conv.weight": (512, 512, 1),
        "wavenet.final_conv.bias": (512,),
        "transformer.layers.0.0.to_gamma_beta.weight": (1024, 4096),
        "transformer.layers.0.1.to_q.weight": (512, 512),
        "transformer.layers.0.3.to_kv.weight": (1024, 512),
        "transformer.layers.0.5.0.weight": (2730, 512),
        "transformer.layers.0.5.2.1.weight": (1365, 1365, 3),
        "transformer.layers.0.5.3.weight": (512, 1365),
        "transformer.to_pred.0.gamma": (512,), "transformer.to_pred.1.weight": (512, 512),
    }
    for k, shp in expect.items():
        assert k in sd, k
        assert tuple(sd[k].shape) == shp, (k, tuple(sd[k].shape), shp)
    assert "wavenet.stacks.0.blocks.0.skip_conv.weight" not in sd
    assert sum(p.numel() for p in Model(dim=512, depth=12, heads=8).parameters()) == 260_425_464


def test_diffusion_oracle_matches_reference():
    z = np.load(GOLDEN / "diffusion_uncond_small.npz")
    _, kwargs, seed = load_model_golden("uncond_small")
    P = numpy_params(build_model(kwargs, seed))
    cfg = oracle_config(kwargs)

    def model_fn(x, t):
        return denoiser_oracle.model_forward(P, cfg, x, t, dtype=np.float64)

    loss, _ = diffusion_oracle.training_loss(model_fn, z["latents"].astype(np.float64),
                                             z["times"].astype(np.float64), z["noise"].astype(np.float64))
    assert abs(loss - float(z["loss"])) < 2e-5 * max(1.0, abs(float(z["loss"]))), (loss, float(z["loss"]))
    out = diffusion_oracle.ddim_sample(model_fn, z["ddim_init"].astype(np.float64), int(z["timesteps"]))
    emax, _ = err_stats(out, z["ddim_out"])
    assert emax < 2e-4, emax  # the reference ran this in fp32
    # the eps / x0 parameterisations (ns2.py:1637-1663, 1412-1421)
    for obj in ("eps", "x0"):
        loss, _ = diffusion_oracle.training_loss(model_fn, z["latents"].astype(np.float64),
                                                 z["times"].astype(np.float64), z["noise"].astype(np.float64),
                                                 objective=obj)
        ref = float(z[f"loss_{obj}"])
        assert abs(loss - ref) < 2e-5 * max(1.0, abs(ref)), (obj, loss, ref)
        out = diffusion_oracle.ddim_sample(model_fn, z["ddim_init"].astype(np.float64), int(z["timesteps"]),
                                           objective=obj)
        emax, _ = err_stats(out, z[f"ddim_out_{obj}"])
        assert emax < 2e-4 * max(1.0, float(np.abs(z[f"ddim_out_{obj}"]).max())), (obj, emax)


def test_rvq_oracle_matches_encodec_port():
    z = np.load(GOLDEN / "rvq_encodec.npz")
    cb, variants = rvq_fixture_inputs()
    cbn = cb.numpy()
    for name, frames in variants.items():
        codes, gaps = rvq_oracle.encode(frames.numpy(), cbn, return_gaps=True)
        ref = z[f"codes_{name}"]
        mism = codes != ref
        # a first mismatch in a row makes every later stage of that row incomparable
        first = mism & (np.cumsum(mism, axis=1) == 1)
        # disagreement is only legitimate where fp32 rounding decides (relative top-2 gap ~1e-6) or on the
        # duplicated codeword (gap exactly 0, where the fp32 formula may pick either copy)
        assert np.all(gaps[first] < 1e-5), (name, int(first.sum()), gaps[first])
        # bit-exact on all 2 x 2048 x 8 fixture codes (incl. the duplicated codeword -> lowest index)
        assert first.sum() == 0, (name, int(first.sum()))
        ff = rvq_oracle.encode_fp32_formula(frames.numpy(), cbn)
        assert (ff != ref).any(axis=1).sum() == 0
    dec = rvq_oracle.decode(z["codes_random"], cbn)
    np.testing.assert_array_equal(dec, z["decoded_random"])
    # duplicate codeword: the oracle must return the lower index
    assert (rvq_oracle.encode(cbn[0, 7][None], cbn)[0, 0]) == 3


@pytest.mark.parametrize("name", ["uncond_small", "cond_small", "cond_samedim"])
def test_torch_port_matches_reference(name):
    """The torch-CPU port used for bench.py's reference arm reproduces the reference fp32/fp64 outputs."""
    from oracle import denoiser_torch_port as tp
    z, kwargs, seed = load_model_golden(name)
    model = build_model(kwargs, seed)
    P = {k: v.detach().double() for k, v in model.state_dict().items()}
    cfg = oracle_config(kwargs)
    extra = {}
    if kwargs.get("condition_on_prompt"):
        extra = dict(prompt=torch.from_numpy(z["in_prompt"]).double(), cond=torch.from_numpy(z["in_cond"]).double())
    out = tp.model_forward(P, cfg, torch.from_numpy(z["in_x"]).double(), torch.from_numpy(z["in_times"]).double(), **extra)
    assert err_stats(out.numpy(), z["out_fp64"])[0] < 1e-9


@pytest.mark.parametrize("case", ["uncond_small", "cond_small"])
def test_torch_port_autograd_matches_reference_gradients(case):
    """`model_forward_autograd` in float64 is the reference of the GPU backward tests at the benchmarked dims
    (tests/test_denoiser_backward_fp64_gpu.py): its autograd through the diffusion loss of make_golden.gradient_goldens
    (sigmoid schedule, v target, min-SNR-5 weight) reproduces the reference's fp64 gradients — every parameter's norm
    and every stored whole tensor."""
    from naturalspeech2_pytorch_b200.diffusion import gamma_to_alpha_sigma, sigmoid_schedule
    from oracle import denoiser_torch_port as tp
    zd = np.load(GOLDEN / "diffusion_uncond_small.npz")
    gz = np.load(GOLDEN / f"grads_{case}.npz")
    zm, kwargs, seed = load_model_golden(case)
    model = build_model(kwargs, seed)
    P = {k: v.detach().double().requires_grad_(True) for k, v in model.named_parameters()}
    latents, times, noise = (torch.from_numpy(zd[k]).double() for k in ("latents", "times", "noise"))
    extra = {}
    if kwargs.get("condition_on_prompt"):
        extra = dict(prompt=torch.from_numpy(zm["in_prompt"]).double(), cond=torch.from_numpy(zm["in_cond"]).double())
    gamma = sigmoid_schedule(times)
    alpha, sigma = gamma_to_alpha_sigma(gamma[:, None, None], 1.)
    pred = tp.model_forward_autograd(P, oracle_config(kwargs), alpha * latents + sigma * noise, times, **extra)
    per_sample = ((pred - (alpha * noise - sigma * latents)) ** 2).reshape(pred.shape[0], -1).mean(dim=1)
    snr = (alpha * alpha) / (sigma * sigma)
    loss = (per_sample * (snr.clamp(max=5) / (snr + 1))).mean()   # the golden's broadcast, as make_golden.py writes it
    assert abs(loss.item() - float(gz["loss"])) < 1e-9 * abs(float(gz["loss"]))
    loss.backward()
    names = [str(n) for n in gz["names"]]
    assert set(names) == set(P)
    for n, ref_norm in zip(names, gz["norms"]):
        g = P[n].grad if P[n].grad is not None else torch.zeros_like(P[n])
        assert abs(float(g.norm()) - float(ref_norm)) <= 1e-9 * max(float(ref_norm), 1e-6), (n, float(g.norm()), ref_norm)
    stored = [k for k in gz.files if k.startswith("grad::")]
    assert len(stored) == 13
    for key in stored:
        n = key[len("grad::"):]
        ref = torch.from_numpy(gz[key]).double()   # stored as float32
        assert float((P[n].grad - ref).abs().max()) <= 2 ** -23 * float(ref.abs().max()), n


@pytest.mark.parametrize("name", BIG_MODEL_CASES)
def test_torch_port_matches_reference_at_benchmarked_dims(name):
    """The port that bench.py uses as the in-run parity checker / CPU arm, pinned at dim 512 / heads 8 / seq 1024
    (fp32 run vs the reference's fp64 output on the stored row subsample; the reference's own fp32 run sits at
    ~4e-6 from its fp64 run, recorded in the fixture)."""
    from oracle import denoiser_torch_port as tp
    z, kwargs, seed = load_model_golden(name)
    model = build_model(kwargs, seed)
    P = {k: v.detach().float() for k, v in model.state_dict().items()}
    inp = golden_inputs(z, kwargs)
    extra = {k: inp[k] for k in ("prompt", "cond") if k in inp}
    out = tp.model_forward(P, oracle_config(kwargs), inp["x"], inp["times"], **extra)
    emax, _ = err_stats(golden_rows(z, out.numpy()), z["out_fp64"])
    ref32 = float(z["stats_out_fp32"][0])
    assert emax < 5 * ref32 + 1e-6, (emax, ref32)


def test_aligner_oracle_matches_reference_goldens():
    """oracle.aligner_oracle.maximum_path == the reference's maximum_path (aligner.py:88-122) on every fixture,
    bit for bit (0/1 path)."""
    from helpers import aligner_golden_cases
    from oracle import aligner_oracle
    n = 0
    for name, value, mask, ref_path in aligner_golden_cases():
        path, idx = aligner_oracle.maximum_path(value, mask, return_index=True)
        np.testing.assert_array_equal(path, ref_path.astype(np.float32), err_msg=name)
        b, t_x, t_y = value.shape
        onehot = (np.arange(t_x)[None, :, None] == idx[:, None, :]).astype(np.float32) * mask
        np.testing.assert_array_equal(onehot, path, err_msg=name)
        n += 1
    assert n >= 6
