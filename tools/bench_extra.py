#!/usr/bin/env python
"""Secondary measurements of SURVEY 8(d) that bench.py (cfg2 only) does not print: the RVQ microbench (config 4),
the RVQ cross-entropy head forward / backward and its share of a training step (`rvq_ce`), the conditional denoiser
(config 3), the README model (config 1) and the DDIM sampling loop.  One JSON line each,
also appended to gpurun_out/bench_extra.jsonl.  CUDA-event timing, >= 3 warm-ups, inputs resident in HBM."""
from __future__ import annotations

import json
import os
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from naturalspeech2_pytorch_b200 import EncodecRVQ, Model, NaturalSpeech2, ops  # noqa: E402

PEAKS = json.loads((ROOT / "MEASURED_PEAKS.json").read_text()) if (ROOT / "MEASURED_PEAKS.json").exists() else \
    {"bf16_tflops": 1590.0, "bf16_tflops_sustained": 1400.0, "hbm_gbs": 6650.0}
OUT = ROOT / "gpurun_out" / "bench_extra.jsonl"
OUT.parent.mkdir(exist_ok=True)


def emit(d):
    line = json.dumps(d)
    print(line, flush=True)
    with open(OUT, "a") as f:
        f.write(line + "\n")


def time_ms(fn, reps, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def rvq():
    from oracle import rvq_oracle
    torch.manual_seed(1234)
    cb = torch.randn(8, 1024, 128, device="cuda")
    prep = ops.rvq_prepare(cb)
    F = 1 << 20
    for variant in ("random", "realistic"):
        torch.manual_seed(1235)
        if variant == "random":
            x = torch.randn(F, 128, device="cuda")
        else:
            idx = torch.randint(0, 1024, (F, 8), device="cuda")
            x = sum(cb[q][idx[:, q]] * (0.5 ** q) for q in range(8)) + 0.05 * torch.randn(F, 128, device="cuda")
        codes = torch.empty(F, 8, device="cuda", dtype=torch.int64)
        stats = torch.zeros(4, device="cuda", dtype=torch.int64)
        ops.rvq_encode(x, cb, prep, codes=codes, stats=stats)
        ms = time_ms(lambda: ops.rvq_encode(x, cb, prep, codes=codes), reps=5)
        ms_dec = time_ms(lambda: ops.rvq_decode(codes, cb), reps=5)
        flops = 2.0 * F * 8 * 1024 * 128
        emit({"bench": "rvq_encode", "variant": variant, "frames": F, "quantizers": 8, "codebook": 1024, "dim": 128,
              "ms": round(ms, 3), "mcodes_per_s": round(F * 8 / ms / 1e3, 1),
              "tensor_tflops": round(flops / ms / 1e9, 1),
              "frac_of_burst_bf16_peak": round(flops / ms / 1e9 / PEAKS["bf16_tflops"], 4),
              "near_ties_rescored_frac": round(float(stats[1]) / float(stats[0]), 4),
              "full_scans": int(stats[2]), "block_scans": int(stats[3]),
              "decode_ms": round(ms_dec, 3),
              "decode_gbs": round((F * 8 * 8 + F * 128 * 4) / ms_dec / 1e6, 1)})
    # CPU baseline: the reference's fp32 formula (numpy port) on a bounded sample
    n = 32768
    xs = torch.randn(n, 128).numpy()
    cbn = cb.cpu().numpy()
    t0 = time.perf_counter()
    rvq_oracle.encode_fp32_formula(xs, cbn)
    dt = time.perf_counter() - t0
    emit({"bench": "rvq_encode_cpu_baseline", "kind": "port", "frames": n, "seconds": round(dt, 3),
          "mcodes_per_s": round(n * 8 / dt / 1e6, 4), "cores": os.cpu_count()})


def card():
    import subprocess
    out = {"name": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=10)
        out["power_limit_w"] = float(r.stdout.strip().splitlines()[0])
    except Exception as e:
        out["power_limit_w"] = None
        out["power_limit_error"] = f"{type(e).__name__}: {e}"
    return out


FP32_DATASHEET_TFLOPS = 67.0   # H100 SXM5 FP32 (non-tensor) data-sheet peak


def rvq_ce(reps=10, train_steps=6):
    """The RVQ cross-entropy head (ns2.py:1682) at the configs[4] shape (32 x 1024 frames, Q = 8, K = 1024, D = 128):
    forward, and forward + backward, with achieved FP32 FLOP/s (one distance pass = 2 F Q K D FLOP; the backward makes a
    second pass of the same size for sum_k p_k c_k).  Then the training step with the CE weight 0 and 0.5, alternated.
    The CE term needs the denoiser's width to equal the codec's (ns2.py:1244), so that step is configs[4]'s conditional
    denoiser (depth 12, heads 8, dim_prompt 512, B = 32, N = 1024) at dim = 128."""
    Fr, Q, K, D = 32 * 1024, 8, 1024, 128
    torch.manual_seed(7)
    cb = torch.randn(Q, K, D, device="cuda")
    codec = EncodecRVQ(cb).cuda()
    x = torch.randn(Fr, D, device="cuda")
    codes, _ = codec.quantize(torch.randn(Fr, D, device="cuda"))
    prep = codec._prep()
    own = ops.rvq_encode(x, cb, prep)
    d_loss = torch.ones(1, device="cuda")
    fwd = lambda: ops.rvq_ce(x, cb, prep[1], own, codes)
    fwd_bwd = lambda: (ops.rvq_ce(x, cb, prep[1], own, codes), ops.rvq_ce_bwd(x, cb, prep[1], own, codes, d_loss))
    ms_f = time_ms(fwd, reps)
    ms_fb = time_ms(fwd_bwd, reps)
    pass_flop = 2.0 * Fr * Q * K * D
    emit({"bench": "rvq_ce_head", "frames": Fr, "quantizers": Q, "codebook": K, "dim": D,
          "fwd_ms": round(ms_f, 3), "fwd_tflops_fp32": round(pass_flop / ms_f / 1e9, 2),
          "fwd_bwd_ms": round(ms_fb, 3), "fwd_bwd_tflops_fp32": round(3 * pass_flop / ms_fb / 1e9, 2),
          "bwd_ms": round(ms_fb - ms_f, 3), "fp32_datasheet_tflops": FP32_DATASHEET_TFLOPS,
          "fwd_bwd_frac_of_fp32_datasheet": round(3 * pass_flop / ms_fb / 1e9 / FP32_DATASHEET_TFLOPS, 3),
          "card": card()})
    # training step, CE weight 0 and 0.5 alternated in the same call
    model = Model(dim=128, depth=12, heads=8, dim_prompt=512, condition_on_prompt=True).cuda().train()
    g = torch.Generator().manual_seed(200)
    lat = torch.randn(32, 1024, 128, generator=g).cuda()
    lat_codes, lat_q = codec.quantize(lat)
    prompt_enc = torch.randn(32, 103, 512, generator=g).cuda()
    cond = torch.randn(32, 512, 1024, generator=g).cuda()
    opt = torch.optim.AdamW(model.parameters(), lr=1e-4, fused=True)
    nets = {w: NaturalSpeech2(model, codec, rvq_cross_entropy_loss_weight=w) for w in (0., 0.5)}

    def step(w):
        opt.zero_grad(set_to_none=True)
        nets[w](lat_q, codes=lat_codes, prompt_enc=prompt_enc, cond=cond).backward()
        opt.step()

    for w in (0., 0.5, 0., 0.5):
        step(w)
    ms = {0.: [], 0.5: []}
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for i in range(2 * train_steps):
        w = (0., 0.5)[i % 2]
        torch.cuda.synchronize()
        a.record()
        step(w)
        b.record()
        torch.cuda.synchronize()
        ms[w].append(a.elapsed_time(b))
    med = {w: sorted(v)[len(v) // 2] for w, v in ms.items()}
    emit({"bench": "train_step_rvq_ce", "model": "configs[4] conditional denoiser at dim 128", "batch": 32, "seq": 1024,
          "ms_weight0": round(med[0.], 3), "ms_weight05": round(med[0.5], 3),
          "ce_share_of_step": round(1 - med[0.] / med[0.5], 4), "steps_each": train_steps, "card": card()})


def denoiser_cfg(name, kwargs, B, N, flops_per_sample, cond=False, reps=20):
    torch.manual_seed(0)
    model = Model(**kwargs).cuda().eval()
    model.packed()
    model.freeze_packed = True
    x = torch.randn(B, N, kwargs["dim"], device="cuda")
    t = torch.rand(B, device="cuda")
    if not cond:
        ms = time_ms(lambda: model(x, t), reps)
        model.use_cuda_graphs = True
        ms_g = time_ms(lambda: model(x, t), reps)
        emit({"bench": name, "batch": B, "seq": N, "ms_per_step_eager": round(ms, 4),
              "ms_per_step_cuda_graph": round(ms_g, 4), "steps_per_s": round(1e3 / ms_g, 2),
              "tflops": round(flops_per_sample * B / ms_g / 1e9, 1)})
        return
    prompt = torch.randn(B, 103, kwargs["dim_prompt"], device="cuda")
    cnd = torch.randn(B, kwargs["dim_prompt"], N, device="cuda")
    ms_full = time_ms(lambda: model(x, t, prompt=prompt, cond=cnd), reps)
    cached = model.precompute_conditioning(prompt, cnd, N)
    ms_cached = time_ms(lambda: model(x, t, _conditioning=cached), reps)
    emit({"bench": name, "batch": B, "seq": N, "prompt_frames": 103,
          "ms_per_step_full": round(ms_full, 4), "steps_per_s_full": round(1e3 / ms_full, 2),
          "ms_per_step_cached_conditioning": round(ms_cached, 4), "steps_per_s_cached": round(1e3 / ms_cached, 2),
          "tflops_cached": round(flops_per_sample * B / ms_cached / 1e9, 1)})


def ddim():
    torch.manual_seed(0)
    model = Model(dim=512, depth=12, heads=8).cuda().eval()
    model.packed()
    model.freeze_packed = True
    ns = NaturalSpeech2(model, target_sample_hz=24000, timesteps=20)
    ns.sample(length=1024, batch_size=32)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ns.sample(length=1024, batch_size=32)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    emit({"bench": "ddim_sample_cfg2", "batch": 32, "seq": 1024, "timesteps": 20, "seconds": round(dt, 4),
          "denoiser_steps_per_s": round(20 / dt, 2), "note": "public API NaturalSpeech2.sample, wall clock incl. host loop"})


if __name__ == "__main__":
    which = set(sys.argv[1:]) or {"rvq", "rvq_ce", "cfg1", "cfg3", "ddim"}
    if "rvq" in which:
        rvq()
    if "rvq_ce" in which:
        rvq_ce()
    if "cfg1" in which:
        denoiser_cfg("denoiser_cfg1_readme", dict(dim=128, depth=6), 4, 1024, 26.74e9)
    if "cfg3" in which:
        denoiser_cfg("denoiser_cfg3_conditional", dict(dim=512, depth=12, dim_prompt=512, condition_on_prompt=True), 16,
                     1024, 331.97e9, cond=True)
    if "ddim" in which:
        ddim()
