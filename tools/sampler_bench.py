#!/usr/bin/env python
"""Per-step time of graph-captured DDIM sampling (`NaturalSpeech2.sample`, one CUDA graph per sampling step).

    python tools/sampler_bench.py [--timesteps T] [--rounds R]

Workloads, B = 32 latents of N = 1024 frames: the cfg2 denoiser Model(512, depth 12, heads 8) and the conditional cfg3
denoiser (dim_prompt 512, prompts of 103 frames), each without latent lengths and with lengths 256 + 24 b, at
cond_scale 1 and 3.  cfg2 is unconditional, so its cond_scale 3 runs the same unguided step as 1; cfg3 at 3 runs the
guided step (conditional and null forward, guidance combine).  Each leg is one `sample` call of T steps after a warm-up
call that captures its graph; the legs alternate within each round, and each reports the median over R rounds of the
CUDA-event time per step.  The noise is seeded, so `sha256` (of the last sample's bytes) compares builds output for
output.  Prints one JSON line with the card name and its enforced power limit.
"""
import argparse
import hashlib
import json
import statistics
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))
from naturalspeech2_pytorch_b200 import Model, NaturalSpeech2  # noqa: E402
from train_cond_bench import card  # noqa: E402

CFGS = {"cfg2": dict(dim=512, depth=12, heads=8),
        "cfg3": dict(dim=512, depth=12, heads=8, dim_prompt=512, condition_on_prompt=True)}
B, N, NP = 32, 1024, 103
MIX = [256 + 24 * b for b in range(B)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--timesteps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    res = {}
    for name, cfg in CFGS.items():
        torch.manual_seed(0)
        model = Model(**cfg).to(dev).eval()
        model.freeze_packed = True
        ns = NaturalSpeech2(model, target_sample_hz=24000, timesteps=args.timesteps, cuda_graphs=True)
        g = torch.Generator(device=dev).manual_seed(1)
        noise = torch.randn(B, N, 512, device=dev, generator=g)
        kw = {}
        if cfg.get("condition_on_prompt"):
            kw = dict(prompt_enc=torch.randn(B, NP, 512, device=dev, generator=g),
                      cond=torch.randn(B, 512, N, device=dev, generator=g))
        legs = {f"{name}_{lens}_cs{cs:g}": dict(kw, cond_scale=cs, latent_lens=None if lens == "full" else MIX)
                for lens in ("full", "mixed") for cs in (1., 3.)}
        out = {}
        with torch.no_grad():
            for k, leg in legs.items():   # warm-up: packing, workspace, one captured step per leg
                out[k] = ns.sample(length=N, batch_size=B, noise=noise, **leg)
            torch.cuda.synchronize()
            times = {k: [] for k in legs}
            for _ in range(args.rounds):
                for k, leg in legs.items():
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    out[k] = ns.sample(length=N, batch_size=B, noise=noise, **leg)
                    e1.record()
                    torch.cuda.synchronize()
                    times[k].append(e0.elapsed_time(e1) / args.timesteps)
        for k in legs:
            res[k] = {"ms_per_step": round(statistics.median(times[k]), 4),
                      "all_ms_per_step": [round(t, 4) for t in times[k]],
                      "sha256": hashlib.sha256(out[k].cpu().numpy().tobytes()).hexdigest()}
        del model, ns, out
        torch.cuda.empty_cache()
    print(json.dumps({"workload": f"B={B}, N={N}, {args.timesteps} DDIM steps per sample call, graph-captured steps; "
                                  f"mixed lengths 256 + 24 b ({MIX[0]}-{MIX[-1]})",
                      "legs": res, "card": card(dev)}))


if __name__ == "__main__":
    main()
