#!/usr/bin/env python
"""Denoiser step time on a batch of latents of different lengths: what skipping each sample's padded tiles saves.

    python tools/latent_lens_bench.py [--rounds R] [--iters I]

Workloads: the cfg2 denoiser Model(512, depth 12, heads 8) unconditional and the conditional cfg3 denoiser (dim_prompt
512, cached conditioning), both at B = 32, N = 1024, one graph-captured forward per step.  Legs, alternated within each
round: (a) no lengths; (b) every length = N (the cost of the length path itself); (c) lengths 256 + 24 b; (d) the sum
of the 32 samples run alone at their own lengths.  Each leg reports the median over R rounds of the CUDA-event time of
I steps, per step.  `tile_share` is the share of 128-row tiles (c) computes; the ratio (c) / (a) is to be compared with
it.  A training step of cfg2 (forward, masked MSE, backward of every parameter) is timed for (a) and (c); training
computes every row (no tile skipping), so the two should take the same time.  Prints one JSON line with the card name
and its enforced power limit.
"""
import argparse
import json
import statistics
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))
from naturalspeech2_pytorch_b200 import Model  # noqa: E402
from train_cond_bench import card  # noqa: E402

CFG2 = dict(dim=512, depth=12, heads=8)
CFG3 = dict(dim=512, depth=12, heads=8, dim_prompt=512, condition_on_prompt=True)
B, N = 32, 1024
MIX = [256 + 24 * b for b in range(B)]


def _time(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def bench(cfg, rounds, iters, dev):
    torch.manual_seed(0)
    model = Model(**cfg).to(dev).eval()
    model.use_cuda_graphs = True
    model.freeze_packed = True
    model.max_cached_shapes = B + 2   # one workspace and graph per alone length: none evicted between rounds
    g = torch.Generator(device=dev).manual_seed(1)
    x = torch.randn(B, N, 512, device=dev, generator=g)
    t = torch.rand(B, device=dev, generator=g)
    kw, alone_kw = {}, [{} for _ in range(B)]
    if cfg.get("condition_on_prompt"):
        prompt = torch.randn(B, 103, 512, device=dev, generator=g)
        cond = torch.randn(B, 512, N, device=dev, generator=g)
        kw = dict(_conditioning=model.precompute_conditioning(prompt, cond, N), cond_drop_prob=0.)
        alone_kw = [dict(_conditioning=model.precompute_conditioning(prompt[b:b + 1], cond[b:b + 1], n), cond_drop_prob=0.)
                    for b, n in enumerate(MIX)]
    full = torch.full((B,), N, dtype=torch.int32, device=dev)
    mix = torch.tensor(MIX, dtype=torch.int32, device=dev)
    out = torch.empty_like(x)
    outs = [torch.empty(1, n, 512, device=dev) for n in MIX]
    legs = {
        "a_no_lengths": lambda: model(x, t, out=out, **kw),
        "b_all_full": lambda: model(x, t, out=out, lengths=full, **kw),
        "c_mixed": lambda: model(x, t, out=out, lengths=mix, **kw),
        "d_sum_alone": lambda: [model(x[b:b + 1, :n], t[b:b + 1], out=outs[b], **alone_kw[b])
                                for b, n in enumerate(MIX)],
    }
    for fn in legs.values():   # warm-up: packing, workspaces, one graph per shape
        fn()
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in legs}
    for _ in range(rounds):
        for name, fn in legs.items():
            times[name].append(_time(fn, iters))
    med = {k: statistics.median(v) for k, v in times.items()}
    tiles = sum(-(-n // 128) for n in MIX) / (B * (N // 128))
    return {"median_ms_per_step": med, "all_ms_per_step": times, "tile_share_c": tiles,
            "ratio_c_over_a": med["c_mixed"] / med["a_no_lengths"],
            "ratio_b_over_a": med["b_all_full"] / med["a_no_lengths"]}


def bench_train(rounds, iters, dev):
    from naturalspeech2_pytorch_b200 import training
    torch.manual_seed(0)
    model = Model(**CFG2).to(dev).train()
    g = torch.Generator(device=dev).manual_seed(1)
    x = torch.randn(B, N, 512, device=dev, generator=g)
    target = torch.randn(B, N, 512, device=dev, generator=g)
    t = torch.rand(B, device=dev, generator=g)
    mix = torch.tensor(MIX, dtype=torch.int32, device=dev)
    params = list(model.parameters())

    def step(lens):
        rows = training.MseRowsFunction.apply(model(x, t, **({} if lens is None else {"lengths": lens})), target, lens)
        torch.autograd.grad(rows.mean(), params, allow_unused=True)
    legs = {"a_no_lengths": lambda: step(None), "c_mixed": lambda: step(mix)}
    for fn in legs.values():
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in legs}
    for _ in range(rounds):
        for name, fn in legs.items():
            times[name].append(_time(fn, iters))
    return {"median_ms_per_step": {k: statistics.median(v) for k, v in times.items()}, "all_ms_per_step": times}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    with torch.no_grad():
        res = {"cfg2": bench(CFG2, args.rounds, args.iters, dev), "cfg3": bench(CFG3, args.rounds, args.iters, dev)}
    res["train_cfg2"] = bench_train(args.rounds, max(1, args.iters // 5), dev)
    print(json.dumps({"workload": f"B={B}, N={N}, lengths 256 + 24 b ({MIX[0]}-{MIX[-1]}), graph-captured forwards",
                      **res, "card": card(dev)}))


if __name__ == "__main__":
    main()
