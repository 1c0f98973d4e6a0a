#!/usr/bin/env python
"""Conditional sampling of prompts and texts of different lengths: one batch with per-sample lengths, against one
B = 1 call per sample, and against the padded batch without lengths (what the masks add).

    python tools/ragged_bench.py [--rounds R]

Workload: Conditioner at the encoders' default dims + the cfg3 denoiser Model(512, depth 12, heads 8, dim_prompt 512)
sampling 10 DDIM steps (captured graphs) at length 1024; B = 16 prompts of 40-103 latent frames and texts of 30-100
phonemes.  The legs alternate in one process; each reports the median over R rounds of CUDA-event time per whole
batch and the library launches of one round.  Prints one JSON line with the card name and its enforced power limit.
"""
import argparse
import json
import statistics
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
sys.path.insert(0, str(Path(__file__).resolve().parent))
from naturalspeech2_pytorch_b200 import Model, NaturalSpeech2, ops  # noqa: E402
from naturalspeech2_pytorch_b200.encoders import Conditioner  # noqa: E402
from train_cond_bench import CFG3, card  # noqa: E402

B, NP, T, LENGTH, TOKENS, STEPS = 16, 103, 100, 1024, 150, 10


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    cn = Conditioner(dim_codebook=128, num_phoneme_tokens=TOKENS)
    with torch.no_grad():   # a few frames per phoneme, so the conditions stay within the 1024-frame latent
        head = cn.duration_pitch.to_duration_pred.to_pred[0]
        head.weight.mul_(0.05)
        head.bias.fill_(4.0)
    cn = cn.to(dev).eval()
    model = Model(**CFG3).to(dev).eval()
    ns = NaturalSpeech2(model, target_sample_hz=24000, timesteps=STEPS, conditioner=cn)
    g = torch.Generator().manual_seed(1)
    plens = torch.linspace(40, NP, B).round().int().tolist()
    tlens = torch.linspace(30, T, B).round().int()[torch.randperm(B, generator=g)].tolist()
    prompt = torch.randn(B, NP, 128, generator=g).to(dev)
    text = torch.randint(0, TOKENS, (B, T), generator=g).to(dev)
    noise = torch.randn(B, LENGTH, 512, generator=g).to(dev)

    legs = {
        "ragged_batch": lambda: ns.sample(length=LENGTH, prompt=prompt, text=text, prompt_lens=plens,
                                          phoneme_lens=tlens, noise=noise),
        "sequential_b1": lambda: [ns.sample(length=LENGTH, prompt=prompt[b:b + 1, :plens[b]],
                                            text=text[b:b + 1, :tlens[b]], noise=noise[b:b + 1]) for b in range(B)],
        "padded_batch": lambda: ns.sample(length=LENGTH, prompt=prompt, text=text, noise=noise),
    }
    times = {k: [] for k in legs}
    launches = {}
    for fn in legs.values():   # warm-up: packing, workspaces, one graph per shape
        fn()
    torch.cuda.synchronize()
    for _ in range(args.rounds):
        for name, fn in legs.items():
            n0 = ops.launch_count()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1))
            launches[name] = ops.launch_count() - n0
    med = {k: statistics.median(v) for k, v in times.items()}
    print(json.dumps({"workload": f"B={B} prompts {min(plens)}-{max(plens)} frames, texts {min(tlens)}-{max(tlens)} "
                                  f"phonemes, length {LENGTH}, {STEPS} DDIM steps, cfg3 denoiser",
                      "median_ms": med, "all_ms": times, "launches_per_call": launches,
                      "speedup_ragged_vs_sequential": med["sequential_b1"] / med["ragged_batch"],
                      "card": card(dev)}))


if __name__ == "__main__":
    main()
