#!/usr/bin/env python
"""Conditional training on prompts and texts of different lengths: one batch with per-sample lengths, against 16
accumulated B = 1 steps, and against the padded batch without lengths (what the masks add).

    python tools/ragged_train_bench.py [--rounds R]

Workload: one conditional training step (NaturalSpeech2.forward + loss.backward, gradients into the denoiser, both
encoders and the pitch embedding; no optimizer step) with the Conditioner at the encoders' default dims and the cfg3
denoiser Model(512, depth 12, heads 8, dim_prompt 512) on 1024 latent frames shared by the batch; B = 16 prompts of
40-103 latent frames and texts of 30-100 phonemes, durations summing to <= 1024 frames.  The legs alternate in one
process; each reports the median over R rounds of CUDA-event time per whole batch and the library launches of one
round.  Prints one JSON line with the card name and its enforced power limit.
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

B, NP, T, SEQ, TOKENS = 16, 103, 100, 1024, 150


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    cn = Conditioner(dim_codebook=128, num_phoneme_tokens=TOKENS).to(dev).train()
    model = Model(**CFG3).to(dev).train()
    ns = NaturalSpeech2(model, target_sample_hz=24000, conditioner=cn)
    trained = [*model.parameters(), *cn.prompt_enc.parameters(), *cn.phoneme_enc.parameters(),
               *cn.pitch_emb.parameters()]
    g = torch.Generator().manual_seed(1)
    plens = torch.linspace(40, NP, B).round().int().tolist()
    tlens = torch.linspace(30, T, B).round().int()[torch.randperm(B, generator=g)].tolist()
    prompt = torch.randn(B, NP, 128, generator=g)
    text = torch.randint(0, TOKENS, (B, T), generator=g)
    dur = torch.randint(1, 20, (B, T), generator=g)
    for b, t in enumerate(tlens):
        dur[b, t:] = 0
    dur = (dur.float() * (SEQ / dur.sum(-1, keepdim=True))).floor().long()   # <= SEQ frames, 0 past the text
    lat = torch.randn(B, SEQ, 512, generator=g)
    pitch = torch.rand(B, SEQ, generator=g) * 300 + 80
    times = torch.rand(B, generator=g)
    noise = torch.randn(B, SEQ, 512, generator=g)
    prompt, text, dur, lat, pitch, times, noise = (t.to(dev) for t in (prompt, text, dur, lat, pitch, times, noise))

    def zero():
        for p in trained:
            p.grad = None

    def ragged():
        zero()
        ns(lat, text=text, prompt=prompt, pitch=pitch, duration=dur, times=times, noise=noise, prompt_lens=plens,
           phoneme_lens=tlens).backward()

    def sequential():
        zero()
        for b in range(B):
            ns(lat[b:b + 1], text=text[b:b + 1, :tlens[b]], prompt=prompt[b:b + 1, :plens[b]], pitch=pitch[b:b + 1],
               duration=dur[b:b + 1, :tlens[b]], times=times[b:b + 1], noise=noise[b:b + 1]).backward()

    def padded():
        zero()
        ns(lat, text=text, prompt=prompt, pitch=pitch, duration=dur, times=times, noise=noise).backward()

    legs = {"ragged_batch": ragged, "sequential_b1": sequential, "padded_batch": padded}
    ms = {k: [] for k in legs}
    launches = {}
    for fn in legs.values():   # warm-up: packing, transposed packs, kernel attributes
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
            ms[name].append(e0.elapsed_time(e1))
            launches[name] = ops.launch_count() - n0
    med = {k: statistics.median(v) for k, v in ms.items()}
    print(json.dumps({"workload": f"one training step (forward + backward), B={B} prompts {min(plens)}-{max(plens)} "
                                  f"frames, texts {min(tlens)}-{max(tlens)} phonemes, {SEQ} latent frames, cfg3 denoiser",
                      "median_ms": med, "all_ms": ms, "launches_per_step": launches,
                      "speedup_ragged_vs_sequential": med["sequential_b1"] / med["ragged_batch"],
                      "ragged_over_padded": med["ragged_batch"] / med["padded_batch"], "card": card(dev)}))


if __name__ == "__main__":
    main()
