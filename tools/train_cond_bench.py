#!/usr/bin/env python
"""Conditional training step with the conditioning front end in the loop, timed beside the same step without it.

    python tools/train_cond_bench.py [--steps K] [--warmup W] [--duration-pitch] [--duration-pitch-dropout]

  cond_e2e   configs[4] training step (cfg3 denoiser Model(512, depth 12, heads 8, dim_prompt 512), B=32, N=1024) with
             SpeechPromptEncoder(dim_codebook=128) on (32, 103, 128) prompt latents, PhonemeEncoder on 100 phoneme ids
             per sample, durations summing to <= 1024 frames, backward through everything (encoders, pitch embedding,
             the denoiser's input gradients) and fused AdamW over the trained parameters
  cfg5       the same denoiser step on precomputed (prompt_enc, cond) — bench.py's secondary train_cfg5 workload
  --duration-pitch  adds cond_e2e_dp: the same step with Conditioner(train_duration_pitch=True), i.e. the duration /
             pitch predictor (dim 512, depth 10, both trunks) run on the encoders' outputs and trained through its L1
             losses, timed alternately with cond_e2e (two rounds each); and dpp_alone: the predictor's forward +
             backward on its own at B 32 x T 100 x Np 103 (CUDA events per call, median of --calls calls, two rounds)
             with the peak memory of one training call
  --duration-pitch-dropout  (implies --duration-pitch) also times cond_e2e_dp with the predictor's dropout drawn
             (Conditioner(duration_pitch_dropout=True): p = 0.2 on its 20 cross attentions) alternately
             with cond_e2e_dp without it (two rounds each), and the predictor alone with it
Prints one JSON line: ms / steps per second of both, the encoders' measured share of the step (1 - cfg5 / cond_e2e),
the card name and its enforced power limit (part of every number).
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from naturalspeech2_pytorch_b200 import Model, NaturalSpeech2  # noqa: E402
from naturalspeech2_pytorch_b200.encoders import Conditioner  # noqa: E402

CFG3 = dict(dim=512, depth=12, heads=8, dim_prompt=512, condition_on_prompt=True)
B, SEQ, NP, T, TOKENS = 32, 1024, 103, 100, 150


def card(dev):
    out = {"name": torch.cuda.get_device_name(dev)}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", str(dev.index)],
                           capture_output=True, text=True, timeout=10)
        out["power_limit_w"] = float(r.stdout.strip().splitlines()[0])
    except Exception as e:
        out["power_limit_w"] = None
        out["power_limit_error"] = f"{type(e).__name__}: {e}"
    return out


def timed(step, steps, warmup):
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        loss = step()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps, float(loss)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--train-dropout", action="store_true",
                    help="train the encoders with the reference's dropout (Conditioner(train_dropout=True))")
    ap.add_argument("--duration-pitch", action="store_true",
                    help="also time the step with the duration / pitch predictor trained, and the predictor alone")
    ap.add_argument("--duration-pitch-dropout", action="store_true",
                    help="also time the --duration-pitch step and the predictor alone with the predictor's dropout")
    ap.add_argument("--calls", type=int, default=20, help="predictor-alone calls per round (median)")
    args = ap.parse_args()
    args.duration_pitch |= args.duration_pitch_dropout
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    model = Model(**CFG3).to(dev).train()
    g = torch.Generator().manual_seed(200)
    lat = torch.randn(B, SEQ, 512, generator=g).to(dev)

    # ---- cfg5: denoiser on precomputed conditioning ----
    ns = NaturalSpeech2(model, target_sample_hz=24000)
    prompt_enc = torch.randn(B, NP, 512, generator=g).to(dev)
    cond = torch.randn(B, 512, SEQ, generator=g).to(dev)
    opt = torch.optim.AdamW(model.parameters(), lr=1e-4, fused=True)

    def step_cfg5():
        opt.zero_grad(set_to_none=True)
        loss = ns(lat, prompt_enc=prompt_enc, cond=cond)
        loss.backward()
        opt.step()
        return loss.detach()

    ms5, loss5 = timed(step_cfg5, args.steps, args.warmup)
    del opt

    # ---- cond_e2e: the encoders trained jointly ----
    cond_net = Conditioner(dim_codebook=128, num_phoneme_tokens=TOKENS, train_dropout=args.train_dropout).to(dev).train()
    ns = NaturalSpeech2(model, target_sample_hz=24000, conditioner=cond_net)
    trained = [*model.parameters(), *cond_net.prompt_enc.parameters(), *cond_net.phoneme_enc.parameters(),
               *cond_net.pitch_emb.parameters()]   # the duration / pitch predictor only feeds the discarded aux loss
    opt = torch.optim.AdamW(trained, lr=1e-4, fused=True)
    prompt = torch.randn(B, NP, 128, generator=g).to(dev)
    text = torch.randint(0, TOKENS, (B, T), generator=g).to(dev)
    dur = torch.randint(0, 20, (B, T), generator=g)
    dur = (dur.float() * (SEQ / dur.sum(-1, keepdim=True).clamp_min(1))).floor().long().to(dev)   # <= SEQ frames
    pitch = (torch.rand(B, SEQ, generator=g) * 300 + 80).to(dev)

    def step_e2e():
        opt.zero_grad(set_to_none=True)
        loss = ns(lat, text=text, prompt=prompt, pitch=pitch, duration=dur)
        loss.backward()
        opt.step()
        return loss.detach()

    ms_e2e, loss_e2e = timed(step_e2e, args.steps, args.warmup)
    res = {
        "cond_e2e": {"ms_per_step": round(ms_e2e, 3), "steps_per_s": round(1e3 / ms_e2e, 3), "loss": round(loss_e2e, 5)},
        "cfg5": {"ms_per_step": round(ms5, 3), "steps_per_s": round(1e3 / ms5, 3), "loss": round(loss5, 5)},
        "encoder_share_of_step": round(1.0 - ms5 / ms_e2e, 4), "train_dropout": args.train_dropout,
        "steps": args.steps, "warmup": args.warmup,
        "batch": B, "card": card(dev)}
    if args.duration_pitch:
        res.update(duration_pitch_legs(args, ns, cond_net, opt, step_e2e, trained, lat, text, prompt, pitch, dur))
    print(json.dumps(res))


def duration_pitch_legs(args, ns, cond_net, opt, step_e2e, trained, lat, text, prompt, pitch, dur):
    """cond_e2e with and without the predictor trained (alternated), and the predictor's forward + backward alone."""
    dev = lat.device
    opt_dp = torch.optim.AdamW([*trained, *cond_net.duration_pitch.parameters()], lr=1e-4, fused=True)

    def step_dp():
        opt_dp.zero_grad(set_to_none=True)
        loss = ns(lat, text=text, prompt=prompt, pitch=pitch, duration=dur)
        loss.backward()
        opt_dp.step()
        return loss.detach()

    rounds = {"cond_e2e": [], "cond_e2e_dp": []}
    for _ in range(2):
        cond_net.train_duration_pitch = False
        rounds["cond_e2e"].append(timed(step_e2e, args.steps, args.warmup)[0])
        cond_net.train_duration_pitch = True
        rounds["cond_e2e_dp"].append(timed(step_dp, args.steps, args.warmup)[0])
    dp = cond_net.duration_pitch
    if args.duration_pitch_dropout:   # the predictor's step with and without its dropout, alternated
        cond_net.train_duration_pitch = True
        rounds["cond_e2e_dp_no_dropout"], rounds["cond_e2e_dp_dropout"] = [], []
        for _ in range(2):
            dp.train_dropout = False
            rounds["cond_e2e_dp_no_dropout"].append(timed(step_dp, args.steps, args.warmup)[0])
            dp.train_dropout = True
            rounds["cond_e2e_dp_dropout"].append(timed(step_dp, args.steps, args.warmup)[0])
        dp.train_dropout = False
    cond_net.train_duration_pitch = False
    # the predictor alone: phoneme encodings and prompts as the encoders hand them over
    g = torch.Generator().manual_seed(300)
    x = torch.randn(B, T, 512, generator=g).to(dev).requires_grad_(True)
    pr = torch.randn(B, NP, 512, generator=g).to(dev).requires_grad_(True)
    d_dur, d_pitch = (torch.randn(B, T, generator=g).to(dev) for _ in range(2))

    def call():
        dp.zero_grad(set_to_none=True)
        x.grad = pr.grad = None
        dur_p, pitch_p = dp(x, pr)
        torch.autograd.backward([dur_p, pitch_p], [d_dur, d_pitch])

    for _ in range(3):
        call()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(dev)
    base = torch.cuda.memory_allocated(dev)
    call()
    torch.cuda.synchronize()
    peak_mb = (torch.cuda.max_memory_allocated(dev) - base) / 2 ** 20
    def median_call_ms():
        ms = []
        for _ in range(args.calls):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            call()
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        return sorted(ms)[len(ms) // 2]

    alone, alone_dropout = [], []
    for _ in range(2):
        alone.append(median_call_ms())
        if args.duration_pitch_dropout:
            dp.train_dropout = True
            alone_dropout.append(median_call_ms())
            dp.train_dropout = False
    dp.eval()
    with torch.no_grad():
        launches_fwd = _launches(lambda: dp(x.detach(), pr.detach()))
    dp.train()
    launches_train = _launches(call)
    extra = {}
    if args.duration_pitch_dropout:
        dp.train_dropout = True
        extra = {"dropout": {
            "cond_e2e_dp_no_dropout_ms_rounds": [round(v, 3) for v in rounds["cond_e2e_dp_no_dropout"]],
            "cond_e2e_dp_dropout_ms_rounds": [round(v, 3) for v in rounds["cond_e2e_dp_dropout"]],
            "dropout_share_of_dp_step": round(1.0 - sum(rounds["cond_e2e_dp_no_dropout"])
                                              / sum(rounds["cond_e2e_dp_dropout"]), 4),
            "alone_fwd_bwd_median_ms_rounds": [round(v, 3) for v in alone_dropout], "p": dp.attn_dropout,
            "launches_fwd_bwd": _launches(call)}}
        dp.train_dropout = False
    return {"duration_pitch": {**extra,
        "cond_e2e_ms_rounds": [round(v, 3) for v in rounds["cond_e2e"]],
        "cond_e2e_dp_ms_rounds": [round(v, 3) for v in rounds["cond_e2e_dp"]],
        "predictor_share_of_step": round(1.0 - sum(rounds["cond_e2e"]) / sum(rounds["cond_e2e_dp"]), 4),
        "alone_fwd_bwd_median_ms_rounds": [round(v, 3) for v in alone], "alone_calls_per_round": args.calls,
        "alone_shape": [B, T, NP], "alone_peak_extra_mib": round(peak_mb, 1),
        "launches_inference_fwd": launches_fwd, "launches_fwd_bwd": launches_train}}


def _launches(fn):
    from naturalspeech2_pytorch_b200 import ops
    n0 = ops.launch_count()
    fn()
    torch.cuda.synchronize()
    return ops.launch_count() - n0


if __name__ == "__main__":
    main()
