"""Timing of SEANetDecoder (Encodec 24 kHz decoder on the sm_90a kernels) against PyTorch (cuDNN LSTM and convs) in
fp32 and bf16 on the same GPU:
    python tools/codec_bench.py [--batch 32] [--frames 1024] [--reps 5] [--out codec_bench.json]
Decodes (batch, frames, 128) latents = batch x frames / 75 s of 24 kHz audio.  Reports ms per decode (CUDA events
around each call after warm-up, runs of the three implementations alternated), audio seconds per second, the output
difference against the PyTorch fp32 decode, and a per-stage split from a separate torch.profiler run.
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

import seanet_oracle  # noqa: E402
from golden.make_golden_seanet import filled_state_dict  # noqa: E402
from naturalspeech2_pytorch_b200 import SEANetDecoder  # noqa: E402


def torch_decoder(sd, dtype):
    """The decoder in plain PyTorch: cuDNN LSTM, cuDNN convs, weight norm folded once."""
    lstm = torch.nn.LSTM(512, 512, 2).cuda().to(dtype)
    lstm.load_state_dict({k[len("layers.1.lstm."):]: v for k, v in sd.items() if k.startswith("layers.1.lstm.")})
    lstm.flatten_parameters()
    sdd = {k: v.to(dtype) for k, v in sd.items()}

    @torch.no_grad()
    def run(emb):
        x = seanet_oracle._conv(emb.to(dtype).transpose(1, 2), sdd, "layers.0.conv", False)
        xt = x.permute(2, 0, 1)
        x = (lstm(xt)[0] + xt).permute(1, 2, 0)
        for si, s in enumerate(seanet_oracle.RATIOS):
            i = 2 + 3 * si
            x = seanet_oracle._conv_t(F.elu(x), sdd, f"layers.{i + 1}.conv", s, False)
            x = seanet_oracle.resnet_block(x, sdd, f"layers.{i + 2}")
        return seanet_oracle._conv(F.elu(x), sdd, "layers.15.conv", False).float()
    return run


def time_ms(fn, emb):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn(emb)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--frames", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    B, N = a.batch, a.frames
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(f"card: {card}")

    sd = filled_state_dict([(k, tuple(v.shape)) for k, v in SEANetDecoder().state_dict().items()])
    dec = SEANetDecoder()
    dec.load_state_dict({k: v.float() for k, v in sd.items()})
    dec = dec.cuda().eval()
    sdc = {k: v.float().cuda() for k, v in sd.items()}
    impls = {"ours": dec, "torch_fp32": torch_decoder(sdc, torch.float32),
             "torch_bf16": torch_decoder(sdc, torch.bfloat16)}
    emb = torch.randn(B, N, 128, device="cuda", generator=torch.Generator(device="cuda").manual_seed(0))
    outs = {k: f(emb) for k, f in impls.items()}     # warm-up (workspaces, packs, cuDNN algorithm choice)
    for f in impls.values():
        f(emb)
    torch.cuda.synchronize()
    times = {k: [] for k in impls}
    for _ in range(a.reps):
        for k, f in impls.items():
            times[k].append(time_ms(f, emb))
    audio_s = B * N / 75.0
    res = {"card": card, "batch": B, "frames": N, "audio_seconds": audio_s}
    ref = outs["torch_fp32"].double()
    for k in impls:
        ms = sorted(times[k])[len(times[k]) // 2]
        d = outs[k].double() - ref
        res[k] = {"ms_median": ms, "ms_all": times[k], "audio_s_per_s": audio_s / (ms / 1e3),
                  "rel_l2_vs_torch_fp32": float(d.norm() / ref.norm()), "max_abs_vs_torch_fp32": float(d.abs().max())}
        print(f"{k:>11}: {ms:8.2f} ms/decode  {audio_s / (ms / 1e3):9.0f} audio s/s  "
              f"rel-L2 vs torch fp32 {res[k]['rel_l2_vs_torch_fp32']:.2e}  runs {[round(t, 2) for t in times[k]]}")

    # per-stage split of our decode, from a separate profiled call
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        dec(emb)
        torch.cuda.synchronize()
    split = {"lstm": 0.0, "gemm": 0.0, "elu_pad": 0.0, "tail": 0.0, "other": 0.0}
    for ev in prof.key_averages():
        name, us = ev.key, ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
        stage = ("lstm" if "lstm_seq_kernel" in name else "tail" if "seanet_tail" in name else
                 "gemm" if "gemm_kernel" in name else "elu_pad" if "elu_pad" in name else "other")
        split[stage] += us / 1e3
    res["stage_ms_profiled"] = split
    print("stage split (ms, profiled call): " + ", ".join(f"{k} {v:.2f}" for k, v in split.items()))
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
