"""Timing of SEANetDecoder and SEANetEncoder (Encodec 24 kHz decoder and encoder on the sm_90a kernels) against
PyTorch (cuDNN LSTM and convs) in fp32 and bf16 on the same GPU:
    python tools/codec_bench.py [--batch 32] [--frames 1024] [--reps 5] [--legs decode,encode,ragged]
                                [--min-frames 256] [--out codec_bench.json]
Decodes (batch, frames, 128) latents and encodes (batch, 320 frames) samples of audio = batch x frames / 75 s of 24 kHz
audio.  Reports ms per call (CUDA events around each call after warm-up, runs of the three implementations
alternated, median), audio seconds per second, the output difference against the PyTorch fp32 path, and a per-stage
split from a separate torch.profiler run; for the encoder also the head kernel's achieved FP32 rate (3,296 MACs per
sample, from shapes).  The `ragged` leg encodes the same batch padded at the end, with per-sample lengths drawn
uniformly from [--min-frames, frames] (seeded), through `SEANetEncoder(lengths=)` against the call without lengths
(which computes every padded tile), alternated the same way; it reports the share of padded frames and checks that each
sample's frames equal the unpadded call's prefix.
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
from golden import make_golden_seanet_encoder as genc  # noqa: E402
from naturalspeech2_pytorch_b200 import SEANetDecoder, SEANetEncoder  # noqa: E402

HEAD_MACS_PER_SAMPLE = 7 * 32 + 3 * 32 * 16 + 32 * 32 + 16 * 32   # conv7 1->32, conv3 32->16, shortcut, conv1x1


def torch_decoder(sd, dtype):
    """The decoder in plain PyTorch: cuDNN LSTM, cuDNN convs, weight norm folded once."""
    lstm = torch.nn.LSTM(512, 512, 2).cuda().to(dtype)
    lstm.load_state_dict({k[len("layers.1.lstm."):]: v for k, v in sd.items() if k.startswith("layers.1.lstm.")})
    lstm.flatten_parameters()
    sdd = {k: v.to(dtype) for k, v in sd.items()}

    @torch.no_grad()
    def run(emb):
        x = seanet_oracle.conv(emb.to(dtype).transpose(1, 2), sdd, "layers.0.conv", False)
        xt = x.permute(2, 0, 1)
        x = (lstm(xt)[0] + xt).permute(1, 2, 0)
        for si, s in enumerate(seanet_oracle.RATIOS):
            i = 2 + 3 * si
            x = seanet_oracle._conv_t(F.elu(x), sdd, f"layers.{i + 1}.conv", s, False)
            x = seanet_oracle.resnet_block(x, sdd, f"layers.{i + 2}")
        return seanet_oracle.conv(F.elu(x), sdd, "layers.15.conv", False).float()
    return run


def torch_encoder(sd, dtype):
    """The encoder in plain PyTorch: cuDNN LSTM, cuDNN convs, weight norm folded once."""
    lstm = torch.nn.LSTM(512, 512, 2).cuda().to(dtype)
    lstm.load_state_dict({k[len("layers.13.lstm."):]: v for k, v in sd.items() if k.startswith("layers.13.lstm.")})
    lstm.flatten_parameters()
    sdd = {k: v.to(dtype) for k, v in sd.items()}

    @torch.no_grad()
    def run(audio):
        x = seanet_oracle.conv(audio.to(dtype)[:, None], sdd, "layers.0.conv", False)
        for si, s in enumerate(reversed(seanet_oracle.RATIOS)):
            i = 1 + 3 * si
            x = seanet_oracle.resnet_block(x, sdd, f"layers.{i}")
            x = seanet_oracle.conv(F.elu(x), sdd, f"layers.{i + 2}.conv", False, stride=s)
        xt = x.permute(2, 0, 1)
        x = (lstm(xt)[0] + xt).permute(1, 2, 0)
        return seanet_oracle.conv(F.elu(x), sdd, "layers.15.conv", False).transpose(1, 2).float()
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
    ap.add_argument("--legs", default="decode,encode")
    ap.add_argument("--min-frames", type=int, default=256, help="ragged leg: shortest length drawn (>= 7)")
    a = ap.parse_args()
    B, N = a.batch, a.frames
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(f"card: {card}")
    res = {"card": card, "batch": B, "frames": N, "audio_seconds": B * N / 75.0}
    for leg in a.legs.split(","):
        if leg == "ragged":
            res[leg] = ragged_leg(B, N, a.reps, a.min_frames)
        else:
            res[leg] = {"decode": decode_leg, "encode": encode_leg}[leg](B, N, a.reps)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(res, indent=1))


def run_impls(impls, inp, reps, audio_s, what):
    outs = {k: f(inp) for k, f in impls.items()}     # warm-up (workspaces, packs, cuDNN algorithm choice)
    for f in impls.values():
        f(inp)
    torch.cuda.synchronize()
    times = {k: [] for k in impls}
    for _ in range(reps):
        for k, f in impls.items():
            times[k].append(time_ms(f, inp))
    res = {}
    ref = outs["torch_fp32"].double()
    for k in impls:
        ms = sorted(times[k])[len(times[k]) // 2]
        d = outs[k].double() - ref
        res[k] = {"ms_median": ms, "ms_all": times[k], "audio_s_per_s": audio_s / (ms / 1e3),
                  "rel_l2_vs_torch_fp32": float(d.norm() / ref.norm()), "max_abs_vs_torch_fp32": float(d.abs().max())}
        print(f"{k:>11}: {ms:8.2f} ms/{what}  {audio_s / (ms / 1e3):9.0f} audio s/s  "
              f"rel-L2 vs torch fp32 {res[k]['rel_l2_vs_torch_fp32']:.2e}  runs {[round(t, 2) for t in times[k]]}")
    return res


def stage_split(fn, inp):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn(inp)
        torch.cuda.synchronize()
    split = {"lstm": 0.0, "gemm": 0.0, "elu_pad": 0.0, "tail": 0.0, "head": 0.0, "other": 0.0}
    for ev in prof.key_averages():
        name, us = ev.key, ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
        stage = ("lstm" if "lstm_seq_kernel" in name else "tail" if "seanet_tail" in name else
                 "head" if "seanet_head" in name else
                 "gemm" if "gemm_kernel" in name else "elu_pad" if "elu_pad" in name else "other")
        split[stage] += us / 1e3
    return split


def encode_leg(B, N, reps):
    print(f"encode: ({B}, {320 * N}) samples")
    keys_shapes = [(k, tuple(v.shape)) for k, v in SEANetEncoder().state_dict().items()]
    sd = genc.filled_state_dict(keys_shapes)
    enc = SEANetEncoder()
    enc.load_state_dict({k: v.float() for k, v in sd.items()})
    enc = enc.cuda().eval()
    sdc = {k: v.float().cuda() for k, v in sd.items()}
    impls = {"ours": enc, "torch_fp32": torch_encoder(sdc, torch.float32),
             "torch_bf16": torch_encoder(sdc, torch.bfloat16)}
    audio = genc.audio(B, N).float().cuda()
    res = run_impls(impls, audio, reps, B * N / 75.0, "encode")
    split = stage_split(enc, audio)
    res["stage_ms_profiled"] = split
    flops = 2.0 * HEAD_MACS_PER_SAMPLE * B * 320 * N
    res["head_tflops_fp32"] = flops / (split["head"] / 1e3) / 1e12
    print("stage split (ms, profiled call): " + ", ".join(f"{k} {v:.2f}" for k, v in split.items() if k != "tail"))
    print(f"head: {HEAD_MACS_PER_SAMPLE} MAC/sample, {res['head_tflops_fp32']:.1f} TFLOP/s FP32 achieved "
          f"(against the 67 TFLOP/s data-sheet FP32 peak)")
    return res


def _seeded_encoder():
    keys_shapes = [(k, tuple(v.shape)) for k, v in SEANetEncoder().state_dict().items()]
    enc = SEANetEncoder()
    enc.load_state_dict({k: v.float() for k, v in genc.filled_state_dict(keys_shapes).items()})
    return enc.cuda().eval()


def ragged_leg(B, N, reps, min_frames):
    lens = torch.randint(min_frames, N + 1, (B,), generator=torch.Generator().manual_seed(0)).tolist()
    padded = 1.0 - sum(lens) / (B * N)
    print(f"ragged encode: ({B}, {320 * N}) samples, lengths in [{min(lens)}, {max(lens)}] frames, "
          f"{100 * padded:.1f} % padding")
    enc = _seeded_encoder()
    audio = genc.audio(B, N).float().cuda()
    impls = {"no_lengths": enc, "lengths": lambda x: enc(x, lengths=lens)}
    outs = {k: f(audio) for k, f in impls.items()}     # warm-up
    for b, n in enumerate(lens):
        assert torch.equal(outs["lengths"][b, :n], outs["no_lengths"][b, :n]), b
    times = {k: [] for k in impls}
    for _ in range(reps):
        for k, f in impls.items():
            times[k].append(time_ms(f, audio))
    res = {"lengths": lens, "padded_share": padded}
    for k in impls:
        ms = sorted(times[k])[len(times[k]) // 2]
        res[k] = {"ms_median": ms, "ms_all": times[k], "audio_s_per_s": sum(lens) / 75.0 / (ms / 1e3)}
        print(f"{k:>11}: {ms:8.2f} ms/encode  {res[k]['audio_s_per_s']:9.0f} unpadded audio s/s  "
              f"runs {[round(t, 2) for t in times[k]]}")
    return res


def decode_leg(B, N, reps):
    print(f"decode: ({B}, {N}, 128) latents")
    sd = filled_state_dict([(k, tuple(v.shape)) for k, v in SEANetDecoder().state_dict().items()])
    dec = SEANetDecoder()
    dec.load_state_dict({k: v.float() for k, v in sd.items()})
    dec = dec.cuda().eval()
    sdc = {k: v.float().cuda() for k, v in sd.items()}
    impls = {"ours": dec, "torch_fp32": torch_decoder(sdc, torch.float32),
             "torch_bf16": torch_decoder(sdc, torch.bfloat16)}
    emb = torch.randn(B, N, 128, device="cuda", generator=torch.Generator(device="cuda").manual_seed(0))
    res = run_impls(impls, emb, reps, B * N / 75.0, "decode")
    split = stage_split(dec, emb)
    res["stage_ms_profiled"] = split
    print("stage split (ms, profiled call): " + ", ".join(f"{k} {v:.2f}" for k, v in split.items() if k != "head"))
    return res


if __name__ == "__main__":
    main()
