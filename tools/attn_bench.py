#!/usr/bin/env python
"""Time the attention forward (and, with --bwd, the backward) with CUDA events, by default at the cfg2 shape
(B=32, H=8, N=1024).  --dropout P runs the dropout kernels (Philox mask drawn in the forward, regenerated in the
backward); --shape B,H,N another shape, e.g. 32,8,103 for the conditioning encoders' prompts.
Usage: python tools/attn_bench.py [iters] [--dropout P] [--shape B,H,N] [--bwd]"""
import argparse
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import torch  # noqa: E402
from naturalspeech2_pytorch_b200 import ops  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("iters", nargs="?", type=int, default=5)
ap.add_argument("--dropout", type=float, default=0.0)
ap.add_argument("--shape", default="32,8,1024")
ap.add_argument("--bwd", action="store_true")
a = ap.parse_args()
iters = a.iters
B, H, N = (int(v) for v in a.shape.split(","))
drop = (0x9E3779B97F4A7C15, 1, a.dropout) if a.dropout > 0 else None
inner = H * 64
torch.manual_seed(0)
qkv = torch.randn(B, N, 3 * inner, device="cuda").bfloat16()
out = torch.empty(B, N, inner, device="cuda", dtype=torch.bfloat16)
lse = torch.empty(B, H, N, device="cuda")
d_o = torch.randn(B, N, inner, device="cuda").bfloat16()
dq = torch.zeros(B, N, inner, device="cuda")
dkv = torch.empty(B, N, 2 * inner, device="cuda", dtype=torch.bfloat16)
args = (qkv[:, :, :inner], qkv[:, :, inner:2 * inner], qkv[:, :, 2 * inner:], out)


def fwd():
    ops.attention(*args, heads=H, lse=lse, dropout=drop)


def bwd():
    ops.attention_bwd(*args[:3], out, d_o, lse, dq, dkv[:, :, :inner], dkv[:, :, inner:], heads=H, dropout=drop)


def timed(fn):
    for _ in range(2):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e3


tag = f"B{B} H{H} N{N} dropout {a.dropout:g}"
us = timed(fwd)
flops = 4.0 * B * H * N * N * 64
print(f"forward {tag}: {us:.1f} us/launch = {flops / us / 1e6:.0f} TFLOP/s (x12 layers = {us * 12 / 1e3:.3f} ms/step)")
if a.bwd:
    fwd()
    us = timed(bwd)
    print(f"backward {tag}: {us:.1f} us/call = {2.5 * flops / us / 1e6:.0f} TFLOP/s")
