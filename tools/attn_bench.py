#!/usr/bin/env python
"""Time the attention forward at the cfg2 shape (B=32, H=8, N=1024) with CUDA events.
Usage: python tools/attn_bench.py [kernel_selector] [iters]   (every selector runs the same sm_90a kernel)"""
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import torch  # noqa: E402
from naturalspeech2_pytorch_b200 import ops  # noqa: E402

kern = int(sys.argv[1]) if len(sys.argv) > 1 else ops.ATTN_AUTO
iters = int(sys.argv[2]) if len(sys.argv) > 2 else 5
B, H, N = 32, 8, 1024
inner = H * 64
torch.manual_seed(0)
qkv = torch.randn(B, N, 3 * inner, device="cuda").bfloat16()
out = torch.empty(B, N, inner, device="cuda", dtype=torch.bfloat16)
args = (qkv[:, :, :inner], qkv[:, :, inner:2 * inner], qkv[:, :, 2 * inner:], out)
for _ in range(2):
    ops.attention(*args, heads=H, kernel=kern)
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(iters):
    ops.attention(*args, heads=H, kernel=kern)
e1.record()
torch.cuda.synchronize()
us = e0.elapsed_time(e1) / iters * 1e3
flops = 4.0 * B * H * N * N * 64
print(f"kernel {kern}: {us:.1f} us/launch = {flops / us / 1e6:.0f} TFLOP/s (x12 layers = {us * 12 / 1e3:.3f} ms/step)")
