#!/usr/bin/env python
"""Time each hot kernel at the cfg2 shapes (B=32, N=1024, D=512) with CUDA events.

Every GEMM shape is timed twice in the same process: the full kernel, and the mainloop alone
(NS2_GEMM_FLAG_SKIP_EPILOGUE: same tiles and MMAs, nothing written).  The difference is what the fused
epilogue costs on top of the MMAs.  Prints the GPU name and power limit first, because every number below
depends on them.

    python tools/prof_kernels.py [conv fold attn wavenet ffin ffout attnout qkv norm rvq sweep]

"conv" is the unfolded FFN causal conv (1408 -> 1408, BF16 out), kept to compare with "fold": the conv with the
output projection folded into its taps, 1408 -> 512, F32 + residual in place, the launch the model runs.  "conv"'s
rate counts the unpadded conv's FLOPs (1365 wide), "fold"'s the FLOPs the launch executes, padding included.
"""
import os
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from naturalspeech2_pytorch_b200 import ops  # noqa: E402

B, N, D, H, Di, Dp = 32, 1024, 512, 8, 1365, 1408
dev = "cuda"
bf = torch.bfloat16
which = set(sys.argv[1:]) or {"conv", "fold", "attn", "wavenet", "ffin", "ffout", "attnout", "qkv", "norm", "rvq"}
reps = int(os.environ.get("NS2_PROF_REPS", "20"))
SKIP_EPILOGUE = 1   # NS2_GEMM_FLAG_SKIP_EPILOGUE


def gpu_info():
    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader",
                            "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        limits = q.stdout.strip() or "power limit unknown"
    except (OSError, subprocess.SubprocessError):
        limits = "power limit unknown"
    return f"{name}, {limits}"


def time_ms(fn):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def rate(ms, flops=None, bytes_=None):
    extra = ""
    if flops:
        extra += f" {flops / ms / 1e9:.0f} TFLOP/s"
    if bytes_:
        extra += f" {bytes_ / ms / 1e6:.0f} GB/s"
    return extra


def timeit(name, fn, flops=None, bytes_=None):
    ms = time_ms(fn)
    print(f"{name}: {ms:.4f} ms{rate(ms, flops, bytes_)}", flush=True)


def time_gemm(name, flops, **kw):
    """kw: the ops.gemm arguments.  Full kernel, then mainloop only; the epilogue's cost is the difference."""
    full = time_ms(lambda: ops.gemm(**kw))
    main = time_ms(lambda: ops.gemm(**kw, flags=SKIP_EPILOGUE))
    print(f"{name}: full {full:.4f} ms{rate(full, flops)} | mainloop {main:.4f} ms{rate(main, flops)} | "
          f"epilogue {full - main:+.4f} ms", flush=True)


print(f"# {gpu_info()}; {reps} launches per timing", flush=True)
torch.manual_seed(0)
if "conv" in which:
    g = (torch.randn(B, N, Dp, device=dev) * 0.5).to(bf)
    wc = (torch.randn(Dp, 3 * Dp, device=dev) * 0.02).to(bf)
    bc = torch.randn(Dp, device=dev)
    out = torch.empty(B, N, Dp, device=dev, dtype=bf)
    time_gemm("ff_conv gemm<256,1,BF16>", 2.0 * B * N * Di * 3 * Di, a=g, w=wc, out=out, n=Dp,
              epilogue=ops.EPI_BF16, bias=bc, segs=ops.conv3_segs(Dp))
if "fold" in which:
    g = (torch.randn(B, N, Dp, device=dev) * 0.5).to(bf)
    wo = (torch.randn(D, 3 * Dp, device=dev) * 0.02).to(bf)
    bo = torch.randn(D, device=dev)
    xr = torch.randn(B, N, D, device=dev)
    time_gemm("ff_conv folded gemm<256,1,F32+resid in place> K=3x1408", 2.0 * B * N * D * 3 * Dp, a=g, w=wo, out=xr,
              n=D, epilogue=ops.EPI_F32, bias=bo, resid=xr, segs=ops.conv3_segs(Dp))
if "attn" in which:
    qkv = torch.randn(B, N, 3 * H * 64, device=dev).to(bf)
    o = torch.empty(B, N, H * 64, device=dev, dtype=bf)
    timeit("attn_fwd", lambda: ops.attention(qkv[:, :, :512], qkv[:, :, 512:1024], qkv[:, :, 1024:], o, heads=H),
           flops=4.0 * B * H * N * N * 64)
if "wavenet" in which:
    G = 8
    x = (torch.randn(B, N, G * D, device=dev) * 0.5).to(bf)
    wp = (torch.randn(G * D, 4 * D, device=dev) * 0.02).to(bf)
    bias = torch.randn(2 * G * D, device=dev)
    film = torch.randn(B, G * 2 * D, device=dev)
    out = torch.empty(B, N, G * D, device=dev, dtype=bf)
    segs = ops.conv3_segs(D) + [(0, 3 * D, D, 0, 1)]
    time_gemm("wavenet stack gemm<128,2,WAVENET>", 2.0 * B * N * D * 4 * D * G, a=x, w=wp, out=out, n=D,
              epilogue=ops.EPI_WAVENET, bias=bias, bias1_off=G * D, segs=segs, film=film, film_group_stride=2 * D,
              groups=G, a_group_col_stride=D, b_group_row_stride=D, out_group_col_stride=D,
              dil=[2 ** i for i in range(G)])
if "ffin" in which:
    h = torch.randn(B, N, D, device=dev).to(bf)
    w1 = (torch.randn(2 * Dp, D, device=dev) * 0.04).to(bf)
    b1 = torch.randn(2 * Dp, device=dev)
    out = torch.empty(B, N, Dp, device=dev, dtype=bf)
    time_gemm("ff_in gemm<256,1,GEGLU>", 2.0 * B * N * D * 2 * Di, a=h, w=w1, out=out, n=2 * Dp,
              epilogue=ops.EPI_GEGLU, bias=b1)
if "ffout" in which:
    c = torch.randn(B, N, Dp, device=dev).to(bf)
    w2 = (torch.randn(D, Dp, device=dev) * 0.03).to(bf)
    b2 = torch.randn(D, device=dev)
    xr = torch.randn(B, N, D, device=dev)
    time_gemm("ff_out gemm<256,1,F32+resid in place> K=1408", 2.0 * B * N * Di * D, a=c, w=w2, out=xr, n=D,
              epilogue=ops.EPI_F32, bias=b2, resid=xr)
if "attnout" in which:
    o = torch.randn(B, N, H * 64, device=dev).to(bf)
    wo = (torch.randn(D, H * 64, device=dev) * 0.04).to(bf)
    xr = torch.randn(B, N, D, device=dev)
    time_gemm("attn_out gemm<256,1,F32+resid in place> K=512", 2.0 * B * N * H * 64 * D, a=o, w=wo, out=xr, n=D,
              epilogue=ops.EPI_F32, resid=xr)
if "qkv" in which:
    h = torch.randn(B, N, D, device=dev).to(bf)
    w = (torch.randn(1536, D, device=dev) * 0.04).to(bf)
    out = torch.empty(B, N, 1536, device=dev, dtype=bf)
    time_gemm("qkv gemm<256,1,BF16>", 2.0 * B * N * D * 1536, a=h, w=w, out=out, n=1536, epilogue=ops.EPI_BF16)
if "norm" in which:
    x = torch.randn(B, N, D, device=dev)
    film = torch.randn(B, 2 * D, device=dev)
    out = torch.empty(B, N, D, device=dev, dtype=bf)
    timeit("rmsnorm_film", lambda: ops.rmsnorm_film(x, out, film=film), bytes_=B * N * D * 6.0)
if "rvq" in which:
    cb = torch.randn(8, 1024, 128, device=dev)
    prep = ops.rvq_prepare(cb)
    F = 1 << 20
    x = torch.randn(F, 128, device=dev)
    codes = torch.empty(F, 8, device=dev, dtype=torch.int64)
    timeit("rvq_encode 1M x 8 x 1024", lambda: ops.rvq_encode(x, cb, prep, codes=codes), flops=2.0 * F * 8 * 1024 * 128)
    print(f"  -> {F * 8 / 1e6:.1f} Mcodes per launch")
if "sweep" in which:
    # plain bf16 GEMMs, M = 32768: tile shape / K depth effects
    for (n, k) in [(1536, 512), (1536, 4096), (2048, 4096), (1408, 4224), (512, 4096), (512, 512), (1024, 1024)]:
        a = (torch.randn(B, N, k, device=dev) * 0.5).to(bf)
        w = (torch.randn(n, k, device=dev) * 0.02).to(bf)
        out = torch.empty(B, N, n, device=dev, dtype=bf)
        time_gemm(f"plain gemm N={n} K={k}", 2.0 * B * N * n * k, a=a, w=w, out=out, n=n, epilogue=ops.EPI_BF16)
