#!/usr/bin/env python
"""Bring-up checks for the CUDA kernels on a real H100.

Each group runs in its own subprocess with a timeout, so a trapped or hung kernel in one group neither
poisons the CUDA context of the others nor stalls the box.  Results go to gpurun_out/check_<group>.log and a
summary is printed.  Usage: python tools/gpu_check.py [group ...]
"""
from __future__ import annotations

import math
import os
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
GROUPS = ["elementwise", "gemm_plain", "gemm_conv", "gemm_fused", "attn", "rvq"]


def _report(name, got, ref, atol, rtol):
    import torch
    got = got.float()
    ref = ref.float()
    err = (got - ref).abs()
    tol = atol + rtol * ref.abs()
    bad = (err > tol)
    nbad = int(bad.sum())
    finite = bool(torch.isfinite(got).all())
    print(f"[{'OK ' if nbad == 0 and finite else 'BAD'}] {name}: max_abs_err={float(err.max()):.3e} "
          f"ref_absmax={float(ref.abs().max()):.3e} bad={nbad}/{err.numel()} finite={finite}", flush=True)
    if nbad or not finite:
        idx = bad.nonzero()[:6]
        for i in idx:
            t = tuple(int(v) for v in i)
            print(f"      at {t}: got {float(got[t]):.5f} ref {float(ref[t]):.5f}")
        # structure of the failure: which rows / columns are wrong
        if got.dim() >= 2:
            flat_bad = bad.reshape(-1, bad.shape[-1])
            rows_bad = flat_bad.any(dim=1).nonzero().flatten()
            cols_bad = flat_bad.any(dim=0).nonzero().flatten()
            print(f"      bad rows: {rows_bad.numel()} (first {rows_bad[:12].tolist()}), "
                  f"bad cols: {cols_bad.numel()} (first {cols_bad[:12].tolist()})")
    return nbad == 0 and finite


def run_elementwise():
    import torch
    from naturalspeech2_pytorch_b200 import _lib, ops
    torch.manual_seed(0)
    dev = "cuda"
    ok = True
    B, N, D = 3, 200, 512
    x = torch.randn(B, N, D, device=dev)
    film = torch.randn(B, 4 * D, device=dev)
    gamma = torch.randn(D, device=dev)
    out = torch.empty(B, N, D, device=dev, dtype=torch.bfloat16)
    ops.rmsnorm_film(x, out, film=film[:, D:3 * D])
    ref = torch.nn.functional.normalize(x, dim=-1) * D ** 0.5 * film[:, None, D:2 * D] + film[:, None, 2 * D:3 * D]
    ok &= _report("rmsnorm_film(film)", out, ref, 2e-2, 1e-2)
    ops.rmsnorm_film(x, out, gamma=gamma)
    ok &= _report("rmsnorm_film(gamma)", out, torch.nn.functional.normalize(x, dim=-1) * D ** 0.5 * gamma, 2e-2, 1e-2)
    o32 = torch.empty(B, N, D, device=dev)
    ops.rmsnorm_f32(x, o32, gamma)
    ok &= _report("rmsnorm_f32", o32, torch.nn.functional.normalize(x, dim=-1) * D ** 0.5 * gamma, 1e-5, 1e-5)
    for D2 in (128, 512):
        half = D2 // 2
        times = torch.rand(5, device=dev)
        freqs = torch.randn(half, device=dev)
        W = torch.randn(4 * D2, D2 + 1, device=dev) / math.sqrt(D2)
        bias = torch.randn(4 * D2, device=dev)
        t_out = torch.empty(5, 8 * D2, device=dev)
        ops.time_cond(times, freqs, W, bias, t_out[:, :4 * D2])
        fr = times[:, None] * freqs[None] * 2 * math.pi
        feat = torch.cat((times[:, None], fr.sin(), fr.cos()), dim=-1)
        ref = torch.nn.functional.silu(feat.double() @ W.double().T + bias.double()).float()
        ok &= _report(f"time_cond(D={D2})", t_out[:, :4 * D2], ref, 2e-4, 1e-4)
    xs = torch.randn(7, 512, device=dev)
    W = torch.randn(2048, 512, device=dev) / 20
    b = torch.randn(2048, device=dev)
    o = torch.empty(7, 2048, device=dev)
    ops.small_linear(xs, W, b, o, act=1)
    ok &= _report("small_linear+silu", o, torch.nn.functional.silu(xs.double() @ W.double().T + b.double()).float(), 1e-4, 1e-4)
    add = torch.randn_like(x)
    cb = torch.empty(B, N, D, device=dev, dtype=torch.bfloat16)
    ops.cast_bf16(x, cb, add=add)
    ok &= _report("cast_bf16(add)", cb, (x + add).bfloat16(), 0, 0)
    m = torch.empty(B, D, device=dev)
    ops.mean_rows(x, m)
    ok &= _report("mean_rows", m, x.mean(dim=1), 1e-5, 1e-5)
    xc = torch.randn(2, 80, 333, device=dev)
    tc = torch.empty(2, 333, 80, device=dev, dtype=torch.bfloat16)
    ops.transpose_cast(xc, tc)
    ok &= _report("transpose_cast", tc, xc.transpose(1, 2).bfloat16(), 0, 0)
    x0, noise = torch.randn(B, N, D, device=dev), torch.randn(B, N, D, device=dev)
    alpha, sigma = torch.rand(B, device=dev), torch.rand(B, device=dev)
    xt, tg = torch.empty_like(x0), torch.empty_like(x0)
    ops.q_sample(x0, noise, alpha, sigma, xt, tg)
    a, s = alpha[:, None, None], sigma[:, None, None]
    ok &= _report("q_sample.x_t", xt, a * x0 + s * noise, 1e-6, 1e-6)
    ok &= _report("q_sample.target", tg, a * noise - s * x0, 1e-6, 1e-6)
    mo = torch.empty(B, device=dev)
    ops.mse_rows(xt, tg, mo)
    ok &= _report("mse_rows", mo, ((xt - tg) ** 2).mean(dim=(1, 2)), 1e-5, 1e-5)
    an, sn = torch.rand(B, device=dev), torch.rand(B, device=dev)
    xx = x0.clone()
    ops.ddim_step(xx, noise, alpha, sigma, an, sn)
    xs0 = a * x0 - s * noise
    eps = (x0 - a * xs0) / s.clamp(min=1e-10)
    ok &= _report("ddim_step", xx, xs0 * an[:, None, None] + eps * sn[:, None, None], 1e-5, 1e-5)
    oc = torch.empty_like(x0)
    ops.cfg_combine(x0, noise, 3.0, oc)
    ok &= _report("cfg_combine", oc, noise + (x0 - noise) * 3.0, 1e-6, 1e-6)
    return ok


def _gemm_ref(a, w, bias=None):
    r = a.float() @ w.float().T
    return r if bias is None else r + bias


def run_gemm_plain():
    import torch
    from naturalspeech2_pytorch_b200 import _lib, ops
    torch.manual_seed(1)
    dev = "cuda"
    ok = True
    cases = [  # (B, N, K, n, epilogue)
        (1, 128, 64, 128, ops.EPI_F32),
        (1, 128, 128, 128, ops.EPI_F32),
        (2, 256, 512, 512, ops.EPI_BF16),
        (2, 256, 512, 1536, ops.EPI_BF16),
        (3, 200, 512, 512, ops.EPI_F32),
        (2, 384, 1408, 512, ops.EPI_F32),
        (1, 32, 2048, 4096, ops.EPI_F32),
        (4, 1024, 512, 1408, ops.EPI_BF16),
        (2, 1024, 128, 128, ops.EPI_BF16),
    ]
    for (B, N, K, n, epi) in cases:
        a = (torch.randn(B, N, K, device=dev) * 0.5).bfloat16()
        w = (torch.randn(n, K, device=dev) / math.sqrt(K)).bfloat16()
        bias = torch.randn(n, device=dev)
        ref = _gemm_ref(a, w, bias)
        if epi == ops.EPI_F32:
            resid = torch.randn(B, N, n, device=dev)
            out = torch.full((B, N, n), float("nan"), device=dev)
            ops.gemm(a, w, out, n=n, epilogue=epi, bias=bias, resid=resid)
            ok &= _report(f"gemm f32+resid B{B} N{N} K{K} n{n}", out, ref + resid, 2e-3, 1e-3)
            # in-place residual (out aliases resid), as the transformer layers use it
            ops.gemm(a, w, resid, n=n, epilogue=epi, bias=bias, resid=resid)
            ok &= _report(f"gemm f32 in-place resid B{B} N{N} K{K} n{n}", resid, out, 0, 0)
        else:
            out = torch.full((B, N, n), float("nan"), device=dev, dtype=torch.bfloat16)
            ops.gemm(a, w, out, n=n, epilogue=epi, bias=bias)
            ok &= _report(f"gemm bf16 B{B} N{N} K{K} n{n}", out, ref, 3e-2, 1e-2)
    # strided A view (column window of a wider buffer) and column-offset output
    a_full = (torch.randn(2, 256, 1024, device=dev) * 0.5).bfloat16()
    w = (torch.randn(512, 512, device=dev) / 22).bfloat16()
    out_full = torch.zeros(2, 256, 1024, device=dev, dtype=torch.bfloat16)
    ops.gemm(a_full[:, :, 512:], w, out_full[:, :, 512:], n=512, epilogue=ops.EPI_BF16)
    ok &= _report("gemm strided views", out_full[:, :, 512:], _gemm_ref(a_full[:, :, 512:], w), 3e-2, 1e-2)
    ok &= _report("gemm strided views (untouched half)", out_full[:, :, :512], torch.zeros_like(out_full[:, :, :512]), 0, 0)
    return ok


def _conv_ref(x, w, bias, dil):
    import torch
    # x: (B, N, C) ; w: (O, I, 3) ; causal dilated conv as in CausalConv1d
    xc = x.float().transpose(1, 2)
    xp = torch.nn.functional.pad(xc, (2 * dil, 0))
    y = torch.nn.functional.conv1d(xp, w.float(), bias, dilation=dil)
    return y.transpose(1, 2)


def run_gemm_conv():
    import torch
    from naturalspeech2_pytorch_b200 import _lib, ops
    torch.manual_seed(2)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = "cuda"
    ok = True
    for (B, N, Cc, O, dil) in [(2, 256, 128, 128, 1), (2, 512, 512, 512, 1), (2, 512, 512, 512, 4),
                              (2, 512, 512, 512, 128), (3, 200, 512, 512, 2), (2, 256, 1408, 1408, 1)]:
        x = (torch.randn(B, N, Cc, device=dev) * 0.5).bfloat16()
        w = (torch.randn(O, Cc, 3, device=dev) / math.sqrt(3 * Cc)).bfloat16()
        bias = torch.randn(O, device=dev)
        wp = torch.cat([w[:, :, t] for t in range(3)], dim=1).contiguous()  # (O, 3*C)
        out = torch.full((B, N, O), float("nan"), device=dev, dtype=torch.bfloat16)
        ops.gemm(x, wp, out, n=O, epilogue=ops.EPI_BF16, bias=bias, segs=ops.conv3_segs(Cc), dil=[dil])
        ok &= _report(f"conv3 B{B} N{N} C{Cc} O{O} dil{dil}", out, _conv_ref(x, w, bias, dil), 3e-2, 1e-2)
    return ok


def run_gemm_fused():
    import torch
    from naturalspeech2_pytorch_b200 import _lib, ops
    torch.manual_seed(3)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = "cuda"
    ok = True
    # ---- GEGLU: Linear(D -> 2*Di) + gelu(gate) * value, Di padded to a multiple of 128 ----
    for (B, N, D, Di) in [(2, 256, 512, 1365), (2, 128, 128, 341)]:
        Dp = (Di + 127) // 128 * 128
        x = (torch.randn(B, N, D, device=dev) * 0.7).bfloat16()
        W = (torch.randn(2 * Di, D, device=dev) / math.sqrt(D)).bfloat16()
        b = torch.randn(2 * Di, device=dev)
        Wv = torch.zeros(Dp, D, device=dev, dtype=torch.bfloat16); Wv[:Di] = W[:Di]
        Wg = torch.zeros(Dp, D, device=dev, dtype=torch.bfloat16); Wg[:Di] = W[Di:]
        bv = torch.zeros(Dp, device=dev); bv[:Di] = b[:Di]
        bg = torch.zeros(Dp, device=dev); bg[:Di] = b[Di:]
        Wp = torch.stack((Wv.view(-1, 128, D), Wg.view(-1, 128, D)), dim=1).reshape(2 * Dp, D).contiguous()
        bp = torch.stack((bv.view(-1, 128), bg.view(-1, 128)), dim=1).reshape(2 * Dp).contiguous()
        out = torch.full((B, N, Dp), float("nan"), device=dev, dtype=torch.bfloat16)
        ops.gemm(x, Wp, out, n=2 * Dp, epilogue=ops.EPI_GEGLU, bias=bp)
        h = x.float() @ W.float().T + b
        ref = torch.nn.functional.gelu(h[..., Di:]) * h[..., :Di]
        ok &= _report(f"geglu D{D} Di{Di}", out[..., :Di], ref, 3e-2, 1e-2)
        ok &= _report(f"geglu D{D} Di{Di} (pad cols zero)", out[..., Di:], torch.zeros_like(out[..., Di:]), 0, 0)
    # ---- wavenet block, up to 8 dilation groups in one launch ----
    # every tile is 128 positions x 128 channels holding both accumulators (dilated conv + res_conv) in registers.
    # (9, 1024, 512, 8): 2304 tiles = 17-18 per persistent CTA on 132 SMs: the smem ring wraps across many tiles
    for (B, N, D, G) in [(2, 512, 512, 8), (2, 256, 128, 8), (3, 200, 512, 3), (9, 1024, 512, 8)]:
        dils = [2 ** i for i in range(G)]
        x = (torch.randn(B, N, G * D, device=dev) * 0.5).bfloat16()  # group g reads columns [g*D, (g+1)*D)
        wc = (torch.randn(G, D, D, 3, device=dev) / math.sqrt(3 * D)).bfloat16()
        wr = (torch.randn(G, D, D, device=dev) / math.sqrt(D)).bfloat16()
        bc, br = torch.randn(G, D, device=dev), torch.randn(G, D, device=dev)
        film = torch.randn(B, G * 2 * D, device=dev)
        wp = torch.cat([wc[..., 0], wc[..., 1], wc[..., 2], wr], dim=2).reshape(G * D, 4 * D).contiguous()
        bias = torch.cat([bc.reshape(-1), br.reshape(-1)]).contiguous()
        out = torch.full((B, N, G * D), float("nan"), device=dev, dtype=torch.bfloat16)
        segs = ops.conv3_segs(D) + [(0, 3 * D, D, 0, 1)]
        ops.gemm(x, wp, out, n=D, epilogue=ops.EPI_WAVENET, bias=bias, bias1_off=G * D, segs=segs,
                 film=film, film_group_stride=2 * D, groups=G, a_group_col_stride=D,
                 b_group_row_stride=D, out_group_col_stride=D, dil=dils)
        refs = []
        for g in range(G):
            xg = x[:, :, g * D:(g + 1) * D]
            y = _conv_ref(xg, wc[g], bc[g], dils[g])
            gm = film[:, None, g * 2 * D:g * 2 * D + D]
            bt = film[:, None, g * 2 * D + D:(g + 1) * 2 * D]
            y = y * gm + bt
            y = y.tanh() * y.sigmoid()
            refs.append(y + xg.float() @ wr[g].float().T + br[g])
        ok &= _report(f"wavenet block B{B} N{N} D{D} G{G}", out, torch.cat(refs, dim=-1), 3e-2, 1e-2)
    return ok


def _attn_ref(q, k, v, B, H, Nq, inner):
    import torch
    qf, kf, vf = (t.float().reshape(B, -1, H, 64).transpose(1, 2) for t in (q, k, v))
    sim = (qf @ kf.transpose(-1, -2)) * 64 ** -0.5
    return (sim.softmax(dim=-1) @ vf).transpose(1, 2).reshape(B, Nq, inner)


def run_attn():
    # every NS2_ATTN_* selector runs the same kernel (tests/test_attention_edges_gpu.py checks they are bit-identical),
    # so the shapes run once; timing lives in tools/attn_bench.py
    import torch
    from naturalspeech2_pytorch_b200 import _lib, ops
    torch.manual_seed(4)
    dev = "cuda"
    ok = True
    shapes = [(1, 1, 128, 128), (2, 8, 1024, 1024), (2, 8, 256, 32), (2, 8, 32, 135), (1, 2, 200, 300),
              (3, 4, 513, 700), (40, 8, 1024, 1024)]
    for (B, H, Nq, Nk) in shapes:
        inner = H * 64
        qkv = (torch.randn(B, max(Nq, Nk), 3 * inner, device=dev)).bfloat16()
        q = qkv[:, :Nq, :inner]
        k = qkv[:, :Nk, inner:2 * inner]
        v = qkv[:, :Nk, 2 * inner:]
        out = torch.full((B, Nq, inner), float("nan"), device=dev, dtype=torch.bfloat16)
        ops.attention(q, k, v, out, heads=H)
        ok &= _report(f"attn B{B} H{H} Nq{Nq} Nk{Nk}", out, _attn_ref(q, k, v, B, H, Nq, inner), 2e-2, 2e-2)
    # adversarial for the online softmax: score magnitudes grow along the key axis (the row maximum moves by far more
    # than 2^8 from tile to tile), a few rows with huge negative scores, and one sample with all-equal scores
    B, H, Nq, Nk = 2, 2, 384, 640
    inner = H * 64
    q = torch.randn(B, Nq, inner, device=dev)
    k = torch.randn(B, Nk, inner, device=dev) * torch.linspace(0.2, 12.0, Nk, device=dev)[None, :, None]
    k[:, ::7] *= -1.0
    q[1, :64] = 0.0
    v = torch.randn(B, Nk, inner, device=dev)
    q, k, v = q.bfloat16(), k.bfloat16(), v.bfloat16()
    out = torch.full((B, Nq, inner), float("nan"), device=dev, dtype=torch.bfloat16)
    ops.attention(q, k, v, out, heads=H)
    ok &= _report("attn growing-max", out, _attn_ref(q, k, v, B, H, Nq, inner), 3e-2, 3e-2)
    return ok


def run_rvq():
    import torch
    from naturalspeech2_pytorch_b200 import _lib, ops
    torch.manual_seed(5)
    dev = "cuda"
    ok = True
    for (F, Q, K, scale) in [(1000, 8, 1024, 1.0), (8192, 8, 1024, 1.0), (4096, 4, 256, 30.0)]:
        cb = torch.randn(Q, K, 128, device=dev) * scale
        cb[0, 7] = cb[0, 3]  # duplicate codeword: ties must resolve to the lowest index
        x = torch.randn(F, 128, device=dev) * scale
        x[:5] = cb[0, 7] + cb[1, 11]  # exact hits
        prep = ops.rvq_prepare(cb)
        stats = torch.zeros(_lib.NS2_RVQ_STATS_LEN, device=dev, dtype=torch.int64)
        codes = ops.rvq_encode(x, cb, prep, stats=stats)
        torch.cuda.synchronize()
        # fp64 oracle of the residual chain (fp32 residual updates, as in the reference)
        r = x.clone()
        ref = torch.empty(F, Q, dtype=torch.int64, device=dev)
        for qi in range(Q):
            d = ((r.double()[:, None, :] - cb[qi].double()[None]) ** 2).sum(-1) if F <= 1000 else \
                torch.cdist(r.double(), cb[qi].double()) ** 2
            idx = d.argmin(dim=1)
            ref[:, qi] = idx
            r = r - cb[qi][idx]
        mism = (codes != ref)
        nm = int(mism.sum())
        print(f"[{'OK ' if nm == 0 else 'BAD'}] rvq_encode F{F} Q{Q} K{K} scale{scale}: mismatches={nm}/{F * Q} "
              f"stats(lookups, near-ties, full scans, block scans)={stats[:4].tolist()}", flush=True)
        if nm:
            bad = mism.nonzero()[:8]
            for i in bad:
                print(f"      frame {int(i[0])} stage {int(i[1])}: got {int(codes[i[0], i[1]])} ref {int(ref[i[0], i[1]])}")
        ok &= nm == 0
        emb = ops.rvq_decode(codes, cb)
        ref_emb = torch.zeros(F, 128, device=dev)
        for qi in range(Q):
            ref_emb = ref_emb + cb[qi][codes[:, qi]]
        ok &= _report("rvq_decode", emb, ref_emb, 0, 0)
    return ok


def main():
    if len(sys.argv) >= 3 and sys.argv[1] == "--child":
        import torch
        torch.backends.cuda.matmul.allow_tf32 = False
        fn = globals()["run_" + sys.argv[2]]
        ok = fn()
        torch.cuda.synchronize()
        print("GROUP_RESULT", sys.argv[2], "PASS" if ok else "FAIL", flush=True)
        sys.exit(0 if ok else 1)
    groups = sys.argv[1:] or GROUPS
    outdir = ROOT / "gpurun_out"
    outdir.mkdir(exist_ok=True)
    summary = []
    for g in groups:
        t0 = time.time()
        log = outdir / f"check_{g}.log"
        try:
            res = subprocess.run([sys.executable, __file__, "--child", g], capture_output=True, text=True,
                                 timeout=float(os.environ.get("NS2_CHECK_TIMEOUT", "240")), cwd=str(ROOT))
            text = res.stdout + "\n--- stderr ---\n" + res.stderr[-6000:]
            status = "PASS" if res.returncode == 0 else f"FAIL(rc={res.returncode})"
        except subprocess.TimeoutExpired as e:
            text = (e.stdout or b"").decode(errors="replace") + "\n--- TIMEOUT ---\n" + (e.stderr or b"").decode(errors="replace")[-6000:]
            status = "TIMEOUT"
        log.write_text(text)
        summary.append((g, status, time.time() - t0))
        print(f"===== {g}: {status} ({time.time() - t0:.1f}s) =====")
        print(text[-5000:])
    print("SUMMARY " + " ".join(f"{g}={s}" for g, s, _ in summary))
    (outdir / "check_summary.txt").write_text("\n".join(f"{g} {s} {t:.1f}s" for g, s, t in summary) + "\n")


if __name__ == "__main__":
    main()
