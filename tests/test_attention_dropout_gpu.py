"""GPU: attention dropout in the flash forward / backward (`ops.attention(..., dropout=)`, `ops.attention_bwd(...,
dropout=)`) and the element-wise dropout (`ops.dropout_`) against the numpy restatement of their Philox streams
(tests/dropout_oracle.py) and float64 references of the masked computation.

The mask is read back exactly: with q = 0 every probability is 1 / kv_len, and with v one-hot over one 64-key block
O[i, j] = M[i, 64 blk + j] * scale / kv_len, so `O != 0` is the kernel's mask of that block.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

import dropout_oracle as do
from kernel_check import U_BF16, U_F32, acc_eps, assert_close, assert_rejects

pytestmark = pytest.mark.gpu
bf = torch.bfloat16
dev = "cuda"
LOG2E = 1.4426950408889634
RL2 = 2.0 ** -6
SEEDS = [0x9E37_79B9_7F4A_7C15, 0x0000_0001_0000_0000, 0xFFFF_FFFF_FFFF_FFFF, 0x1234_5678_0000_0042]


def _readback(B, H, Nq, Nk, drop):
    """The kernel's keep mask (B, H, Nq, Nk) from the one-hot runs, and whether every kept value is exactly
    bf16(float(scale) / kv_len)."""
    from naturalspeech2_pytorch_b200 import ops
    inner = H * 64
    q = torch.zeros(B, Nq, inner, device=dev, dtype=bf)
    k = torch.zeros(B, Nk, inner, device=dev, dtype=bf)
    mask = torch.zeros(B, H, Nq, Nk, dtype=torch.bool, device=dev)
    want = torch.tensor(float(np.float32(do.keep_scale(drop[2])) / np.float32(Nk)), dtype=torch.float32).to(bf)
    exact = True
    for blk in range((Nk + 63) // 64):
        n = min(64, Nk - 64 * blk)
        v = torch.zeros(B, Nk, H, 64, device=dev, dtype=bf)
        v[:, 64 * blk + torch.arange(n), :, torch.arange(n)] = 1.0
        o = torch.full((B, Nq, inner), float("nan"), device=dev, dtype=bf)
        ops.attention(q, k, v.view(B, Nk, inner), o, heads=H, dropout=drop)
        o = o.view(B, Nq, H, 64).transpose(1, 2)[..., :n]
        mask[..., 64 * blk:64 * blk + n] = o != 0
        exact &= bool(((o == 0) | (o == want.to(dev))).all())
    return mask.cpu().numpy(), exact


LENS = [1, 63, 65, 128, 129, 300]
READBACK = [(nq, nk) for nq in LENS for nk in LENS]


@pytest.mark.parametrize("Nq,Nk", READBACK)
def test_mask_read_back_bit_exactly(Nq, Nk):
    i = READBACK.index((Nq, Nk))
    H, B = (1, 8)[i % 2], (1, 3)[(i // 2) % 2]
    p = (0.1, 0.2, 0.5, 0.9)[i % 4]
    seed, site = SEEDS[i % len(SEEDS)], (0, 5)[(i // 3) % 2]
    got, exact = _readback(B, H, Nq, Nk, (seed, site, p))
    ref = do.attention_mask(seed, site, p, B, H, Nq, Nk)
    assert np.array_equal(got, ref), f"{int((got != ref).sum())} of {ref.size} keep bits differ"
    assert exact, "kept outputs must be exactly bf16(scale / kv_len)"


# ---- forward / backward against float64 ----
def _inputs(B, H, Nq, Nk, seed):
    inner = H * 64
    g = torch.Generator(device=dev).manual_seed(seed)
    qkv = torch.randn(B, max(Nq, Nk), 3 * inner, device=dev, generator=g).to(bf)
    do_full = torch.randn(B, Nq, inner + 64, device=dev, generator=g).to(bf)
    return qkv[:, :Nq, :inner], qkv[:, :Nk, inner:2 * inner], qkv[:, :Nk, 2 * inner:], do_full[..., :inner]


def _heads(t, B, H):
    return t.double().reshape(B, t.shape[1], H, 64).transpose(1, 2)


def _merge(t):
    B, H, N, _ = t.shape
    return t.transpose(1, 2).reshape(B, N, H * 64)


def reference(q, k, v, d_o, H, scale, ms):
    """float64 o and lse of (softmax(q k^T scale) * ms) v (ms = keep * 1 / (1 - p)), and the error terms of the kernels'
    arithmetic (those of test_attention_edges_gpu.py with the mask applied)."""
    B = q.shape[0]
    qh, kh, vh, doh = (_heads(t, B, H) for t in (q, k, v, d_o))
    s = qh @ kh.transpose(-1, -2) * scale
    p = torch.softmax(s, dim=-1)
    o = (p * ms) @ vh
    lse = torch.logsumexp(s, dim=-1) * LOG2E
    nq, nk = qh.shape[2], kh.shape[2]
    ds = acc_eps(64) * (qh.abs() @ kh.abs().transpose(-1, -2)).amax(-1) * abs(scale) * LOG2E
    dlse = ds + acc_eps(nk) * LOG2E + 2.0 ** -18 * (1.0 + lse.abs())
    ep = 2.0 ** -9 + math.log(2.0) * (ds + dlse)
    pm = p * ms
    b_o = 2 * (ep[..., None] + acc_eps(nk)) * (pm @ vh.abs() + o.abs()) + U_BF16 * o.abs()
    dp = (doh @ vh.transpose(-1, -2)) * ms
    D = (doh * o).sum(-1, keepdim=True)
    dS = p * (dp - D)
    dD = (U_BF16 + acc_eps(64)) * (doh.abs() * o.abs()).sum(-1, keepdim=True)
    e_p = ep[..., None] * p
    e_dS = (e_p * (dp - D).abs() + p * (acc_eps(64) * (doh.abs() @ vh.abs().transpose(-1, -2)) * ms + dD)
            + 2.0 ** -9 * dS.abs()) * abs(scale)
    return dict(o=_merge(o), lse=lse, b_o=_merge(b_o), b_lse=dlse, e_dS=e_dS, e_p=e_p, pm=pm, dS=dS, nq=nq, nk=nk)


def grads_reference(q, k, v, d_o, H, scale, ms):
    """reference() plus dq, dk, dv by float64 autograd of the masked attention, and their bounds."""
    B = q.shape[0]
    qh, kh, vh = (_heads(t, B, H).requires_grad_(True) for t in (q, k, v))
    doh = _heads(d_o, B, H)
    o = (torch.softmax(qh @ kh.transpose(-1, -2) * scale, dim=-1) * ms) @ vh
    o.backward(doh)
    r = reference(q, k, v, d_o, H, scale, ms)
    e_dS, e_p, pm, dS = r["e_dS"], r["e_p"], r["pm"], r["dS"]
    qa, ka, da = qh.detach().abs(), kh.detach().abs(), doh.abs()
    dq, dk, dv = qh.grad, kh.grad, vh.grad
    nq, nk = r["nq"], r["nk"]
    b_dv = 2 * ((e_p * ms).transpose(-1, -2) @ da + acc_eps(nq) * (pm.transpose(-1, -2) @ da)) + U_BF16 * dv.abs()
    b_dk = 2 * (e_dS.transpose(-1, -2) @ qa + acc_eps(nq) * (dS.abs().transpose(-1, -2) @ qa) * abs(scale)) \
        + U_BF16 * dk.abs()
    b_dq = 2 * (e_dS @ ka + acc_eps(nk) * (dS.abs() @ ka) * abs(scale))
    r.update(dq=_merge(dq), dk=_merge(dk), dv=_merge(dv), b_dq=_merge(b_dq), b_dk=_merge(b_dk), b_dv=_merge(b_dv))
    return r


def _run(q, k, v, d_o, H, drop, dq_start=None):
    from naturalspeech2_pytorch_b200 import ops
    B, Nq, inner = q.shape
    Nk = k.shape[1]
    o = torch.full((B, Nq, inner), float("nan"), device=dev, dtype=bf)
    lse = torch.full((B, H, Nq), float("nan"), device=dev)
    ops.attention(q, k, v, o, heads=H, lse=lse, dropout=drop)
    dq = torch.zeros(B, Nq, inner, device=dev) if dq_start is None else dq_start.clone()
    dk_full = torch.full((B, Nk, inner + 64), float("nan"), device=dev, dtype=bf)
    dv_full = torch.full((B, Nk, inner + 64), float("nan"), device=dev, dtype=bf)
    ops.attention_bwd(q, k, v, o, d_o, lse, dq, dk_full[..., :inner], dv_full[..., :inner], heads=H, dropout=drop)
    assert bool(torch.isnan(dk_full[..., inner:].float()).all() and torch.isnan(dv_full[..., inner:].float()).all())
    return dict(o=o, lse=lse, dq=dq, dk=dk_full[..., :inner], dv=dv_full[..., :inner])


def _ms(drop, B, H, Nq, Nk):
    return do.mask_tensor(do.attention_mask(*drop, B, H, Nq, Nk), drop[2]).to(dev)


SHAPES = [
    (1, 2, 1, 300),       # q_len = 1 over three key tiles
    (2, 4, 64, 129),      # last key tile holds one valid key
    (2, 2, 65, 128),      # ragged query tiles
    (3, 3, 513, 385),     # ragged in both
    (2, 8, 1024, 1024),   # the benchmarked attention shape
]


@pytest.mark.parametrize("p", [0.2, 0.5])
@pytest.mark.parametrize("B,H,Nq,Nk", SHAPES)
def test_attention_dropout_fwd_bwd(B, H, Nq, Nk, p):
    from naturalspeech2_pytorch_b200 import ops
    q, k, v, d_o = _inputs(B, H, Nq, Nk, seed=B * 1000 + Nq + Nk)
    drop = (SEEDS[(Nq + Nk) % len(SEEDS)], 3, p)
    dq_start = torch.randn(B, Nq, H * 64, device=dev, generator=torch.Generator(device=dev).manual_seed(1))
    got = _run(q, k, v, d_o, H, drop, dq_start=dq_start)
    ref = grads_reference(q, k, v, d_o, H, 64 ** -0.5, _ms(drop, B, H, Nq, Nk))
    what = f"B{B} H{H} Nq{Nq} Nk{Nk} p{p}"
    assert_close(got["o"], ref["o"], ref["b_o"], RL2, f"{what} o")
    plain_lse = torch.full((B, H, Nq), float("nan"), device=dev)
    ops.attention(q, k, v, torch.empty_like(got["o"]), heads=H, lse=plain_lse)
    assert torch.equal(got["lse"], plain_lse), "lse must be that of the undropped probabilities, bit for bit"
    dq = got["dq"].double() - dq_start.double()
    b_dq = ref["b_dq"] + U_F32 * (got["dq"].double().abs() + dq_start.double().abs())
    assert_close(dq, ref["dq"], b_dq, RL2, f"{what} dq")
    assert_close(got["dk"], ref["dk"], ref["b_dk"], RL2, f"{what} dk")
    assert_close(got["dv"], ref["dv"], ref["b_dv"], RL2, f"{what} dv")


def test_attention_dropout_qkv_windows():
    """q / k / v as column windows of one fused projection and d_o as a window of a wider buffer (the encoders' layout)
    are what _inputs builds; here additionally k / v come from a different batch stride than q."""
    B, H, Nq, Nk = 2, 4, 200, 300
    q, _, _, d_o = _inputs(B, H, Nq, Nk, seed=21)
    kv = torch.randn(B, Nk + 5, 2 * H * 64 + 64, device=dev, generator=torch.Generator(device=dev).manual_seed(2)).to(bf)
    k, v = kv[:, :Nk, :H * 64], kv[:, :Nk, H * 64 + 64:]
    drop = (SEEDS[0], 9, 0.3)
    got = _run(q, k, v, d_o, H, drop)
    ref = grads_reference(q, k, v, d_o, H, 64 ** -0.5, _ms(drop, B, H, Nq, Nk))
    for n in ("o", "dq", "dk", "dv"):
        assert_close(got[n], ref[n], ref["b_" + n], RL2, f"windows {n}")


def test_sensitivity_shifted_mask_and_wrong_site():
    """The bounds reject a reference whose mask is shifted by one key or drawn for site + 1."""
    B, H, Nq, Nk = 2, 4, 130, 200
    q, k, v, d_o = _inputs(B, H, Nq, Nk, seed=33)
    drop = (SEEDS[1], 2, 0.2)
    got = _run(q, k, v, d_o, H, drop)
    ref = grads_reference(q, k, v, d_o, H, 64 ** -0.5, _ms(drop, B, H, Nq, Nk))
    for n in ("o", "dq", "dk", "dv"):
        assert_close(got[n], ref[n], ref["b_" + n], RL2, f"exact {n}")
    shifted = torch.roll(_ms(drop, B, H, Nq, Nk), 1, dims=-1)
    other = _ms((drop[0], drop[1] + 1, drop[2]), B, H, Nq, Nk)
    for name, ms in (("mask shifted by one key", shifted), ("site + 1", other)):
        wrong = grads_reference(q, k, v, d_o, H, 64 ** -0.5, ms)
        for n in ("o", "dq", "dk", "dv"):
            assert_rejects(got[n], wrong[n], ref["b_" + n], RL2, f"{name}: {n}")


def _raw_calls(q, k, v, o, d_o, lse, dq, dk, dv, H, drop):
    """ns2_attn_fwd / ns2_attn_bwd called directly with the dropout field set (ops passes NULL for p = 0)."""
    from naturalspeech2_pytorch_b200 import _lib
    lib = _lib.load()
    stream = torch.cuda.current_stream().cuda_stream
    a = _lib.AttnArgs()
    a.q, a.q_row_stride, a.q_batch_stride = q.data_ptr(), q.stride(1), q.stride(0)
    a.k, a.k_row_stride, a.k_batch_stride = k.data_ptr(), k.stride(1), k.stride(0)
    a.v, a.v_row_stride, a.v_batch_stride = v.data_ptr(), v.stride(1), v.stride(0)
    a.out, a.o_row_stride, a.o_batch_stride = o.data_ptr(), o.stride(1), o.stride(0)
    a.batches, a.heads, a.q_len, a.kv_len, a.dim_head, a.scale = q.shape[0], H, q.shape[1], k.shape[1], 64, 0.125
    a.lse = lse.data_ptr()
    d = _lib.Dropout(*drop)
    a.dropout = ctypes.pointer(d)
    _lib.check(lib.ns2_attn_fwd(ctypes.byref(a), stream), "ns2_attn_fwd")
    g = _lib.AttnBwdArgs()
    for n, t in (("q", q), ("k", k), ("v", v), ("o", o), ("d_o", d_o)):
        setattr(g, n, t.data_ptr())
    g.q_row_stride, g.q_batch_stride = q.stride(1), q.stride(0)
    g.k_row_stride, g.k_batch_stride = k.stride(1), k.stride(0)
    g.v_row_stride, g.v_batch_stride = v.stride(1), v.stride(0)
    g.o_row_stride, g.o_batch_stride = o.stride(1), o.stride(0)
    g.do_row_stride, g.do_batch_stride = d_o.stride(1), d_o.stride(0)
    delta = torch.empty(q.shape[0], H, q.shape[1], device=dev)
    g.lse, g.delta, g.dq_accum = lse.data_ptr(), delta.data_ptr(), dq.data_ptr()
    g.dk, g.dk_row_stride, g.dk_batch_stride = dk.data_ptr(), dk.stride(1), dk.stride(0)
    g.dv, g.dv_row_stride, g.dv_batch_stride = dv.data_ptr(), dv.stride(1), dv.stride(0)
    g.batches, g.heads, g.q_len, g.kv_len, g.dim_head, g.scale = q.shape[0], H, q.shape[1], k.shape[1], 64, 0.125
    g.dropout = ctypes.pointer(d)
    _lib.check(lib.ns2_attn_bwd(ctypes.byref(g), stream), "ns2_attn_bwd")


def test_p0_entry_points_bit_identical_and_repeatable():
    """dropout p = 0 = no dropout, bit for bit; the same dropout arguments twice = the same bits."""
    B, H, Nq, Nk = 2, 4, 300, 257
    q, k, v, d_o = _inputs(B, H, Nq, Nk, seed=8)
    plain = _run(q, k, v, d_o, H, None)
    outs = {}
    for name, drop in (("raw p0", (SEEDS[2], 1, 0.0)), ("ops p0", (SEEDS[2], 1, 0.0))):
        o = torch.empty_like(plain["o"])
        lse = torch.empty_like(plain["lse"])
        dq = torch.zeros_like(plain["dq"])
        dk, dv = torch.empty_like(plain["dk"]), torch.empty_like(plain["dv"])
        if name == "raw p0":
            _raw_calls(q, k, v, o, d_o, lse, dq, dk, dv, H, drop)
        else:
            r = _run(q, k, v, d_o, H, drop)
            o, lse, dq, dk, dv = r["o"], r["lse"], r["dq"], r["dk"], r["dv"]
        outs[name] = dict(o=o, lse=lse, dq=dq, dk=dk, dv=dv)
    for name, r in outs.items():
        for n in ("o", "lse", "dk", "dv"):
            assert torch.equal(r[n], plain[n]), f"{name}: {n}"
        ref = grads_reference(q, k, v, d_o, H, 64 ** -0.5, torch.ones(1, device=dev, dtype=torch.float64))
        assert_close(r["dq"], plain["dq"], 2 * ref["b_dq"], RL2, f"{name}: dq (fp32 atomics)")
    drop = (SEEDS[3], 4, 0.4)
    a, b = _run(q, k, v, d_o, H, drop), _run(q, k, v, d_o, H, drop)
    for n in ("o", "lse", "dk", "dv"):
        assert torch.equal(a[n], b[n]), n


def test_mask_statistics():
    """Keep fraction within 6 sigma of 1 - p over 10.5M elements; adjacent (q, k + 8) / (q + 8, k) / (q, k + 1) pairs
    keep together at ~(1 - p)^2; other (b, h), site or seed give other masks."""
    B, H, Nq, Nk, p = 2, 10, 8192, 64, 0.3
    seed = SEEDS[0]
    m, exact = _readback(B, H, Nq, Nk, (seed, 6, p))
    assert exact
    n = m.size
    frac = m.mean()
    assert abs(frac - (1 - p)) < 6 * math.sqrt(p * (1 - p) / n), frac
    for name, a, b in (("k+8", m[..., :, 0:8], m[..., :, 8:16]), ("q+8", m[..., 0:8, :], m[..., 8:16, :]),
                       ("k+1", m[..., :, 0:63], m[..., :, 1:64])):
        both = (a & b).mean()
        assert abs(both - (1 - p) ** 2) < 6 * math.sqrt((1 - p) ** 2 * (1 - (1 - p) ** 2) / a.size), (name, both)
    assert not np.array_equal(m[0, 0], m[0, 1]) and not np.array_equal(m[0, 0], m[1, 0])
    m2, _ = _readback(1, 1, 256, 64, (seed, 7, p))
    m3, _ = _readback(1, 1, 256, 64, (seed ^ (1 << 40), 6, p))
    assert (m2 != m[0, 0, :256]).mean() > 0.3 and (m3 != m[0, 0, :256]).mean() > 0.3


# ---- element-wise ----
@pytest.mark.parametrize("n", [1, 3, 4, 5, 4097, 2 ** 20 + 3])
def test_dropout_f32_bit_exact(n):
    from naturalspeech2_pytorch_b200 import ops
    seed, site, p = SEEDS[n % len(SEEDS)], 11, 0.35
    x = torch.randn(n, device=dev, generator=torch.Generator(device=dev).manual_seed(n))
    buf = torch.full((n + 8,), float("nan"), device=dev)
    buf[:n] = x
    ops.dropout_(buf[:n], dropout=(seed, site, p))
    keep = torch.from_numpy(do.elementwise_mask(seed, site, p, n)).to(dev)
    want = x * keep.float() * float(do.keep_scale(p))
    assert torch.equal(buf[:n], want)
    assert bool(torch.isnan(buf[n:]).all()), "elements past n were written"
    same = x.clone()
    ops.dropout_(same, dropout=(seed, site, 0.0))
    assert torch.equal(same, x)


def test_dropout_f32_statistics():
    from naturalspeech2_pytorch_b200 import ops
    n, p = 10_000_000, 0.2
    x = torch.ones(n, device=dev)
    ops.dropout_(x, dropout=(SEEDS[0], 0, p))
    frac = float((x != 0).double().mean())
    assert abs(frac - (1 - p)) < 6 * math.sqrt(p * (1 - p) / n), frac
    assert bool((x[x != 0] == float(do.keep_scale(p))).all())
