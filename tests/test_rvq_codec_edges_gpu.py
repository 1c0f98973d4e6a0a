"""GPU: the RVQ cross-entropy forward (ns2_rvq_ce), the codeword decode (ns2_rvq_decode), the codebook preparation
(ns2_rvq_prepare) and the mean-pool gradient broadcast (ns2_add_rows_bcast) at their edges against float64 references.

ns2_rvq_ce is called through the C ABI with a caller-owned scratch of F*Q + 64 floats filled with NaN, so every
(frame, stage) CE value is checked, not only the loss, and a write past F*Q shows.  Its tiling has these edges:
32 frames per CTA as 8 warps x 4 frames (F % 32, F % 4); 128-code shared-memory chunks where lane cg scores codes
cg + 32 b (K < 128 leaves most lanes without a code in slots b >= 1, K % 128 != 0 a partial last chunk); an online
log-sum-exp per lane merged by warp shuffles; and a one-CTA reduce that counts the valid targets in fp32.  Own codes
come from ns2_rvq_encode when K % 128 == 0 and from the fp64 argmin otherwise (the encoder needs K % 128 == 0).

Bound (the protocol of test_rvq_ce_backward_gpu.py): per entry, |ours - fp64| <= ERR_MULT * max|fp32 - fp64| +
2^-16 max|fp64|, and rel-L2 <= ERR_MULT * rel-L2(fp32) + 1e-6, where fp32 is the same expanded-distance formula
(||r||^2 - 2 r.c + ||c||^2, clamped at 0) run by torch in fp32 on the kernel's fp32 residual chain.  The loss bound
is ERR_MULT * |loss32 - loss64| + 2^-16 |loss64| plus the reduce's fp32 sums, sum_q acc_eps(F) * sum_f |ce| / count_q.
The fp64 loss is rvq_ce_restatement.residual_vq_ce's (frame chunks of the same formula for the 2^18 + 5 frame case).
Four wrong references must fail these bounds: a residual chain that never advances, targets shifted by one code, a
mean over all frames instead of those with a valid target (loss only: the entries are the same), and -d^2 logits.

Measured on an H100 80GB HBM3 (700 W power limit); each test prints its numbers under `pytest -s`.  ERR_MULT: the
kernel's worst max|ours - fp64| / max|fp32 - fp64| is 2.14 (F 4, Q 1, K 1000) over every case with two or more
entries, 1.43 (logit spread) and 1.12 (targets at 0, 127, 128, K - 1 with K 129) among the special inputs, 0.96 at
2^18 + 5 frames.  A single entry's fp32 error can be near zero by chance (F 1, Q 1, K 2048: 1.1e4 x it); the floor
covers that case, at 1% of its bound.  Tightest use of a bound: 17% (frames on a codeword, whose d^2 clamps to 0 with
rounding noise that is large next to the distance), otherwise 3% or less; the loss uses at most 10% of its bound.
The wrong references fail by at least 1.8e4 x the entry bound and 1.8e3 x the loss bound (the chain that never
advances), 2.9e3 x the loss bound for the mean over all frames.  The module runs in about 26 s.

ns2_rvq_decode is bit-exact against the in-order fp32 sum, including its clamp of out-of-range codes.  ns2_rvq_prepare:
||c||^2 within acc_eps(128) of fp64, max ||c|| (inflated by 1.0001, so it bounds the fp32 norms from above), the
power-of-two scale 2^e with max|c| < 2^e <= 2 max|c|, and the fp16 copy fp16(c / 2^e) compared chunk by chunk as sorted
sets of rows (the codes are permuted inside each 128-code chunk).  ns2_add_rows_bcast is one fp32 fma per element:
exact against the fp64 value rounded once.
"""
import math

import numpy as np
import pytest
import torch

from kernel_check import acc_eps, assert_close, assert_nan, assert_rejects, gen as _gen, nan_buf as _nan_buf, sm_limit
from rvq_ce_restatement import residual_vq_ce

pytestmark = pytest.mark.gpu
dev = "cuda"
NAN = float("nan")
ERR_MULT = 4.0    # measured worst 2.14 (module docstring)
FLOOR = 2.0 ** -16
CHUNK = 1 << 15   # frames per block of the reference: a (CHUNK, K) fp64 logit matrix at a time


# ---------------------------------------------------------------------------------------------------------------
# ns2_rvq_ce
# ---------------------------------------------------------------------------------------------------------------
def _ce_entries(x, cb, own, tgt, dtype, *, advance=True, squared=False):
    """(F, Q) CE of every frame and stage in `dtype`, 0 where the target is -1: logits -||r_q - c_k|| by the expanded
    formula on the residual chain r_{q+1} = r_q - C_q[own_q], computed CHUNK frames at a time.  The sensitivity test's
    wrong variants: advance=False keeps r_q = x, squared=True uses -||r_q - c_k||^2 as the logits."""
    F, Q = own.shape
    cbd = cb.to(dtype)
    cn2 = (cbd * cbd).sum(-1)
    out = torch.zeros(F, Q, dtype=dtype, device=x.device)
    for f0 in range(0, F, CHUNK):
        r = x[f0:f0 + CHUNK].to(dtype)
        for q in range(Q):
            d2 = ((r * r).sum(-1, keepdim=True) - 2.0 * (r @ cbd[q].t()) + cn2[q][None]).clamp_min(0.0)
            lg = -d2 if squared else -d2.sqrt()
            t = tgt[f0:f0 + CHUNK, q]
            ce = lg.logsumexp(-1) - lg.gather(1, t.clamp_min(0)[:, None])[:, 0]
            out[f0:f0 + CHUNK, q] = torch.where(t >= 0, ce, torch.zeros_like(ce))
            if advance:
                r = r - cbd[q][own[f0:f0 + CHUNK, q]]
    return out


def _loss(ce, tgt, *, all_frames=False):
    """sum_q mean over the frames with a valid target (NaN for a stage without one); all_frames=True is the wrong mean
    over every frame."""
    valid = (tgt >= 0).to(ce.dtype)
    count = torch.full_like(valid[0], tgt.shape[0]) if all_frames else valid.sum(0)
    return float(((ce * valid).sum(0) / count).sum())


def _own_codes(x, cb):
    """The residual chain's own codes: ns2_rvq_encode where it applies, else the fp64 argmin (first on ties)."""
    from naturalspeech2_pytorch_b200 import ops
    Q, K, _ = cb.shape
    if K % 128 == 0:
        return ops.rvq_encode(x, cb, ops.rvq_prepare(cb))
    own = torch.empty(x.shape[0], Q, dtype=torch.int64, device=x.device)
    cbd = cb.double()
    for f0 in range(0, x.shape[0], CHUNK):
        r = x[f0:f0 + CHUNK].double()
        for q in range(Q):
            own[f0:f0 + CHUNK, q] = torch.cdist(r, cbd[q]).argmin(-1)
            r = r - cbd[q][own[f0:f0 + CHUNK, q]]
    return own


def _cn2(cb):
    """||c||^2 as the codec hands it to the CE head: ns2_rvq_prepare's where it applies, else fp64 rounded once."""
    from naturalspeech2_pytorch_b200 import ops
    if cb.shape[1] % 128 == 0:
        return ops.rvq_prepare(cb)[1]
    return (cb.double() ** 2).sum(-1).float()


def _targets(own, K, g, *, ignored=0.1):
    """Half the targets are the own code, half random; a share `ignored` of them -1, in every stage."""
    F, Q = own.shape
    tgt = torch.randint(0, K, (F, Q), device=own.device, generator=g)
    tgt = torch.where(torch.rand(F, Q, device=own.device, generator=g) < 0.5, own, tgt)
    tgt[torch.rand(F, Q, device=own.device, generator=g) < ignored] = -1
    return tgt


def _launch_ce(x, cb, cn2, own, tgt):
    """ns2_rvq_ce with NaN-filled, caller-owned scratch (64 spare floats) and loss (1 spare float)."""
    from naturalspeech2_pytorch_b200 import _lib
    lib = _lib.load()
    F, Q = own.shape
    scratch = torch.full((F * Q + 64,), NAN, device=dev)
    loss = torch.full((2,), NAN, device=dev)
    rc = lib.ns2_rvq_ce(x.data_ptr(), F, 128, cb.data_ptr(), cn2.data_ptr(), Q, cb.shape[1], own.data_ptr(),
                        tgt.data_ptr(), scratch.data_ptr(), loss.data_ptr(), torch.cuda.current_stream().cuda_stream)
    _lib.check(rc, "ns2_rvq_ce")
    torch.cuda.synchronize()
    assert_nan(scratch[F * Q:], "scratch past F * Q")
    assert_nan(loss[1:], "past the loss")
    return scratch[:F * Q].view(F, Q), loss[0]


def _check_ce(x, cb, cn2, own, tgt, what, *, restated_loss=True):
    """Run the kernel and check every entry and the loss; returns what the sensitivity test needs."""
    got, loss = _launch_ce(x, cb, cn2, own, tgt)
    ce64 = _ce_entries(x, cb, own, tgt, torch.float64)
    ce32 = _ce_entries(x, cb, own, tgt, torch.float32).double()
    err32 = float((ce32 - ce64).abs().max())
    bound = ERR_MULT * err32 + FLOOR * float(ce64.abs().max())
    nref = float(ce64.norm())
    rel = ERR_MULT * (float((ce32 - ce64).norm()) / nref if nref > 0 else 0.0) + 1e-6
    assert_close(got, ce64, bound, rel, what)
    assert bool((got[tgt < 0] == 0).all()), f"{what}: an ignored target's entry is not 0"
    err = float((got.double() - ce64).abs().max())
    print(f"[rvq_ce] {what}: entries err/err32 {err / err32 if err32 else 0.0:.2f}, {err / bound:.0%} of the bound")

    F = tgt.shape[0]
    valid = tgt >= 0
    count = valid.sum(0)
    loss64 = _loss(ce64, tgt)
    if restated_loss:   # the per-entry restatement agrees with the one the CE-gradient tests use
        _, l_ref, _ = residual_vq_ce(x.double(), cb.double(), tgt, own=own)
        assert math.isclose(loss64, float(l_ref), rel_tol=1e-12) or (math.isnan(loss64) and math.isnan(float(l_ref)))
    if bool((count == 0).any()):
        assert math.isnan(float(loss)), f"{what}: a stage without a valid target gives a NaN loss, as torch does"
        lbound = None
    else:
        reduce_err = sum(acc_eps(F) * float(ce64[:, q].abs().sum()) / int(count[q]) for q in range(tgt.shape[1]))
        lbound = ERR_MULT * abs(_loss(ce32, tgt) - loss64) + FLOOR * abs(loss64) + reduce_err
        lerr = abs(float(loss) - loss64)
        assert lerr <= lbound, f"{what}: loss {float(loss)!r} vs fp64 {loss64!r}: error {lerr:.3e} > bound {lbound:.3e}"
        print(f"[rvq_ce] {what}: loss {lerr / lbound:.0%} of its bound")
    return dict(got=got, loss=float(loss), ce64=ce64, bound=bound, rel=rel, lbound=lbound)


def _problem(F, Q, K, seed):
    g = _gen(seed)
    cb = torch.randn(Q, K, 128, device=dev, generator=g)
    x = torch.randn(F, 128, device=dev, generator=g)
    return x, cb, g


@pytest.mark.parametrize("K", [32, 33, 100, 128, 129, 1000, 1024, 2048])
@pytest.mark.parametrize("Q", [1, 3, 8])
@pytest.mark.parametrize("F", [1, 3, 4, 31, 32, 33, 4097])
def test_rvq_ce_entries_and_loss_shapes(F, Q, K):
    x, cb, g = _problem(F, Q, K, seed=F * 7919 + Q * 131 + K)
    own = _own_codes(x, cb)
    tgt = _targets(own, K, g)
    empty = (tgt >= 0).sum(0) == 0   # a stage without a valid target is the NaN case, tested on its own
    tgt[:, empty] = own[:, empty]
    _check_ce(x, cb, _cn2(cb), own, tgt, f"F={F} Q={Q} K={K}")


def test_rvq_ce_large_frame_count_and_determinism():
    """2^18 + 5 frames (8193 CTAs, the last with 5 frames; a 262 149-frame fp32 reduce per stage), Q 8, K 1024; the
    fp64 reference in frame blocks.  Two launches are bit-identical (no atomics)."""
    F, Q, K = (1 << 18) + 5, 8, 1024
    x, cb, g = _problem(F, Q, K, seed=77)
    own = _own_codes(x, cb)
    tgt = _targets(own, K, g)
    cn2 = _cn2(cb)
    r = _check_ce(x, cb, cn2, own, tgt, f"F={F} Q={Q} K={K}", restated_loss=False)
    again, loss = _launch_ce(x, cb, cn2, own, tgt)
    assert torch.equal(again, r["got"]) and float(loss) == r["loss"], "two launches differ"


def _special(case):
    """(x, codebooks, own, targets) of one special input."""
    if case.startswith("chunk_edge_targets"):
        F, Q, K = 64, 3, int(case.split("K")[1])
        x, cb, g = _problem(F, Q, K, seed=K)
        own = _own_codes(x, cb)
        tgt = _targets(own, K, g)
        tgt[:, 1] = torch.tensor([0, 127, 128, K - 1], device=dev).repeat(F // 4)   # both sides of the chunk boundary
        return x, cb, own, tgt
    if case == "targets_are_own":
        x, cb, g = _problem(300, 8, 1024, seed=11)
        own = _own_codes(x, cb)
        return x, cb, own, own.clone()
    if case == "on_codeword":
        # frames exactly on a codeword of stage 0: d^2 clamps to 0 there and that logit is the largest
        x, cb, g = _problem(97, 3, 256, seed=12)
        x[:40] = cb[0, 3:43]
        own = _own_codes(x, cb)
        assert torch.equal(own[:40, 0], torch.arange(3, 43, device=dev))
        tgt = _targets(own, 256, g)
        tgt[:20, 0] = own[:20, 0]
        return x, cb, own, tgt
    if case == "logit_spread":
        # codeword norms over three decades: each frame's logits spread over more than 100, so exp underflows to 0
        # in the online softmax and in the shuffle merge
        Q, K = 2, 1000
        x, cb, g = _problem(129, Q, K, seed=13)
        cb = cb * torch.exp(torch.empty(Q, K, 1, device=dev).uniform_(math.log(0.05), math.log(40.0), generator=g))
        x = x * 3.0
        spread = torch.cdist(x.double(), cb[0].double())
        assert float((spread.amax(-1) - spread.amin(-1)).min()) > 100.0
        own = _own_codes(x, cb)
        return x, cb, own, _targets(own, K, g)
    if case == "degenerate":
        x, cb, g = _problem(300, 2, 256, seed=14)
        cb = cb[:, :1] + 1e-3 * torch.randn(2, 256, 128, device=dev, generator=g)
        own = _own_codes(x, cb)
        return x, cb, own, _targets(own, 256, g)
    if case == "large_magnitude":
        # x 50: ||r||^2 and ||c||^2 near 3e5 cancel in the expansion down to distances of a few hundred
        x, cb, g = _problem(200, 3, 256, seed=15)
        x, cb = x * 50.0, cb * 50.0
        own = _own_codes(x, cb)
        return x, cb, own, _targets(own, 256, g)
    raise ValueError(case)


@pytest.mark.parametrize("case", ["chunk_edge_targets_K129", "chunk_edge_targets_K1000", "chunk_edge_targets_K2048",
                                  "targets_are_own", "on_codeword", "logit_spread", "degenerate", "large_magnitude"])
def test_rvq_ce_special_inputs(case):
    x, cb, own, tgt = _special(case)
    r = _check_ce(x, cb, _cn2(cb), own, tgt, case)
    if case == "degenerate":   # a nearly flat softmax: every stage's CE is log K
        assert abs(r["loss"] - 2 * math.log(256)) < 1e-2, r["loss"]


def test_rvq_ce_all_ignored_stage():
    """Every target of stage 1 is -1: the loss is NaN (torch's mean over no frames), that stage's entries are exactly 0
    and the other stages' entries are finite and within the bound."""
    x, cb, g = _problem(200, 3, 256, seed=16)
    own = _own_codes(x, cb)
    tgt = _targets(own, 256, g)
    tgt[:, 1] = -1
    r = _check_ce(x, cb, _cn2(cb), own, tgt, "all-ignored stage")
    got = r["got"]
    assert math.isnan(r["loss"])
    assert bool((got[:, 1] == 0).all()) and bool(torch.isfinite(got).all())
    assert float(got[:, [0, 2]].abs().max()) > 0


def test_rvq_ce_bounds_reject_wrong_references():
    """Sensitivity: each wrong reference fails the bounds the kernel passes, on the entries (max-abs and rel-L2) where
    it changes them, and on the loss."""
    F, Q, K = 257, 3, 1000
    x, cb, g = _problem(F, Q, K, seed=17)
    own = _own_codes(x, cb)
    tgt = _targets(own, K, g)
    r = _check_ce(x, cb, _cn2(cb), own, tgt, "sensitivity baseline")
    got, loss, bound, rel, lbound = r["got"], r["loss"], r["bound"], r["rel"], r["lbound"]
    shifted = torch.where(tgt >= 0, (tgt + 1) % K, tgt)
    wrong = {
        "(a) chain never advances": _ce_entries(x, cb, own, tgt, torch.float64, advance=False),
        "(b) targets shifted by one code": _ce_entries(x, cb, own, shifted, torch.float64),
        "(d) logits -d^2": _ce_entries(x, cb, own, tgt, torch.float64, squared=True),
    }
    for what, ce in wrong.items():
        assert_rejects(got, ce, bound, rel, what)
        lw = _loss(ce, tgt)
        assert abs(loss - lw) > lbound, f"{what}: the loss bound accepts it"
        print(f"[rvq_ce] {what}: entries {float((got.double() - ce).abs().max()) / bound:.3g} x the bound, loss "
              f"{abs(loss - lw) / lbound:.3g} x")
    lw = _loss(r["ce64"], tgt, all_frames=True)
    assert abs(loss - lw) > lbound, "(c) mean over all frames: the loss bound accepts it"
    print(f"[rvq_ce] (c) mean over all frames: loss {abs(loss - lw) / lbound:.3g} x the bound")


def test_rvq_wrappers_reject_bad_arguments_before_launch():
    """On the GPU the wrappers reject what would make the kernels read past a buffer or through a host pointer: int32
    codes, codebooks or cn2 on the host, a misaligned output.  Nothing launches."""
    from naturalspeech2_pytorch_b200 import _lib, ops
    lib = _lib.load()
    cb = torch.randn(8, 128, 128, device=dev)
    before = lib.ns2_launch_count()
    with pytest.raises(ValueError, match="int64"):
        ops.rvq_decode(torch.zeros(4, 8, dtype=torch.int32, device=dev), cb)
    with pytest.raises(ValueError, match="codebooks must be a CUDA tensor"):
        ops.rvq_decode(torch.zeros(4, 8, dtype=torch.int64, device=dev), cb.cpu())
    flat = torch.empty(4 * 128 + 1, device=dev)
    with pytest.raises(ValueError, match="16-byte aligned"):
        ops.rvq_decode(torch.zeros(4, 8, dtype=torch.int64, device=dev), cb, out=flat[1:].view(4, 128))
    codes = torch.zeros(4, 8, dtype=torch.int64, device=dev)
    with pytest.raises(ValueError, match="cn2 must be a CUDA tensor"):
        ops.rvq_ce(torch.zeros(4, 128, device=dev), cb, torch.zeros(8, 128), codes, codes)
    assert lib.ns2_launch_count() == before


# ---------------------------------------------------------------------------------------------------------------
# ns2_rvq_decode
# ---------------------------------------------------------------------------------------------------------------
def _in_order_sum(cb, codes):
    acc = torch.zeros(codes.shape[0], 128, device=dev)
    for q in range(cb.shape[0]):
        acc = acc + cb[q][codes[:, q]]
    return acc


def _tail_codebooks(Q, K, g, pad=4096):
    """Codebooks at the very end of their allocation: a wrong stride or an unclamped code reads past it."""
    store = torch.randn(pad + Q * K * 128, device=dev, generator=g)
    return store[pad:].view(Q, K, 128)


@pytest.mark.parametrize("K", [128, 2048])
@pytest.mark.parametrize("Q", [1, 2, 8])
@pytest.mark.parametrize("F", [1, 7, 8, 9, 4097])
def test_rvq_decode_is_the_in_order_sum(F, Q, K):
    """8 frames per CTA (one warp each): F around it.  The last frame picks the last codeword of every stage; the
    output is a window of a NaN-filled buffer whose spare rows stay NaN."""
    from naturalspeech2_pytorch_b200 import EncodecRVQ, ops
    g = _gen(F * 31 + Q * 7 + K)
    cb = _tail_codebooks(Q, K, g)
    codes = torch.randint(0, K, (F, Q), device=dev, generator=g)
    codes[-1] = K - 1
    buf = torch.full((F + 3, 128), NAN, device=dev)
    got = ops.rvq_decode(codes, cb, out=buf[:F])
    assert got.data_ptr() == buf.data_ptr()
    assert torch.equal(got, _in_order_sum(cb, codes))
    assert_nan(buf[F:], "spare rows")
    codec = EncodecRVQ(cb.cpu()).cuda()   # the codec converts int32 codes before the wrapper sees them
    assert torch.equal(codec.get_emb_from_indices(codes.int().view(1, F, Q)), got.view(1, F, 128))


def test_rvq_decode_clamps_out_of_range_codes():
    """Documented in ns2_b200.h: a code < 0 reads codeword 0, a code >= K reads codeword K - 1."""
    from naturalspeech2_pytorch_b200 import ops
    Q, K = 3, 128
    g = _gen(5)
    cb = _tail_codebooks(Q, K, g)
    codes = torch.randint(0, K, (40, Q), device=dev, generator=g)
    codes[0] = -1
    codes[1] = K + 5
    codes[2] = K
    codes[3, 0], codes[3, 1], codes[3, 2] = -(1 << 40), 1 << 40, -7
    codes[4, Q - 1] = K + 5
    ref = _in_order_sum(cb, codes.clamp(0, K - 1))
    assert torch.equal(ops.rvq_decode(codes, cb), ref)


# ---------------------------------------------------------------------------------------------------------------
# ns2_rvq_prepare
# ---------------------------------------------------------------------------------------------------------------
def _sorted_rows(h):
    """(chunks, 128, 128) fp16 -> each chunk's rows sorted bytewise (a multiset of rows, independent of their order)."""
    a = np.ascontiguousarray(h.view(torch.int16).cpu().numpy())
    return np.sort(a.view(np.dtype((np.void, 256))), axis=1)


@pytest.mark.parametrize("K", [128, 256, 2048])
@pytest.mark.parametrize("Q", [1, 8])
def test_rvq_prepare_norms_scale_and_fp16_copy(Q, K):
    """Stage scales from 1e-3 to 300 (2^e from 2^-8 to 2^11); with Q = 8 stage 3 is all zero."""
    from naturalspeech2_pytorch_b200 import ops
    g = _gen(Q * 100 + K)
    scales = torch.tensor([1.0, 1e-3, 300.0, 0.3, 7.0, 0.02, 60.0, 1.5], device=dev)[:Q].view(Q, 1, 1)
    cb = torch.randn(Q, K, 128, device=dev, generator=g) * scales
    if Q > 1:
        cb[3] = 0.0
    cb16, cn2, meta = ops.rvq_prepare(cb)
    assert cb16.shape == (Q * K * 144,) and cn2.shape == (Q, K) and meta.shape == (Q, 2)

    n2 = (cb.double() ** 2).sum(-1)
    assert bool(((cn2.double() - n2).abs() <= acc_eps(128) * n2).all()), "||c||^2"
    nmax = n2.sqrt().amax(-1) * 1.0001
    assert bool(((meta[:, 0].double() - nmax).abs() <= acc_eps(128) * nmax).all()), "max ||c|| * 1.0001"
    assert bool((meta[:, 0].double() >= n2.sqrt().amax(-1)).all()), "meta[:, 0] bounds every norm from above"

    scale = meta[:, 1].double()
    mant, _ = torch.frexp(scale)
    assert bool((mant == 0.5).all()), f"meta[:, 1] is a power of two: {scale.tolist()}"
    amax = cb.abs().amax((1, 2)).double()
    ok = torch.where(amax > 0, (amax < scale) & (scale <= 2 * amax), scale == 1.0)
    assert bool(ok.all()), f"max|c| < 2^e <= 2 max|c| (2^e = 1 for an all-zero stage): {amax.tolist()} {scale.tolist()}"

    got = cb16[:Q * K * 128].view(Q * K // 128, 128, 128)
    ref = (cb / meta[:, 1].view(Q, 1, 1)).half().view(Q * K // 128, 128, 128)
    assert np.array_equal(_sorted_rows(got), _sorted_rows(ref)), "fp16 copy of a chunk differs from fp16(c / 2^e)"


# ---------------------------------------------------------------------------------------------------------------
# ns2_add_rows_bcast
# ---------------------------------------------------------------------------------------------------------------
def _add_rows_case(B, R, D, scale, seed):
    from naturalspeech2_pytorch_b200 import ops
    g = _gen(seed)
    xbuf, x = _nan_buf((B, R, D))
    x.copy_(torch.randn(B, R, D, device=dev, generator=g))
    vbuf, v = _nan_buf((B, D))
    v.copy_(torch.randn(B, D, device=dev, generator=g))
    x0 = x.clone()
    assert ops.add_rows_bcast(x, v, scale) is x
    s = float(torch.tensor(scale, dtype=torch.float32))   # the scale the kernel multiplies by
    ref = (x0.double() + s * v.double()[:, None, :]).float()
    assert torch.equal(x, ref), f"B={B} R={R} D={D} scale={scale}: max err {float((x - ref).abs().max()):.3g}"
    assert_nan(xbuf[x.numel():], "past x")
    assert_nan(vbuf[v.numel():], "past v")


@pytest.mark.parametrize("scale", [1.0, 1.0 / 7.0])
@pytest.mark.parametrize("D", [1, 5, 512])
@pytest.mark.parametrize("R", [1, 1000])
@pytest.mark.parametrize("B", [1, 3])
def test_add_rows_bcast_exact(B, R, D, scale):
    """x += scale * v per row: one fp32 fma per element, so exact against fp64 rounded once.  B 3, R 1000, D 512 is
    1.5 M elements, past the grid cap of 8 CTAs x 256 threads per SM."""
    _add_rows_case(B, R, D, scale, seed=B * 1000 + R + D)


def test_add_rows_bcast_grid_stride():
    """Capped to 2 SMs (16 CTAs, 4096 threads) every thread loops over 15 000 elements a few times."""
    with sm_limit(2):
        _add_rows_case(3, 1000, 5, 1.0 / 7.0, seed=3)
