"""torch-tensor front end of the C ABI (include/ns2_b200.h).

Every function takes CUDA tensors, validates what the kernels assume (dtype, contiguity of the channel
dimension, alignment) and enqueues ONE library call on the current torch CUDA stream.  Nothing here computes
on the host or falls back to PyTorch math: if the library is missing, `_lib.load()` raises.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence, Tuple

import torch

from . import _lib
from ._lib import (AttnArgs, GemmArgs, NS2_EPI_BF16, NS2_EPI_F32, NS2_EPI_GEGLU, NS2_EPI_WAVENET,
                   NS2_MSE_SCRATCH_PER_SAMPLE, check)

EPI_BF16, EPI_F32, EPI_GEGLU, EPI_WAVENET = NS2_EPI_BF16, NS2_EPI_F32, NS2_EPI_GEGLU, NS2_EPI_WAVENET

Seg = Tuple[int, int, int, int, int]  # (a_col_off, b_col_off, k_len, shift_units, acc)


def _stream(t: Optional[torch.Tensor] = None) -> int:
    """Raw handle of torch's current stream.  The library launches on the CURRENT device (tensor maps, kernel
    attributes and the SM count are per device), so a tensor that lives elsewhere is rejected instead of being
    launched on the wrong GPU — wrap the call in `torch.cuda.device(t.device)`."""
    if t is not None and t.device.index != torch.cuda.current_device():
        raise ValueError(f"tensor is on {t.device} but the current CUDA device is cuda:{torch.cuda.current_device()}")
    return torch.cuda.current_stream().cuda_stream


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _req(t: torch.Tensor, dtype: torch.dtype, name: str) -> None:
    if not t.is_cuda:
        raise ValueError(f"{name} must be a CUDA tensor (the ns2_b200 ops have no CPU path)")
    if t.dtype != dtype:
        raise ValueError(f"{name} must be {dtype}, got {t.dtype}")
    if t.dim() > 0 and t.shape[-1] > 1 and t.stride(-1) != 1:
        raise ValueError(f"{name} must be contiguous in its last dimension")


def _req_flat(t: torch.Tensor, dtype: torch.dtype, name: str, numel: int, align: int = 16) -> None:
    """`t` is read or written as one flat array of `numel` elements, in vectors of `align` bytes (float4 loads of fp32
    data, 4 x bf16 stores; align=1 for per-sample scalars read one element at a time)."""
    _req(t, dtype, name)
    if not t.is_contiguous():
        raise ValueError(f"{name} must be contiguous")
    if t.numel() != numel:
        raise ValueError(f"{name} must hold {numel} elements, got {t.numel()}")
    if t.data_ptr() % align:
        raise ValueError(f"{name} must be {align}-byte aligned")


def set_sm_limit(sms: int) -> int:
    """Size every kernel's persistent grid for at most `sms` SMs (0 = all).  Returns the previous limit."""
    return int(_lib.load().ns2_set_sm_limit(int(sms)))


def launch_count() -> int:
    return int(_lib.load().ns2_launch_count())


# --------------------------------------------------------------------------------------------------
# GEMM family
# --------------------------------------------------------------------------------------------------
def gemm(a: torch.Tensor, w: torch.Tensor, out: torch.Tensor, *, n: int, epilogue: int,
         segs: Optional[Sequence[Seg]] = None, bias: Optional[torch.Tensor] = None,
         resid: Optional[torch.Tensor] = None, film: Optional[torch.Tensor] = None,
         film_group_stride: int = 0, bias1_off: int = 0, groups: int = 1,
         a_group_col_stride: int = 0, b_group_row_stride: int = 0, out_group_col_stride: int = 0,
         dil: Optional[Sequence[int]] = None, flags: int = 0) -> torch.Tensor:
    """out = epilogue(segmented_gemm(a, w)).  `a`: (batches, rows, cols) bf16 (may be a strided view),
    `w`: packed bf16 weight (rows, K).  See include/ns2_b200.h section 1 for the exact semantics."""
    lib = _lib.load()
    _req(a, torch.bfloat16, "a")
    _req(w, torch.bfloat16, "w")
    if a.dim() != 3 or w.dim() != 2:
        raise ValueError("a must be (batches, rows, cols) and w (rows, K)")
    out_dtype = torch.float32 if epilogue == EPI_F32 else torch.bfloat16
    _req(out, out_dtype, "out")
    if out.dim() != 3 or out.shape[0] != a.shape[0] or out.shape[1] != a.shape[1]:
        raise ValueError(f"out must be (batches, rows, *), got {tuple(out.shape)} for a {tuple(a.shape)}")
    if out.shape[0] > 1 and out.stride(0) != out.shape[1] * out.stride(1):
        raise ValueError("out rows must be uniformly strided across batches")
    if segs is None:
        segs = [(0, 0, a.shape[2], 0, 0)]
    args = GemmArgs()
    args.A = a.data_ptr()
    args.a_row_stride, args.a_batch_stride = a.stride(1), a.stride(0)
    args.a_batches, args.a_rows, args.a_cols = a.shape
    args.B = w.data_ptr()
    args.b_row_stride = w.stride(0)
    args.b_rows, args.b_cols = w.shape
    args.n = n
    args.groups = groups
    args.a_group_col_stride = a_group_col_stride
    args.b_group_row_stride = b_group_row_stride
    args.out_group_col_stride = out_group_col_stride
    for g in range(_lib.NS2_GEMM_MAX_GROUPS):
        args.dil[g] = int(dil[g]) if dil is not None and g < len(dil) else 1
    args.num_segs = len(segs)
    for i, s in enumerate(segs):
        sg = args.segs[i]
        sg.a_col_off, sg.b_col_off, sg.k_len, sg.shift_units, sg.acc = (int(v) for v in s)
    args.epilogue = epilogue
    if bias is not None:
        _req(bias, torch.float32, "bias")
        # the epilogue reads bias[g * b_group_row_stride + col] for every output column col < n (and + bias1_off)
        need = (groups - 1) * b_group_row_stride + n + (bias1_off if epilogue == EPI_WAVENET else 0)
        if not bias.is_contiguous() or bias.numel() < need:
            raise ValueError(f"bias must be contiguous with >= {need} elements for n={n}, got {bias.numel()}")
    args.bias = _ptr(bias)
    args.bias1_off = bias1_off
    args.out = out.data_ptr()
    args.out_row_stride = out.stride(1)
    if resid is not None:
        _req(resid, torch.float32, "resid")
        if resid.shape != out.shape or (resid.shape[0] > 1 and resid.stride(0) != resid.shape[1] * resid.stride(1)):
            raise ValueError("resid must match out's shape with uniformly strided rows")
        args.resid_row_stride = resid.stride(1)
    args.resid = _ptr(resid)
    if film is not None:
        _req(film, torch.float32, "film")
        args.film_batch_stride = film.stride(0)
    args.film = _ptr(film)
    args.film_group_stride = film_group_stride
    args.flags = int(flags)
    check(lib.ns2_gemm(C.byref(args), _stream(out)), "ns2_gemm")
    return out


def wgrad(dy: torch.Tensor, x: torch.Tensor, dw: torch.Tensor, *, n: int, k: int, shift_units: int = 0,
          x_col_off: int = 0, groups: int = 1, dy_group_col_stride: int = 0, x_group_col_stride: int = 0,
          dw_group_row_stride: int = 0, dil: Optional[Sequence[int]] = None, splits: int = 0) -> torch.Tensor:
    """dw[g][:n, :k] += dy[..., g-th n columns]^T @ x[..., rows shifted by shift_units*dil[g], g-th k columns].
    dy, x: (batches, rows, cols) bf16 (strided views are fine); dw: fp32 2-D (rows >= groups' n rows, cols >= k)."""
    lib = _lib.load()
    _req(dy, torch.bfloat16, "dy")
    _req(x, torch.bfloat16, "x")
    _req(dw, torch.float32, "dw")
    if dy.dim() != 3 or x.dim() != 3 or dy.shape[:2] != x.shape[:2] or dw.dim() != 2:
        raise ValueError("wgrad: dy and x must be (batches, rows, cols) with equal leading dims; dw 2-D")
    if groups > 1 and n % 128 != 0:
        raise ValueError("wgrad: n must be a multiple of 128 for grouped weights")
    args = _lib.WgradArgs()
    args.dY, args.dy_row_stride, args.dy_batch_stride, args.dy_cols = dy.data_ptr(), dy.stride(1), dy.stride(0), dy.shape[2]
    args.X, args.x_row_stride, args.x_batch_stride, args.x_cols = x.data_ptr(), x.stride(1), x.stride(0), x.shape[2]
    args.batches, args.rows = dy.shape[0], dy.shape[1]
    args.n, args.k = n, k
    args.groups = groups
    args.dy_group_col_stride, args.x_group_col_stride, args.x_col_off = dy_group_col_stride, x_group_col_stride, x_col_off
    for g in range(_lib.NS2_GEMM_MAX_GROUPS):
        args.dil[g] = int(dil[g]) if dil is not None and g < len(dil) else 1
    args.shift_units = shift_units
    args.dW, args.dw_row_stride, args.dw_group_row_stride = dw.data_ptr(), dw.stride(0), dw_group_row_stride
    args.splits = splits
    check(lib.ns2_wgrad(C.byref(args), _stream(dw)), "ns2_wgrad")
    return dw


def fold_conv_linear(w2: torch.Tensor, wc: torch.Tensor, bc: torch.Tensor, b2: torch.Tensor, i_pad: int):
    """Stacked (conv, Linear) pairs with nothing between them as one conv each (include/ns2_b200.h section 1c):
    w2 (L, O, K), wc (L, K, I, taps), bc (L, K), b2 (L, O) fp32 -> (bf16 (L, O, taps*i_pad) tap-major pack of the taps
    w2 @ wc[..., t], zero-padded from I to i_pad; fp32 (L, O) bias w2 @ bc + b2)."""
    lib = _lib.load()
    for t, name in ((w2, "w2"), (wc, "wc"), (bc, "bc"), (b2, "b2")):
        _req(t, torch.float32, name)
        if not t.is_contiguous():
            raise ValueError(f"{name} must be contiguous")
    if w2.dim() != 3 or wc.dim() != 4 or bc.dim() != 2 or b2.dim() != 2:
        raise ValueError("fold_conv_linear: w2 (L, O, K), wc (L, K, I, taps), bc (L, K), b2 (L, O)")
    L, O, K = w2.shape
    _, _, I, taps = wc.shape
    if wc.shape[:2] != (L, K) or bc.shape != (L, K) or b2.shape != (L, O) or i_pad < I:
        raise ValueError(f"fold_conv_linear: shapes w2 {tuple(w2.shape)}, wc {tuple(wc.shape)}, bc {tuple(bc.shape)}, "
                         f"b2 {tuple(b2.shape)}, i_pad {i_pad} do not fit")
    out = torch.empty(L, O, taps * i_pad, device=w2.device, dtype=torch.bfloat16)
    bias = torch.empty(L, O, device=w2.device, dtype=torch.float32)
    check(lib.ns2_fold_conv_linear(w2.data_ptr(), wc.data_ptr(), bc.data_ptr(), b2.data_ptr(), L, O, K, I, taps, i_pad,
                                   out.data_ptr(), bias.data_ptr(), _stream(out)), "ns2_fold_conv_linear")
    return out, bias


def conv_segs(c_in: int, kernel: int, first_shift: int) -> list:
    """Segments of a stride-1 convolution whose packed weight holds tap t at columns [t*c_in, (t+1)*c_in): tap t reads
    x[n - (first_shift - t) * dilation].  Causal k=3 (CausalConv1d, ns2.py:583-595): first_shift = 2; "same" padding p:
    first_shift = p."""
    return [(0, t * c_in, c_in, first_shift - t, 0) for t in range(kernel)]


def conv3_segs(c_in: int) -> list:
    """`conv_segs` of the denoiser's causal k=3 convs (CausalConv1d, ns2.py:583-595)."""
    return conv_segs(c_in, 3, 2)


def conv_dgrad_segs(c_out: int, kernel: int, first_shift: int) -> list:
    """Segments of the input gradient of a `conv_segs` convolution on the transposed pack ([in][tap][out]): tap t reads
    d out at n + (first_shift - t), the mirrored shift."""
    return [(0, t * c_out, c_out, t - first_shift, 0) for t in range(kernel)]


# --------------------------------------------------------------------------------------------------
# dropout (training): (seed, site, p) of one dropout site, see include/ns2_b200.h section 2b
# --------------------------------------------------------------------------------------------------
DropoutSpec = Tuple[int, int, float]   # (64-bit seed, site, p)


def _dropout_args(dropout: Optional[DropoutSpec]) -> Optional["_lib.Dropout"]:
    """ctypes parameters of `dropout`, or None when it draws nothing (None or p = 0: no dropout)."""
    if dropout is None:
        return None
    seed, site, p = dropout
    if not 0.0 <= float(p) < 1.0:
        raise ValueError(f"dropout p must be in [0, 1), got {p}")
    if not 0 <= int(seed) < 2 ** 64 or not 0 <= int(site) < 2 ** 32:
        raise ValueError(f"dropout seed must fit in 64 bits and site in 32 bits, got {seed}, {site}")
    if float(p) == 0.0:
        return None
    return _lib.Dropout(int(seed), int(site), float(p))


def dropout_(x: torch.Tensor, *, dropout: Optional[DropoutSpec]) -> torch.Tensor:
    """x (f32, contiguous, in place) *= keep * 1 / (1 - p): element i's keep bit is word i & 3 of Philox block i >> 2
    of (seed, site).  Applying the same (seed, site, p) to a gradient gives the backward of the forward call."""
    lib = _lib.load()
    _req_flat(x, torch.float32, "x", x.numel())
    d = _dropout_args(dropout)
    if d is not None:
        check(lib.ns2_dropout_f32(x.data_ptr(), x.numel(), C.byref(d), _stream(x)), "ns2_dropout_f32")
    return x


# --------------------------------------------------------------------------------------------------
# per-sample lengths: a batch of sequences padded at the end to the longest one
# --------------------------------------------------------------------------------------------------
def lengths(lens, batch: int, max_len: Optional[int], *, device, name: str = "lengths", lo: int = 1) -> torch.Tensor:
    """`lens` (a sequence of ints, or an integer tensor anywhere) as the contiguous int32 CUDA tensor the ragged kernels
    read, after checking it holds `batch` values in [lo, max_len] (max_len None: no upper bound)."""
    if isinstance(lens, torch.Tensor):
        if lens.is_floating_point() or lens.is_complex() or lens.dtype == torch.bool:
            raise ValueError(f"{name} must hold integers, got {lens.dtype}")
        host = lens.detach().reshape(-1).tolist() if lens.dim() <= 1 else None
    else:
        host = [int(v) for v in lens]
    if host is None or len(host) != batch:
        raise ValueError(f"{name} must hold one length per sample ({batch}), got {host if host is None else len(host)}")
    _check_range(name, min(host), max(host), lo, max_len)
    out = torch.tensor(host, dtype=torch.int32).to(device)
    out._ns2_range = (out._version, min(host), max(host))
    return out


def _check_range(name: str, mn: int, mx: int, lo: int, hi: Optional[int]) -> None:
    if mn < lo or (hi is not None and mx > hi):
        raise ValueError(f"{name} must lie in [{lo}, {hi if hi is not None else 'inf'}], got values in [{mn}, {mx}]")


def _check_lens(lens: torch.Tensor, batch: int, lo: int, hi: Optional[int], name: str) -> int:
    """Check per-sample lengths before a ragged launch: an int32 CUDA tensor of `batch` values in [lo, hi] on the current
    device.  The range is read once per tensor version (one device sync) and remembered on the tensor; while a CUDA graph
    is being captured values cannot be read, and the kernels clamp them instead.  Returns the data pointer."""
    if not isinstance(lens, torch.Tensor) or not lens.is_cuda:
        raise ValueError(f"{name} must be a CUDA int32 tensor")
    if lens.dtype != torch.int32:
        raise ValueError(f"{name} must be int32, got {lens.dtype}")
    if lens.dim() != 1 or lens.numel() != batch or not lens.is_contiguous():
        raise ValueError(f"{name} must be a contiguous ({batch},) tensor, got {tuple(lens.shape)}")
    _stream(lens)
    rng = getattr(lens, "_ns2_range", None)
    if rng is None or rng[0] != lens._version:
        if torch.cuda.is_current_stream_capturing():
            return lens.data_ptr()
        mn, mx = torch.stack((lens.min(), lens.max())).tolist()
        rng = lens._ns2_range = (lens._version, mn, mx)
    _check_range(name, rng[1], rng[2], lo, hi)
    return lens.data_ptr()


def mask_rows(x: torch.Tensor, lens: torch.Tensor) -> torch.Tensor:
    """x (B, N, C) f32 or bf16, in place: rows r >= lens[b] of sample b become exact zeros.  Row- and batch-strided
    views are fine (channels contiguous); lens in [0, N]."""
    lib = _lib.load()
    if x.dtype not in (torch.float32, torch.bfloat16):
        raise ValueError(f"x must be float32 or bfloat16, got {x.dtype}")
    _req(x, x.dtype, "x")
    if x.dim() != 3:
        raise ValueError(f"x must be (B, N, C), got {tuple(x.shape)}")
    B, N, Cc = x.shape
    lp = _check_lens(lens, B, 0, N, "lens")
    check(lib.ns2_mask_rows(x.data_ptr(), int(x.dtype == torch.float32), x.stride(1), x.stride(0), B, N, Cc, lp,
                            _stream(x)), "ns2_mask_rows")
    return x


def pack_rows(a: torch.Tensor, a_lens: torch.Tensor, b: torch.Tensor, b_lens: torch.Tensor,
              out: torch.Tensor) -> torch.Tensor:
    """bf16 out[s] = [a[s, :a_lens[s]] ; b[s, :b_lens[s]] ; 0]: two end-padded segments (B, Na, C), (B, Nb, C) as one
    prefix of length a_lens + b_lens of out (B, No >= Na + Nb, C).  Row- and batch-strided views are fine."""
    lib = _lib.load()
    for name, t in (("a", a), ("b", b), ("out", out)):
        _req(t, torch.bfloat16, name)
        if t.dim() != 3:
            raise ValueError(f"{name} must be (B, N, C), got {tuple(t.shape)}")
    B, Na, Cc = a.shape
    if b.shape[0] != B or out.shape[0] != B or b.shape[2] != Cc or out.shape[2] != Cc:
        raise ValueError(f"pack_rows: inconsistent shapes {tuple(a.shape)}, {tuple(b.shape)}, {tuple(out.shape)}")
    Nb, No = b.shape[1], out.shape[1]
    if No < Na + Nb:
        raise ValueError(f"out holds {No} rows, fewer than {Na} + {Nb}")
    ap = _check_lens(a_lens, B, 0, Na, "a_lens")
    bp = _check_lens(b_lens, B, 0, Nb, "b_lens")
    check(lib.ns2_pack_rows(a.data_ptr(), a.stride(1), a.stride(0), Na, ap, b.data_ptr(), b.stride(1), b.stride(0), Nb,
                            bp, B, Cc, out.data_ptr(), out.stride(1), out.stride(0), No, _stream(out)), "ns2_pack_rows")
    return out


# --------------------------------------------------------------------------------------------------
# attention
# --------------------------------------------------------------------------------------------------
def attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, out: torch.Tensor, *, heads: int,
              scale: Optional[float] = None, lse: Optional[torch.Tensor] = None,
              dropout: Optional[DropoutSpec] = None, kv_lens: Optional[torch.Tensor] = None) -> torch.Tensor:
    """q: (B, Nq, heads*64), k/v: (B, Nk, heads*64) bf16 (strided views into a fused projection are fine).
    dropout=(seed, site, p): attention dropout on the softmax probabilities (lse stays that of the undropped ones).
    kv_lens: int32 CUDA (B,) in [1, Nk]: sample b attends to its keys [0, kv_lens[b]) only (K / V rows past it must be
    finite); its output is bit-identical to the call on that sample's keys alone.  No dropout with kv_lens."""
    lib = _lib.load()
    for name, t in (("q", q), ("k", k), ("v", v), ("out", out)):
        _req(t, torch.bfloat16, name)
        if t.dim() != 3 or t.shape[2] != heads * 64:
            raise ValueError(f"{name} must be (B, N, heads*64), got {tuple(t.shape)}")
    lens_ptr = None
    if kv_lens is not None:
        if dropout is not None:
            raise ValueError("attention: dropout with kv_lens is not supported")
        lens_ptr = _check_lens(kv_lens, q.shape[0], 1, k.shape[1], "kv_lens")
    args = AttnArgs()
    args.q, args.q_row_stride, args.q_batch_stride = q.data_ptr(), q.stride(1), q.stride(0)
    args.k, args.k_row_stride, args.k_batch_stride = k.data_ptr(), k.stride(1), k.stride(0)
    args.v, args.v_row_stride, args.v_batch_stride = v.data_ptr(), v.stride(1), v.stride(0)
    args.out, args.o_row_stride, args.o_batch_stride = out.data_ptr(), out.stride(1), out.stride(0)
    args.batches, args.heads = q.shape[0], heads
    args.q_len, args.kv_len, args.dim_head = q.shape[1], k.shape[1], 64
    args.scale = float(scale if scale is not None else 64 ** -0.5)
    if lse is not None:
        _req(lse, torch.float32, "lse")
        if not lse.is_contiguous() or tuple(lse.shape) != (q.shape[0], heads, q.shape[1]):
            raise ValueError("lse must be a contiguous (B, heads, Nq) float tensor")
    args.lse, args.kv_lens = _ptr(lse), lens_ptr
    d = _dropout_args(dropout)
    args.dropout = None if d is None else C.pointer(d)
    check(lib.ns2_attn_fwd(C.byref(args), _stream(out)), "ns2_attn_fwd")
    return out


# --------------------------------------------------------------------------------------------------
# norms, small layers, casts
# --------------------------------------------------------------------------------------------------
def rmsnorm_film(x: torch.Tensor, out: torch.Tensor, *, gamma: Optional[torch.Tensor] = None,
                 film: Optional[torch.Tensor] = None) -> torch.Tensor:
    """x: (B, N, D) f32 -> out (B, N, D) bf16.  film: (B, >=2D) f32 view whose row b holds [gamma_b | beta_b]."""
    lib = _lib.load()
    _req(x, torch.float32, "x")
    _req(out, torch.bfloat16, "out")
    if not (x.is_contiguous() and out.is_contiguous()):
        raise ValueError("x and out must be contiguous")
    B, N, D = x.shape
    if gamma is not None:
        _req(gamma, torch.float32, "gamma")
    film_bs = 0
    if film is not None:
        _req(film, torch.float32, "film")
        film_bs = film.stride(0)
    check(lib.ns2_rmsnorm_film(x.data_ptr(), D, B * N, D, N, _ptr(gamma), _ptr(film), film_bs,
                               out.data_ptr(), D, _stream(out)), "ns2_rmsnorm_film")
    return out


def rmsnorm_f32(x: torch.Tensor, out: torch.Tensor, gamma: Optional[torch.Tensor]) -> torch.Tensor:
    """out (f32, x's shape) = RMSNorm(x) (* gamma) over the last dimension; x and out contiguous."""
    lib = _lib.load()
    D = x.shape[-1]
    _req_flat(x, torch.float32, "x", x.numel())
    _req_flat(out, torch.float32, "out", x.numel())
    if gamma is not None:
        _req_flat(gamma, torch.float32, "gamma", D)
    rows = x.numel() // D
    check(lib.ns2_rmsnorm_f32(x.data_ptr(), D, rows, D, _ptr(gamma), out.data_ptr(), D, _stream()),
          "ns2_rmsnorm_f32")
    return out


_SMALL_BATCH_MAX = 64          # kMaxSmallBatch in csrc/elementwise.cu
_SMALL_SMEM_BYTES = 200 * 1024  # dynamic shared memory the small-layer kernel may use for its (batch, k) input tile


def _small_chunk(k: int) -> int:
    return max(1, min(_SMALL_BATCH_MAX, _SMALL_SMEM_BYTES // (4 * k)))


def time_cond(times: torch.Tensor, freqs: torch.Tensor, w: torch.Tensor, bias: torch.Tensor,
              out: torch.Tensor) -> torch.Tensor:
    """out[b] = silu(W @ [t_b, sin(2 pi t_b f), cos(2 pi t_b f)] + bias); out may be a column slice.
    Batches larger than the kernel's per-launch limit are processed in row chunks."""
    lib = _lib.load()
    for name, t in (("times", times), ("freqs", freqs), ("w", w), ("bias", bias), ("out", out)):
        _req(t, torch.float32, name)
    step = _small_chunk(2 * freqs.shape[0] + 1)
    for b0 in range(0, times.shape[0], step):
        tb, ob = times[b0:b0 + step], out[b0:b0 + step]
        check(lib.ns2_time_cond(tb.data_ptr(), tb.shape[0], freqs.data_ptr(), freqs.shape[0], w.data_ptr(),
                                bias.data_ptr(), w.shape[0], ob.data_ptr(), out.stride(0), _stream()),
              "ns2_time_cond")
    return out


def small_linear(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor], out: torch.Tensor,
                 act: int = 0) -> torch.Tensor:
    lib = _lib.load()
    for name, t in (("x", x), ("w", w), ("out", out)):
        _req(t, torch.float32, name)
    step = _small_chunk(x.shape[1])
    for b0 in range(0, x.shape[0], step):
        xb, ob = x[b0:b0 + step], out[b0:b0 + step]
        check(lib.ns2_small_linear(xb.data_ptr(), x.stride(0), xb.shape[0], x.shape[1], w.data_ptr(), _ptr(bias),
                                   w.shape[0], act, ob.data_ptr(), out.stride(0), _stream()), "ns2_small_linear")
    return out


def cast_bf16(x: torch.Tensor, out: torch.Tensor, add: Optional[torch.Tensor] = None) -> torch.Tensor:
    lib = _lib.load()
    _req(x, torch.float32, "x")
    _req(out, torch.bfloat16, "out")
    if not (x.is_contiguous() and out.is_contiguous()) or x.numel() != out.numel():
        raise ValueError("cast_bf16 needs contiguous tensors of equal size")
    if add is not None:
        _req(add, torch.float32, "add")
        if not add.is_contiguous() or add.numel() != x.numel():
            raise ValueError("add must be contiguous and the same size as x")
    check(lib.ns2_cast_bf16(x.data_ptr(), _ptr(add), x.numel(), out.data_ptr(), _stream()),
          "ns2_cast_bf16")
    return out


def cond_inject(x: torch.Tensor, cproj: torch.Tensor, out: torch.Tensor, drop_mask: Optional[torch.Tensor] = None,
                null_cond: Optional[torch.Tensor] = None, *, cond_lens: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out (B, N, D) bf16 = x (B, N, D) f32 + [padded / curtailed, null-substituted] cproj (B, L, D) f32.
    cond_lens: int32 CUDA (B,) >= 0: sample b's condition ends at frame min(L, cond_lens[b])."""
    lib = _lib.load()
    _req(x, torch.float32, "x")
    _req(cproj, torch.float32, "cproj")
    _req(out, torch.bfloat16, "out")
    B, N, D = x.shape
    if not (x.is_contiguous() and cproj.is_contiguous() and out.is_contiguous()) or cproj.shape[0] != B \
            or cproj.shape[2] != D or out.shape != x.shape:
        raise ValueError("cond_inject: x/out (B, N, D) and cproj (B, L, D) must be contiguous and consistent")
    if drop_mask is not None:
        if drop_mask.dtype != torch.bool or drop_mask.numel() != B or not drop_mask.is_cuda:
            raise ValueError("drop_mask must be a CUDA bool tensor of B elements")
        _req(null_cond, torch.float32, "null_cond")
        if null_cond.numel() != D or not null_cond.is_contiguous():
            raise ValueError("null_cond must be a contiguous (D,) float tensor")
    lp = None if cond_lens is None else _check_lens(cond_lens, B, 0, None, "cond_lens")
    check(lib.ns2_cond_inject(x.data_ptr(), cproj.data_ptr(), _ptr(drop_mask), _ptr(null_cond), B, N, cproj.shape[1], D,
                              out.data_ptr(), lp, _stream(out)), "ns2_cond_inject")
    return out


def select_rows(drop_mask: torch.Tensor, null_row: torch.Tensor, src: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """out[b] = null_row if drop_mask[b] else src[b]; src/out are (B, ...) with contiguous trailing dims; out may be a
    column slice of a wider f32 matrix (row stride > row length) or a bf16 tensor."""
    lib = _lib.load()
    _req(null_row, torch.float32, "null_row")
    _req(src, torch.float32, "src")
    B = src.shape[0]
    row_len = src.numel() // B
    if drop_mask.dtype != torch.bool or drop_mask.numel() != B or not drop_mask.is_cuda:
        raise ValueError("drop_mask must be a CUDA bool tensor of B elements")
    if null_row.numel() != row_len or not null_row.is_contiguous() or not src.is_contiguous():
        raise ValueError("null_row must hold one row; src must be contiguous")
    if out.dtype not in (torch.float32, torch.bfloat16) or out.shape[0] != B or out.numel() != B * row_len:
        raise ValueError("out must be (B, ...) f32/bf16 with src's row length")
    if out.dim() > 2 and not out.is_contiguous():
        raise ValueError("multi-dimensional out must be contiguous")
    check(lib.ns2_select_rows(drop_mask.data_ptr(), null_row.data_ptr(), src.data_ptr(), row_len, B, row_len,
                              out.data_ptr(), out.stride(0), int(out.dtype == torch.bfloat16), _stream(out)),
          "ns2_select_rows")
    return out


def mean_rows(x: torch.Tensor, out: torch.Tensor, *, lens: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out (B, D) = mean over the rows of x (B, N, D) f32; lens: int32 CUDA (B,) in [1, N], the mean of sample b over
    its rows [0, lens[b])."""
    lib = _lib.load()
    _req(x, torch.float32, "x")
    _req(out, torch.float32, "out")
    B, N, D = x.shape
    lp = None if lens is None else _check_lens(lens, B, 1, N, "lens")
    if not out.is_contiguous() or tuple(out.shape) != (B, D):
        raise ValueError(f"out must be a contiguous ({B}, {D}) tensor")
    check(lib.ns2_mean_rows(x.contiguous().data_ptr(), B, N, D, out.data_ptr(), lp, _stream()), "ns2_mean_rows")
    return out


def transpose_cast(x: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """(B, C, L) f32 channel-first -> (B, L, C) bf16."""
    lib = _lib.load()
    _req(x, torch.float32, "x")
    _req(out, torch.bfloat16, "out")
    B, Cc, L = x.shape
    check(lib.ns2_transpose_cast(x.contiguous().data_ptr(), B, Cc, L, out.data_ptr(), _stream()),
          "ns2_transpose_cast")
    return out


# --------------------------------------------------------------------------------------------------
# diffusion element-wise
# --------------------------------------------------------------------------------------------------
OBJECTIVES = {"v": _lib.NS2_OBJ_V, "eps": _lib.NS2_OBJ_EPS, "x0": _lib.NS2_OBJ_X0}


def groupnorm_silu(x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor, groups: int, *, eps: float = 1e-5,
                   resid: Optional[torch.Tensor] = None, out_f32: Optional[torch.Tensor] = None,
                   out_bf16: Optional[torch.Tensor] = None, lens: Optional[torch.Tensor] = None):
    """silu(GroupNorm(groups)(x)) (+ resid) for token-major x (B, N, C) f32 -> out_f32 and/or out_bf16 (B, N, C).
    lens: int32 CUDA (B,) in [1, N]: sample b is normalised over its rows [0, lens[b]) (bit-identical to the call on
    those rows alone); its rows past that are written as zeros."""
    lib = _lib.load()
    _req(x, torch.float32, "x")
    _req(weight, torch.float32, "weight")
    _req(bias, torch.float32, "bias")
    if x.dim() != 3 or not x.is_contiguous():
        raise ValueError("x must be a contiguous (B, N, C) tensor")
    for name, t, dt in (("resid", resid, torch.float32), ("out_f32", out_f32, torch.float32),
                        ("out_bf16", out_bf16, torch.bfloat16)):
        if t is not None:
            _req(t, dt, name)
            if t.shape != x.shape or not t.is_contiguous():
                raise ValueError(f"{name} must be contiguous with x's shape")
    if out_f32 is None and out_bf16 is None:
        raise ValueError("groupnorm_silu needs at least one output")
    B, N, Cn = x.shape
    lp = None if lens is None else _check_lens(lens, B, 1, N, "lens")
    check(lib.ns2_groupnorm_silu(x.data_ptr(), B, N, Cn, int(groups), weight.data_ptr(), bias.data_ptr(), float(eps),
                                 _ptr(resid), _ptr(out_f32), _ptr(out_bf16), lp, _stream(x)), "ns2_groupnorm_silu")
    return out_f32, out_bf16


def rowdot(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor], out: torch.Tensor, relu: bool = False):
    """out[...] = (relu)(x[..., :] . w + bias): Linear(dim, 1) heads.  x f32 contiguous, w (dim,), out one value per row."""
    lib = _lib.load()
    _req(x, torch.float32, "x")
    _req(w, torch.float32, "w")
    _req(out, torch.float32, "out")
    if not (x.is_contiguous() and w.is_contiguous() and out.is_contiguous()) or out.numel() * x.shape[-1] != x.numel():
        raise ValueError("rowdot needs contiguous x (..., dim), w (dim,) and one output per row")
    if bias is not None:
        _req(bias, torch.float32, "bias")
    check(lib.ns2_rowdot(x.data_ptr(), out.numel(), x.shape[-1], w.data_ptr(), _ptr(bias), int(relu), out.data_ptr(),
                         _stream(x)), "ns2_rowdot")
    return out


def expand_encodings(phon: torch.Tensor, coarse: torch.Tensor, pitch_table: torch.Tensor, idx: torch.Tensor) -> torch.Tensor:
    """(B, D, L) f32 channel-first: phon[b, idx[b, n], :] + pitch_table[coarse[b, idx[b, n]], :], 0 where idx < 0
    (expand_encodings, ns2.py:1449-1455).  phon (B, T, D) f32, coarse (B, T) int32, idx (B, L) int32."""
    lib = _lib.load()
    _req(phon, torch.float32, "phon")
    _req(pitch_table, torch.float32, "pitch_table")
    _req(coarse, torch.int32, "coarse")
    _req(idx, torch.int32, "idx")
    if not all(t.is_contiguous() for t in (phon, coarse, pitch_table, idx)):
        raise ValueError("expand_encodings needs contiguous tensors")
    B, T, D = phon.shape
    if coarse.shape != (B, T) or idx.dim() != 2 or idx.shape[0] != B or pitch_table.shape[1] != D:
        raise ValueError("expand_encodings: inconsistent shapes")
    L = idx.shape[1]
    out = torch.empty(B, D, L, device=phon.device, dtype=torch.float32)
    check(lib.ns2_expand_encodings(phon.data_ptr(), coarse.data_ptr(), pitch_table.data_ptr(), pitch_table.shape[0],
                                   idx.data_ptr(), B, T, D, L, out.data_ptr(), _stream(phon)), "ns2_expand_encodings")
    return out


def embedding_bf16(ids: torch.Tensor, table: torch.Tensor, out: torch.Tensor, pad_id: int) -> torch.Tensor:
    """out[..., :] = bf16(table[ids < 0 ? pad_id : ids]) — nn.Embedding + padding substitution (ns2.py:279-282)."""
    lib = _lib.load()
    _req(ids, torch.int64, "ids")
    _req(table, torch.float32, "table")
    _req(out, torch.bfloat16, "out")
    if not (ids.is_contiguous() and table.is_contiguous() and out.is_contiguous()):
        raise ValueError("embedding_bf16 needs contiguous tensors")
    if out.numel() != ids.numel() * table.shape[1]:
        raise ValueError("out must hold one table row per id")
    check(lib.ns2_embedding_bf16(ids.data_ptr(), ids.numel(), table.data_ptr(), table.shape[0], table.shape[1],
                                 int(pad_id), out.data_ptr(), _stream(out)), "ns2_embedding_bf16")
    return out


def q_sample(x0, noise, alpha, sigma, x_t, target=None, objective: str = "v"):
    """x_t = alpha x0 + sigma noise; target of the chosen parameterisation (ns2.py:1631-1644)."""
    lib = _lib.load()
    B = x0.shape[0]
    per = x0.numel() // B
    for name, t in (("x0", x0), ("noise", noise), ("x_t", x_t)) + ((("target", target),) if target is not None else ()):
        _req_flat(t, torch.float32, name, x0.numel())
    for name, t in (("alpha", alpha), ("sigma", sigma)):
        _req_flat(t, torch.float32, name, B, align=1)
    check(lib.ns2_q_sample(x0.data_ptr(), noise.data_ptr(), alpha.data_ptr(), sigma.data_ptr(), B, per,
                           x_t.data_ptr(), _ptr(target), OBJECTIVES[objective], _stream()), "ns2_q_sample")
    return x_t, target


def mse_rows(pred, target, out, scratch=None, mean_out=None):
    """out[b] = mean((pred[b] - target[b])^2); `mean_out` (0-d / 1-element f32) additionally receives out.mean()."""
    lib = _lib.load()
    B = pred.shape[0]
    per = pred.numel() // B
    for name, t in (("pred", pred), ("target", target), ("out", out)):
        _req(t, torch.float32, name)
    if not (pred.is_contiguous() and target.is_contiguous()):
        raise ValueError("pred and target must be contiguous")
    if scratch is None:
        scratch = torch.empty(B * NS2_MSE_SCRATCH_PER_SAMPLE, device=pred.device, dtype=torch.float32)
    if mean_out is not None:
        _req(mean_out, torch.float32, "mean_out")
    check(lib.ns2_mse_rows(pred.data_ptr(), target.data_ptr(), B, per, scratch.data_ptr(),
                           out.data_ptr(), _ptr(mean_out), _stream()), "ns2_mse_rows")
    return out


def ddim_step(x, v, alpha, sigma, alpha_next, sigma_next, objective: str = "v"):
    """In-place DDIM update of x from the model output `v` (ns2.py:1412-1429)."""
    lib = _lib.load()
    B = x.shape[0]
    per = x.numel() // B
    for name, t in (("x", x), ("v", v)):
        _req_flat(t, torch.float32, name, x.numel())
    for name, t in (("alpha", alpha), ("sigma", sigma), ("alpha_next", alpha_next), ("sigma_next", sigma_next)):
        _req_flat(t, torch.float32, name, B, align=1)
    check(lib.ns2_ddim_step(x.data_ptr(), v.data_ptr(), alpha.data_ptr(), sigma.data_ptr(),
                            alpha_next.data_ptr(), sigma_next.data_ptr(), B, per, OBJECTIVES[objective],
                            _stream()),
          "ns2_ddim_step")
    return x


def x_start_from_pred(x, pred, alpha, sigma, out, objective: str = "v"):
    """x_start implied by the model output under the chosen parameterisation (ns2.py:1673-1680)."""
    lib = _lib.load()
    B = x.shape[0]
    per = x.numel() // B
    for name, t in (("x", x), ("pred", pred), ("out", out)):
        _req_flat(t, torch.float32, name, x.numel())
    for name, t in (("alpha", alpha), ("sigma", sigma)):
        _req_flat(t, torch.float32, name, B, align=1)
    check(lib.ns2_x_start(x.data_ptr(), pred.data_ptr(), alpha.data_ptr(), sigma.data_ptr(), B, per, out.data_ptr(),
                          OBJECTIVES[objective], _stream(out)), "ns2_x_start")
    return out


def cfg_combine(cond, null, scale, out):
    """out = null + (cond - null) * scale (classifier-free guidance); out may be cond or null itself."""
    lib = _lib.load()
    for name, t in (("cond", cond), ("null", null), ("out", out)):
        _req_flat(t, torch.float32, name, cond.numel())
    check(lib.ns2_cfg_combine(cond.data_ptr(), null.data_ptr(), float(scale), cond.numel(),
                              out.data_ptr(), _stream()), "ns2_cfg_combine")
    return out


# --------------------------------------------------------------------------------------------------
# RVQ
# --------------------------------------------------------------------------------------------------
def rvq_prepare(codebooks: torch.Tensor):
    """codebooks (Q, K, 128) f32 -> (fp16 copy, ||c||^2 (Q, K) f32, meta (Q, 2) f32)."""
    lib = _lib.load()
    _req(codebooks, torch.float32, "codebooks")
    cb = codebooks.contiguous()
    Q, K, D = cb.shape
    # fp16 copy (Q, K, D) followed by the (Q, K, 16) norm blocks: NS2_RVQ_PREPARED_HALFS
    cb16 = torch.empty((Q * K * (D + 16),), device=cb.device, dtype=torch.float16)
    cn2 = torch.empty((Q, K), device=cb.device, dtype=torch.float32)
    meta = torch.empty((Q, 2), device=cb.device, dtype=torch.float32)
    check(lib.ns2_rvq_prepare(cb.data_ptr(), Q, K, D, cb16.data_ptr(), cn2.data_ptr(), meta.data_ptr(),
                              _stream()), "ns2_rvq_prepare")
    return cb16, cn2, meta


def rvq_encode(frames: torch.Tensor, codebooks: torch.Tensor, prepared, codes: Optional[torch.Tensor] = None,
               stats: Optional[torch.Tensor] = None) -> torch.Tensor:
    """frames (F, 128) f32 -> codes (F, Q) int64."""
    lib = _lib.load()
    _req(frames, torch.float32, "frames")
    cb16, cn2, meta = prepared
    cb = codebooks.contiguous()
    Q, K, D = cb.shape
    fr = frames.contiguous()
    F = fr.shape[0]
    if codes is None:
        codes = torch.empty((F, Q), device=fr.device, dtype=torch.int64)
    if stats is not None and not (stats.is_cuda and stats.dtype == torch.int64 and stats.is_contiguous()
                                  and stats.numel() >= _lib.NS2_RVQ_STATS_LEN):
        raise ValueError(f"stats must be a contiguous CUDA int64 tensor with >= {_lib.NS2_RVQ_STATS_LEN} elements")
    check(lib.ns2_rvq_encode(fr.data_ptr(), F, D, cb.data_ptr(), cb16.data_ptr(), cn2.data_ptr(),
                             meta.data_ptr(), Q, K, codes.data_ptr(), _ptr(stats), _stream(codes)),
          "ns2_rvq_encode")
    return codes


def _req_dense(t: torch.Tensor, dtype: torch.dtype, shape: Tuple[Optional[int], ...], name: str) -> None:
    """dtype, shape (None = any size) and contiguity: the checks that need no device, so they fail the same way on a
    machine without a GPU."""
    if t.dtype != dtype:
        raise ValueError(f"{name} must be {dtype}, got {t.dtype}")
    if t.dim() != len(shape) or any(s is not None and s != n for s, n in zip(shape, t.shape)):
        want = ", ".join("*" if s is None else str(s) for s in shape)
        raise ValueError(f"{name} must have shape ({want}), got {tuple(t.shape)}")
    if not t.is_contiguous():
        raise ValueError(f"{name} must be contiguous")


def _req_device(device: torch.device, **tensors: torch.Tensor) -> None:
    """Every tensor is a CUDA tensor on `device`."""
    for name, t in tensors.items():
        if not t.is_cuda:
            raise ValueError(f"{name} must be a CUDA tensor (the ns2_b200 ops have no CPU path)")
        if t.device != device:
            raise ValueError(f"{name} is on {t.device}, expected {device}")


def rvq_decode(codes: torch.Tensor, codebooks: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """codes (F, Q) int64 -> emb (F, 128) f32 = sum_q codebooks[q, codes[:, q]], added in order q = 0..Q-1.  Codes
    outside [0, K) are clamped to 0 / K - 1.  `out` (optional) is a contiguous (F, 128) f32 tensor."""
    lib = _lib.load()
    _req_dense(codebooks, torch.float32, (None, None, 128), "codebooks")
    cb = codebooks.contiguous()
    Q, K, D = cb.shape
    _req_dense(codes, torch.int64, (None, Q), "codes")
    F = codes.shape[0]
    if out is None:
        out = torch.empty((F, D), device=codes.device, dtype=torch.float32)
    _req_dense(out, torch.float32, (F, D), "out")
    _req_device(codes.device, codes=codes, codebooks=cb, out=out)
    for name, t in (("codebooks", cb), ("out", out)):   # read / written as float4
        if t.data_ptr() % 16:
            raise ValueError(f"{name} must be 16-byte aligned")
    check(lib.ns2_rvq_decode(codes.data_ptr(), F, Q, K, D, cb.data_ptr(), out.data_ptr(), _stream(codes)),
          "ns2_rvq_decode")
    return out


def _rvq_ce_args(frames, codebooks, cn2, own_codes, target_codes):
    """Checks shared by rvq_ce and rvq_ce_bwd; returns (frames, codebooks) contiguous and F, Q, K."""
    fr, cb = frames.contiguous(), codebooks.contiguous()
    _req_dense(fr, torch.float32, (None, 128), "frames")
    _req_dense(cb, torch.float32, (None, None, 128), "codebooks")
    F = fr.shape[0]
    Q, K, _ = cb.shape
    _req_dense(cn2, torch.float32, (Q, K), "cn2")
    _req_dense(own_codes, torch.int64, (F, Q), "own_codes")
    _req_dense(target_codes, torch.int64, (F, Q), "target_codes")
    _req_device(fr.device, frames=fr, codebooks=cb, cn2=cn2, own_codes=own_codes, target_codes=target_codes)
    return fr, cb, F, Q, K


def rvq_ce(frames: torch.Tensor, codebooks: torch.Tensor, cn2: torch.Tensor, own_codes: torch.Tensor,
           target_codes: torch.Tensor) -> torch.Tensor:
    """Cross-entropy head of the residual VQ (`codec.rq`): frames (F, 128) f32, codebooks (Q, K, 128) f32, their
    squared norms cn2 (Q, K) f32, codes (F, Q) int64 -> 0-d loss."""
    lib = _lib.load()
    fr, cb, F, Q, K = _rvq_ce_args(frames, codebooks, cn2, own_codes, target_codes)
    D = 128
    scratch = torch.empty(F * Q, device=fr.device, dtype=torch.float32)
    loss = torch.empty((), device=fr.device, dtype=torch.float32)
    check(lib.ns2_rvq_ce(fr.data_ptr(), F, D, cb.data_ptr(), cn2.data_ptr(), Q, K, own_codes.data_ptr(),
                         target_codes.data_ptr(), scratch.data_ptr(), loss.data_ptr(), _stream(fr)), "ns2_rvq_ce")
    return loss


def rvq_ce_bwd(frames: torch.Tensor, codebooks: torch.Tensor, cn2: torch.Tensor, own_codes: torch.Tensor,
               target_codes: torch.Tensor, d_loss: torch.Tensor, row_scale: Optional[torch.Tensor] = None,
               rows_per_sample: int = 1, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """d loss / d frames of `rvq_ce` given d_loss (1-element f32 on the device): frames (F, 128) f32 -> (F, 128) f32.
    `row_scale` (optional, F / rows_per_sample f32) multiplies each sample's rows; `out` may be a (F, >= 128) f32 view
    with unit column stride (only its first 128 columns are written)."""
    lib = _lib.load()
    fr, cb, F, Q, K = _rvq_ce_args(frames, codebooks, cn2, own_codes, target_codes)
    D = 128
    _req(d_loss, torch.float32, "d_loss")
    if d_loss.numel() != 1:
        raise ValueError("d_loss must hold one element")
    if row_scale is not None:
        _req(row_scale, torch.float32, "row_scale")
        if not row_scale.is_contiguous() or rows_per_sample <= 0 or row_scale.numel() * rows_per_sample < F:
            raise ValueError("row_scale must be contiguous with one value per rows_per_sample rows")
    if out is None:
        out = torch.empty((F, D), device=fr.device, dtype=torch.float32)
    _req(out, torch.float32, "out")
    if out.dim() != 2 or out.shape[0] != F or out.shape[1] < D:
        raise ValueError("out must be (F, >= 128)")
    coef = torch.empty(Q, device=fr.device, dtype=torch.float32)
    check(lib.ns2_rvq_ce_bwd(fr.data_ptr(), F, D, cb.data_ptr(), cn2.data_ptr(), Q, K, own_codes.data_ptr(),
                             target_codes.data_ptr(), d_loss.data_ptr(), _ptr(row_scale), int(rows_per_sample),
                             coef.data_ptr(), out.data_ptr(), out.stride(0), _stream(fr)), "ns2_rvq_ce_bwd")
    return out


# --------------------------------------------------------------------------------------------------
# backward pass
# --------------------------------------------------------------------------------------------------
def attention_bwd(q, k, v, o, d_o, lse, dq_accum, dk, dv, *, heads: int, scale: Optional[float] = None,
                  delta: Optional[torch.Tensor] = None, dropout: Optional[DropoutSpec] = None):
    """(dq_accum f32 (B, Nq, inner) += dQ, dk, dv bf16) of softmax(q k^T scale) v given d_o; zero dq_accum for a plain dQ.
    dropout: the forward's (seed, site, p); the mask is regenerated, not stored."""
    lib = _lib.load()
    for name, t in (("q", q), ("k", k), ("v", v), ("o", o), ("d_o", d_o), ("dk", dk), ("dv", dv)):
        _req(t, torch.bfloat16, name)
        if t.dim() != 3 or t.shape[2] != heads * 64:
            raise ValueError(f"{name} must be (B, N, heads*64), got {tuple(t.shape)}")
    _req(lse, torch.float32, "lse")
    _req(dq_accum, torch.float32, "dq_accum")
    B, Nq, Nk = q.shape[0], q.shape[1], k.shape[1]
    if not dq_accum.is_contiguous() or tuple(dq_accum.shape) != (B, Nq, heads * 64):
        raise ValueError("dq_accum must be contiguous (B, Nq, heads*64) float32")
    if delta is None:
        delta = torch.empty(B, heads, Nq, device=q.device, dtype=torch.float32)
    a = _lib.AttnBwdArgs()
    a.q, a.q_row_stride, a.q_batch_stride = q.data_ptr(), q.stride(1), q.stride(0)
    a.k, a.k_row_stride, a.k_batch_stride = k.data_ptr(), k.stride(1), k.stride(0)
    a.v, a.v_row_stride, a.v_batch_stride = v.data_ptr(), v.stride(1), v.stride(0)
    a.o, a.o_row_stride, a.o_batch_stride = o.data_ptr(), o.stride(1), o.stride(0)
    a.d_o, a.do_row_stride, a.do_batch_stride = d_o.data_ptr(), d_o.stride(1), d_o.stride(0)
    a.lse, a.delta, a.dq_accum = lse.data_ptr(), delta.data_ptr(), dq_accum.data_ptr()
    a.dk, a.dk_row_stride, a.dk_batch_stride = dk.data_ptr(), dk.stride(1), dk.stride(0)
    a.dv, a.dv_row_stride, a.dv_batch_stride = dv.data_ptr(), dv.stride(1), dv.stride(0)
    a.batches, a.heads, a.q_len, a.kv_len, a.dim_head = B, heads, Nq, Nk, 64
    a.scale = float(scale if scale is not None else 64 ** -0.5)
    d = _dropout_args(dropout)
    a.dropout = None if d is None else C.pointer(d)
    check(lib.ns2_attn_bwd(C.byref(a), _stream(dq_accum)), "ns2_attn_bwd")
    return dq_accum, dk, dv


def rmsnorm_film_bwd(x, dh, dxr, dxr_bf, *, rows_per_batch: int, gamma=None, film=None, dfilm=None, dgamma=None):
    """dxr (f32, in place) += d/dx of rmsnorm_film(x) given dh (bf16); dxr_bf = bf16(dxr); dfilm / dgamma accumulate."""
    lib = _lib.load()
    _req(x, torch.float32, "x")
    _req(dh, torch.bfloat16, "dh")
    _req(dxr, torch.float32, "dxr")
    _req(dxr_bf, torch.bfloat16, "dxr_bf")
    for t in (x, dh, dxr, dxr_bf):
        if not t.is_contiguous():
            raise ValueError("rmsnorm_film_bwd needs contiguous tensors")
    D = x.shape[-1]
    rows = x.numel() // D
    film_bs = dfilm_bs = 0
    if film is not None:
        _req(film, torch.float32, "film")
        _req(dfilm, torch.float32, "dfilm")
        film_bs, dfilm_bs = film.stride(0), dfilm.stride(0)
    check(lib.ns2_rmsnorm_film_bwd(x.data_ptr(), dh.data_ptr(), rows, D, rows_per_batch, _ptr(gamma), _ptr(film), film_bs,
                                   _ptr(dfilm), dfilm_bs, _ptr(dgamma), dxr.data_ptr(), dxr_bf.data_ptr(), _stream(dxr)),
          "ns2_rmsnorm_film_bwd")
    return dxr


def geglu_bwd(pre, dg):
    """pre (rows, 2*Dp) bf16 packed [128 value | 128 gate] tiles -> overwritten by its gradient given dg (rows, Dp)."""
    lib = _lib.load()
    _req(pre, torch.bfloat16, "pre")
    _req(dg, torch.bfloat16, "dg")
    if not (pre.is_contiguous() and dg.is_contiguous()) or pre.shape[-1] != 2 * dg.shape[-1]:
        raise ValueError("geglu_bwd: pre (.., 2*Dp) and dg (.., Dp) must be contiguous")
    dp = dg.shape[-1]
    check(lib.ns2_geglu_bwd(pre.data_ptr(), dg.data_ptr(), dg.numel() // dp, dp, _stream(pre)), "ns2_geglu_bwd")
    return pre


def wavenet_gate_bwd(c, dy, dc, film, dfilm, *, dim: int, groups: int, film_group_stride: int):
    """c, dy, dc: (B, N, >= groups*dim) bf16 views (first groups*dim columns used); film/dfilm (B, ...) f32 views whose
    row b holds, for group g at g*film_group_stride, [gamma | beta]."""
    lib = _lib.load()
    for name, t in (("c", c), ("dy", dy), ("dc", dc)):
        _req(t, torch.bfloat16, name)
        if t.dim() != 3 or t.stride(0) != t.shape[1] * t.stride(1):
            raise ValueError(f"{name} must be (B, N, cols) with uniformly strided rows")
    _req(film, torch.float32, "film")
    _req(dfilm, torch.float32, "dfilm")
    B, N = c.shape[0], c.shape[1]
    check(lib.ns2_wavenet_gate_bwd(c.data_ptr(), c.stride(1), dy.data_ptr(), dy.stride(1), dc.data_ptr(), dc.stride(1), B,
                                   N, dim, groups, film.data_ptr(), film.stride(0), film_group_stride, dfilm.data_ptr(),
                                   dfilm.stride(0), _stream(dc)), "ns2_wavenet_gate_bwd")
    return dc


def colsum(t, out):
    """out[c] (f32) += sum over all leading dims of t[..., c] (bf16; last dim contiguous, uniform row stride)."""
    lib = _lib.load()
    _req(t, torch.bfloat16, "t")
    _req(out, torch.float32, "out")
    cols = t.shape[-1]
    rows = t.numel() // cols
    rs = t.stride(-2) if t.dim() >= 2 else cols
    if t.dim() == 3 and t.stride(0) != t.shape[1] * t.stride(1):
        raise ValueError("colsum: rows must be uniformly strided")
    check(lib.ns2_colsum_bf16(t.data_ptr(), rows, cols, rs, out.data_ptr(), _stream(out)), "ns2_colsum_bf16")
    return out


def group_sum(t, out, *, dim: int, groups: int):
    lib = _lib.load()
    _req(t, torch.bfloat16, "t")
    _req(out, torch.bfloat16, "out")
    if not (t.is_contiguous() and out.is_contiguous()):
        raise ValueError("group_sum needs contiguous tensors")
    check(lib.ns2_group_sum_bf16(t.data_ptr(), out.numel() // dim, dim, groups, out.data_ptr(), _stream(out)),
          "ns2_group_sum_bf16")
    return out


def mse_bwd(pred, target, coef, out_bf=None, out_f32=None):
    """coef[b] * (pred - target) as bf16 and/or f32: the seed of the backward pass."""
    lib = _lib.load()
    B = pred.shape[0]
    for name, t in (("pred", pred), ("target", target)):
        _req_flat(t, torch.float32, name, pred.numel())
    _req_flat(coef, torch.float32, "coef", B, align=1)
    if out_bf is not None:
        _req_flat(out_bf, torch.bfloat16, "out_bf", pred.numel(), align=8)
    if out_f32 is not None:
        _req_flat(out_f32, torch.float32, "out_f32", pred.numel())
    check(lib.ns2_mse_bwd(pred.data_ptr(), target.data_ptr(), coef.data_ptr(), B, pred.numel() // B, _ptr(out_bf),
                          _ptr(out_f32), _stream(pred)), "ns2_mse_bwd")
    return out_bf if out_bf is not None else out_f32


def film_wgrad(dfilm, t, dw, accumulate: bool = True):
    """dw (rows, cols) f32 (+)= dfilm (B, rows)^T @ t (B, cols).  accumulate=False overwrites dw (which then need not be
    initialised: one pass over the gradient buffer instead of zero-fill + read-modify-write).  `dfilm` may be a column
    window of a wider (B, total_rows) buffer (unit column stride)."""
    lib = _lib.load()
    for name, x in (("dfilm", dfilm), ("t", t), ("dw", dw)):
        _req(x, torch.float32, name)
    if not (t.is_contiguous() and dw.is_contiguous()) or dfilm.dim() != 2 or (dfilm.shape[1] > 1 and dfilm.stride(1) != 1):
        raise ValueError("t and dw must be contiguous, dfilm (B, rows) with unit column stride")
    B, rows = dfilm.shape
    if tuple(dw.shape) != (rows, t.shape[1]) or t.shape[0] != B:
        raise ValueError("film_wgrad: inconsistent shapes")
    for b0 in range(0, B, 32):
        check(lib.ns2_film_wgrad(dfilm[b0:b0 + 32].data_ptr(), dfilm.stride(0), t[b0:b0 + 32].data_ptr(), min(32, B - b0),
                                 rows, t.shape[1], dw.data_ptr(), int(accumulate or b0 > 0), _stream(dw)),
              "ns2_film_wgrad")
    return dw


def accum_bf16(acc, t, acc_bf=None):
    """acc (f32, contiguous) += t (bf16, contiguous, same numel); acc_bf (optional) = bf16(acc)."""
    lib = _lib.load()
    _req(acc, torch.float32, "acc")
    _req(t, torch.bfloat16, "t")
    if not (acc.is_contiguous() and t.is_contiguous()) or acc.numel() != t.numel():
        raise ValueError("accum_bf16 needs contiguous tensors of equal size")
    if acc_bf is not None:
        _req(acc_bf, torch.bfloat16, "acc_bf")
    check(lib.ns2_accum_bf16(acc.data_ptr(), t.data_ptr(), acc.numel(), _ptr(acc_bf), _stream(acc)), "ns2_accum_bf16")
    return acc


# --------------------------------------------------------------------------------------------------
# backward of the conditioning front end (encoders, pitch embedding, length regulation)
# --------------------------------------------------------------------------------------------------
def silu_bwd(pre: torch.Tensor, dout: torch.Tensor, dpre: Optional[torch.Tensor] = None) -> torch.Tensor:
    """d pre of out = silu(pre) given d out; pre, dout, dpre bf16 contiguous of one size.  dpre defaults to pre (in place)."""
    lib = _lib.load()
    dpre = pre if dpre is None else dpre
    for name, t in (("pre", pre), ("dout", dout), ("dpre", dpre)):
        _req(t, torch.bfloat16, name)
        if not t.is_contiguous() or t.numel() != pre.numel():
            raise ValueError("silu_bwd needs contiguous tensors of equal size")
    check(lib.ns2_silu_bwd(pre.data_ptr(), dout.data_ptr(), pre.numel(), dpre.data_ptr(), _stream(dpre)), "ns2_silu_bwd")
    return dpre


def embedding_bwd(ids: torch.Tensor, de: torch.Tensor, dtable: torch.Tensor, pad_id: int) -> torch.Tensor:
    """dtable[ids < 0 ? pad_id : ids] += de (f32, accumulated): the backward of `embedding_bf16`."""
    lib = _lib.load()
    _req(ids, torch.int64, "ids")
    _req(de, torch.float32, "de")
    _req(dtable, torch.float32, "dtable")
    if not (ids.is_contiguous() and de.is_contiguous() and dtable.is_contiguous()) or dtable.dim() != 2:
        raise ValueError("embedding_bwd needs contiguous tensors and a 2-D table")
    if de.numel() != ids.numel() * dtable.shape[1]:
        raise ValueError("de must hold one table row per id")
    check(lib.ns2_embedding_bwd(ids.data_ptr(), ids.numel(), de.data_ptr(), dtable.shape[0], dtable.shape[1], int(pad_id),
                                dtable.data_ptr(), _stream(dtable)), "ns2_embedding_bwd")
    return dtable


def groupnorm_silu_bwd(x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor, groups: int, dy: torch.Tensor,
                       dx: torch.Tensor, *, eps: float = 1e-5) -> Tuple[torch.Tensor, torch.Tensor]:
    """Backward of `groupnorm_silu` (without its residual): x, dy f32 (B, N, C) contiguous -> dx bf16 (B, N, C) written,
    returns (d weight, d bias) f32 (C,), reduced over the batch in a fixed order (bit-reproducible)."""
    lib = _lib.load()
    for name, t, dt in (("x", x, torch.float32), ("dy", dy, torch.float32), ("dx", dx, torch.bfloat16)):
        _req(t, dt, name)
        if t.shape != x.shape or not t.is_contiguous() or t.dim() != 3:
            raise ValueError(f"{name} must be a contiguous (B, N, C) tensor of x's shape")
    B, N, Cn = x.shape
    _req_flat(weight, torch.float32, "weight", Cn)
    _req_flat(bias, torch.float32, "bias", Cn)
    partial = torch.empty(2 * B * Cn, device=x.device)
    dw, db = torch.empty(Cn, device=x.device), torch.empty(Cn, device=x.device)
    check(lib.ns2_groupnorm_silu_bwd(x.data_ptr(), B, N, Cn, int(groups), weight.data_ptr(), bias.data_ptr(), float(eps),
                                     dy.data_ptr(), dx.data_ptr(), partial.data_ptr(), dw.data_ptr(), db.data_ptr(),
                                     _stream(x)), "ns2_groupnorm_silu_bwd")
    return dw, db


def rowdot_bwd(x: torch.Tensor, w: torch.Tensor, pred: torch.Tensor, dpred: torch.Tensor,
               dx: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """Backward of `rowdot(..., relu=True)` from its output `pred`: dx (f32, x's shape) += d pre * w in place, returns
    (d w (dim,), d bias (1,)) f32, reduced in a fixed order.  d pre = d pred where pred > 0, else 0."""
    lib = _lib.load()
    for name, t in (("x", x), ("w", w), ("pred", pred), ("dpred", dpred), ("dx", dx)):
        _req(t, torch.float32, name)
        if not t.is_contiguous():
            raise ValueError(f"rowdot_bwd: {name} must be contiguous")
    dim = x.shape[-1]
    rows = pred.numel()
    if rows * dim != x.numel() or dpred.numel() != rows or dx.shape != x.shape or w.numel() != dim:
        raise ValueError("rowdot_bwd needs x (..., dim), w (dim,), pred / dpred one value per row, dx of x's shape")
    chunks = (rows + _lib.NS2_ROWDOT_BWD_ROWS - 1) // _lib.NS2_ROWDOT_BWD_ROWS
    partial = torch.empty(max(chunks, 1) * (dim + 4), device=x.device)
    dw, db = torch.empty(dim, device=x.device), torch.empty(1, device=x.device)
    check(lib.ns2_rowdot_bwd(x.data_ptr(), rows, dim, w.data_ptr(), pred.data_ptr(), dpred.data_ptr(), dx.data_ptr(),
                             partial.data_ptr(), dw.data_ptr(), db.data_ptr(), _stream(x)), "ns2_rowdot_bwd")
    return dw, db


def expand_encodings_bwd(dcond: torch.Tensor, coarse: torch.Tensor, idx: torch.Tensor, dphon: Optional[torch.Tensor],
                         dtable: Optional[torch.Tensor]):
    """Backward of `expand_encodings` given d cond TOKEN-MAJOR (B, L, D) f32 (unit channel stride, uniform row stride):
    dphon (B, T, D) += per-phoneme sums over its frames; dtable[coarse] += the same sums.  Both accumulate."""
    lib = _lib.load()
    _req(dcond, torch.float32, "dcond")
    _req(coarse, torch.int32, "coarse")
    _req(idx, torch.int32, "idx")
    B, L, D = dcond.shape
    if dcond.stride(2) != 1 or (B > 1 and dcond.stride(0) != L * dcond.stride(1)):
        raise ValueError("dcond must be (B, L, D) with unit channel stride and uniformly strided rows")
    T = coarse.shape[1]
    if not (coarse.is_contiguous() and idx.is_contiguous()) or coarse.shape[0] != B or tuple(idx.shape) != (B, L):
        raise ValueError("expand_encodings_bwd: coarse (B, T) and idx (B, L) must be contiguous int32")
    rows = 1
    for name, t in (("dphon", dphon), ("dtable", dtable)):
        if t is not None:
            _req(t, torch.float32, name)
            if not t.is_contiguous() or t.shape[-1] != D:
                raise ValueError(f"{name} must be contiguous with D columns")
    if dphon is not None and tuple(dphon.shape) != (B, T, D):
        raise ValueError("dphon must be (B, T, D)")
    if dtable is not None:
        rows = dtable.shape[0]
    check(lib.ns2_expand_encodings_bwd(dcond.data_ptr(), max(dcond.stride(1), D), coarse.data_ptr(), rows, idx.data_ptr(),
                                       B, T, D, L, _ptr(dphon), _ptr(dtable), _stream(dcond)), "ns2_expand_encodings_bwd")
    return dphon, dtable


def add_rows_bcast(x: torch.Tensor, v: torch.Tensor, scale: float = 1.0) -> torch.Tensor:
    """x[b, r, :] += scale * v[b, :] in place; x (B, R, D) f32 contiguous, v (B, D) f32 contiguous."""
    lib = _lib.load()
    _req(x, torch.float32, "x")
    _req(v, torch.float32, "v")
    B, R, D = x.shape
    if not (x.is_contiguous() and v.is_contiguous()) or tuple(v.shape) != (B, D):
        raise ValueError("add_rows_bcast: x (B, R, D) and v (B, D) must be contiguous")
    check(lib.ns2_add_rows_bcast(x.data_ptr(), B, R, D, v.data_ptr(), float(scale), _stream(x)), "ns2_add_rows_bcast")
    return x


# --------------------------------------------------------------------------------------------------
# Monotonic alignment search (aligner.py:88-122)
# --------------------------------------------------------------------------------------------------
def maximum_path(value: torch.Tensor, mask: torch.Tensor, neg_const: float = float("-inf"), *,
                 want_path: bool = True) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    """(idx (b, t_y) int32, path (b, t_x, t_y) f32 or None) for value/mask (b, t_x, t_y) f32 contiguous."""
    lib = _lib.load()
    _req(value, torch.float32, "value")
    _req(mask, torch.float32, "mask")
    if value.dim() != 3 or value.shape != mask.shape:
        raise ValueError(f"value and mask must both be (b, t_x, t_y); got {tuple(value.shape)} / {tuple(mask.shape)}")
    if not (value.is_contiguous() and mask.is_contiguous()):
        raise ValueError("value and mask must be contiguous")
    b, t_x, t_y = value.shape
    idx = torch.empty((b, t_y), dtype=torch.int32, device=value.device)
    path = torch.empty_like(value) if want_path else None
    ws_bytes = int(lib.ns2_maximum_path_workspace_bytes(b, t_x, t_y))
    ws = torch.empty(max(ws_bytes, 16), dtype=torch.uint8, device=value.device)
    check(lib.ns2_maximum_path(value.data_ptr(), mask.data_ptr(), b, t_x, t_y, float(neg_const), ws.data_ptr(),
                               ws_bytes, idx.data_ptr(), _ptr(path), _stream(value)), "ns2_maximum_path")
    return idx, path


# --------------------------------------------------------------------------------------------------
# SEANet decoder and encoder (Encodec 24 kHz): LSTM recurrence, conv operand preparation, 32-channel tail and head
# --------------------------------------------------------------------------------------------------
def _rows3(t: torch.Tensor, name: str, cols: int) -> Tuple[int, int]:
    """(row stride, batch stride) of a (B, T, >= cols) view with unit channel stride."""
    if t.dim() != 3 or t.shape[2] < cols or (t.shape[2] > 1 and t.stride(2) != 1):
        raise ValueError(f"{name} must be a (B, T, >= {cols}) view with unit channel stride, got {tuple(t.shape)}")
    return t.stride(1), t.stride(0)


def lstm_seq(xproj: torch.Tensor, w_hh: torch.Tensor, *, skip: Optional[torch.Tensor] = None,
             out: Optional[torch.Tensor] = None, out_bf16: Optional[torch.Tensor] = None) -> None:
    """One nn.LSTM(512, 512) layer over the sequence: xproj (B, T, 2048) f32 holds x W_ih^T + b_ih + b_hh in the
    kernel's gate order (see include/ns2_b200.h section 10), w_hh (2048, 512) bf16 in the same row order.
    Writes h_t (+ skip) into out (B, T, 512) f32 and/or out_bf16 (B, T, 512) bf16; all may be strided views."""
    lib = _lib.load()
    _req(xproj, torch.float32, "xproj")
    _req(w_hh, torch.bfloat16, "w_hh")
    if tuple(w_hh.shape) != (2048, 512) or not w_hh.is_contiguous():
        raise ValueError("w_hh must be a contiguous (2048, 512) bf16 tensor")
    if out is None and out_bf16 is None:
        raise ValueError("lstm_seq needs out and/or out_bf16")
    B, T = xproj.shape[:2]
    xrs, xbs = _rows3(xproj, "xproj", 2048)
    strides = {}
    for name, t, dt in (("skip", skip, torch.float32), ("out", out, torch.float32), ("out_bf16", out_bf16, torch.bfloat16)):
        if t is None:
            strides[name] = (0, 0)
            continue
        _req(t, dt, name)
        if t.shape[:2] != (B, T):
            raise ValueError(f"{name} must be (B, T, 512) like xproj's (B, T)")
        strides[name] = _rows3(t, name, 512)
    check(lib.ns2_lstm_seq(xproj.data_ptr(), xrs, xbs, w_hh.data_ptr(), B, T, 512, _ptr(skip), *strides["skip"],
                           _ptr(out), *strides["out"], _ptr(out_bf16), *strides["out_bf16"], _stream(xproj)),
          "ns2_lstm_seq")


def elu_pad(x: torch.Tensor, out: torch.Tensor, *, pad: int, elu: bool = True, raw: bool = False) -> torch.Tensor:
    """out[:, r, :C] = bf16(ELU(xpad[:, r - pad])) for r < pad + T (ELU only with elu=True), xpad = x reflect-padded
    on the left (Encodec's causal padding); raw=True also writes bf16(xpad) in columns [C, 2C).  x (B, T, C) f32 and
    out (B, pad + T, >= C or 2C) bf16 may be row-strided views (e.g. a GEMM output past its scratch rows)."""
    lib = _lib.load()
    _req(x, torch.float32, "x")
    _req(out, torch.bfloat16, "out")
    B, T, Cc = x.shape
    xrs, xbs = _rows3(x, "x", Cc)
    ors, obs = _rows3(out, "out", Cc * (2 if raw else 1))
    if out.shape[0] != B or out.shape[1] != pad + T:
        raise ValueError(f"out must have {pad + T} rows per batch element, got {tuple(out.shape)}")
    flags = (_lib.NS2_ELU_PAD_ELU if elu else 0) | (_lib.NS2_ELU_PAD_RAW if raw else 0)
    check(lib.ns2_elu_pad(x.data_ptr(), xrs, xbs, B, T, Cc, int(pad), flags, out.data_ptr(), ors, obs, _stream(out)),
          "ns2_elu_pad")
    return out


def seanet_tail(x: torch.Tensor, params: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """out (B, T) f32 = conv7(ELU(ResnetBlock(x))) for x (B, T, 32) f32 (row-strided view allowed); params: the
    NS2_SEANET_TAIL_PARAMS packed f32 weights (SEANetDecoder packs them)."""
    lib = _lib.load()
    _req(x, torch.float32, "x")
    _req(out, torch.float32, "out")
    _req_flat(params, torch.float32, "params", _lib.NS2_SEANET_TAIL_PARAMS)
    B, T, Cc = x.shape
    if Cc != 32:
        raise ValueError("seanet_tail takes 32 channels")
    xrs, xbs = _rows3(x, "x", 32)
    if out.dim() != 2 or tuple(out.shape) != (B, T) or (T > 1 and out.stride(1) != 1):
        raise ValueError("out must be (B, T) with unit time stride")
    check(lib.ns2_seanet_tail(x.data_ptr(), xrs, xbs, B, T, params.data_ptr(), out.data_ptr(), out.stride(0),
                              _stream(out)), "ns2_seanet_tail")
    return out


def seanet_head(x: torch.Tensor, params: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """out (B, T + 2, 32) bf16 = elu_pad(ResnetBlock(conv7(x)), pad=2) for audio x (B, T) f32 (unit time stride,
    any batch stride): the encoder's full-rate stage, ready as the first strided conv's A operand.  params: the
    NS2_SEANET_HEAD_PARAMS packed f32 weights (SEANetEncoder packs them).  out may be a row-strided view."""
    lib = _lib.load()
    _req(x, torch.float32, "x")
    _req(out, torch.bfloat16, "out")
    _req_flat(params, torch.float32, "params", _lib.NS2_SEANET_HEAD_PARAMS)
    if x.dim() != 2:
        raise ValueError(f"seanet_head takes (B, T) audio, got {tuple(x.shape)}")
    B, T = x.shape
    ors, obs = _rows3(out, "out", 32)
    if tuple(out.shape) != (B, T + 2, 32):
        raise ValueError(f"out must be (B, T + 2, 32) = {(B, T + 2, 32)}, got {tuple(out.shape)}")
    check(lib.ns2_seanet_head(x.data_ptr(), x.stride(0), B, T, params.data_ptr(), out.data_ptr(), ors, obs,
                              _stream(out)), "ns2_seanet_head")
    return out
