"""torch-tensor front end of the C ABI (include/ns2_b200.h).

Every function takes CUDA tensors and enqueues ONE library call on the current torch CUDA stream.  Before that it
states each tensor argument through `_check` (dtype, shape, layout, alignment, current device) and compares related
arguments explicitly, so that no kernel touches memory outside the tensors it was given; a failed check raises
ValueError and launches nothing.  Nothing here computes on the host or falls back to PyTorch math: if the library is
missing, `_lib.load()` raises.
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


F32, BF16, I32, I64 = torch.float32, torch.bfloat16, torch.int32, torch.int64
DENSE, ROWS, LAST = "dense", "rows", "last"   # layouts of `_check`


def _check(*specs) -> None:
    """Check an op's tensor arguments.  Each spec is (name, tensor, dtype, shape, layout[, align]):
      tensor  None for an optional argument that was not given, which passes;
      shape   a tuple of ints and None (any size), or None for any rank and sizes;
      layout  DENSE: contiguous.  ROWS: unit channel (last) stride, and every leading dim of more than one entry
              uniformly strided, so the rows of all batches form one strided matrix.  LAST: unit channel stride only;
      align   the byte alignment of the data pointer (vector loads and stores, e.g. float4 = 16).
    Dtype, shape and layout are checked on every argument before any device, so a malformed call fails the same way on
    a machine without a GPU.  Then every tensor must be on the current CUDA device: the library launches there (tensor
    maps, kernel attributes and the SM count are per device), so wrap a call in `torch.cuda.device(t.device)`."""
    # plain loops instead of generator expressions: this runs before every eager launch
    for spec in specs:
        name, t, dtype, shape, layout = spec[:5]
        if t is None:
            continue
        if not isinstance(t, torch.Tensor):
            raise ValueError(f"{name} must be a tensor, got {type(t).__name__}")
        if t.dtype != dtype:
            raise ValueError(f"{name} must be {dtype}, got {t.dtype}")
        size = t.shape
        if shape is not None:
            ok = len(size) == len(shape)
            for want, n in zip(shape, size):
                if want is not None and want != n:
                    ok = False
            if not ok:
                want = ", ".join("*" if s is None else str(s) for s in shape)
                raise ValueError(f"{name} must have shape ({want}), got {tuple(size)}")
        if layout is ROWS or not t.is_contiguous():
            if layout is DENSE:
                raise ValueError(f"{name} must be contiguous")
            stride = t.stride()
            if size and size[-1] > 1 and stride[-1] != 1:
                raise ValueError(f"{name} must be contiguous in its last dimension")
            if layout is ROWS:
                for i in range(len(size) - 2):
                    if size[i] > 1 and stride[i] != size[i + 1] * stride[i + 1]:
                        raise ValueError(f"{name} must have uniformly strided rows")
        if len(spec) > 5 and t.data_ptr() % spec[5]:
            raise ValueError(f"{name} must be {spec[5]}-byte aligned")
    device = None
    for spec in specs:
        t = spec[1]
        if t is None:
            continue
        if not t.is_cuda:
            raise ValueError(f"{spec[0]} must be a CUDA tensor (the ns2_b200 ops have no CPU path)")
        if device is None:
            device = torch.cuda.current_device()
        if t.get_device() != device:
            raise ValueError(f"{spec[0]} is on {t.device} but the current CUDA device is cuda:{device}")


def _stream() -> int:
    """Raw handle of torch's current stream."""
    return torch.cuda.current_stream().cuda_stream


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


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
         dil: Optional[Sequence[int]] = None, flags: int = 0,
         row_lens: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out = epilogue(segmented_gemm(a, w)).  `a`: (batches, rows, cols) bf16 (may be a strided view),
    `w`: packed bf16 weight (rows, K).  See include/ns2_b200.h section 1 for the exact semantics.
    row_lens: int32 CUDA (batches,) in [1, rows], at most NS2_GEMM_ROW_LENS_MAX_BATCHES batches: only the 128-row tiles
    of batch b that start before row_lens[b] are computed (bit-identical to the call without it); rows of the other
    tiles of `out` are left as they were."""
    lib = _lib.load()
    # the epilogue reads bias[g * b_group_row_stride + col] for every output column col < n (and + bias1_off)
    need = (groups - 1) * b_group_row_stride + n + (bias1_off if epilogue == EPI_WAVENET else 0)
    if bias is not None and bias.numel() < need:
        raise ValueError(f"bias must have >= {need} elements for n={n}, got {bias.numel()}")
    Ba, M, _ = a.shape
    if row_lens is not None and Ba > _lib.NS2_GEMM_ROW_LENS_MAX_BATCHES:
        raise ValueError(f"row_lens: at most {_lib.NS2_GEMM_ROW_LENS_MAX_BATCHES} batches, got {Ba}")
    _check(("a", a, BF16, None, LAST), ("w", w, BF16, (None, None), LAST),
           ("out", out, F32 if epilogue == EPI_F32 else BF16, (Ba, M, None), ROWS), ("bias", bias, F32, None, DENSE),
           ("resid", resid, F32, out.shape, ROWS), ("film", film, F32, None, LAST),
           ("row_lens", row_lens, I32, (Ba,), DENSE))
    lens_ptr = _check_lens(row_lens, 1, M, "row_lens")
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
    args.bias = _ptr(bias)
    args.bias1_off = bias1_off
    args.out = out.data_ptr()
    args.out_row_stride = out.stride(1)
    if resid is not None:
        args.resid_row_stride = resid.stride(1)
    args.resid = _ptr(resid)
    if film is not None:
        args.film_batch_stride = film.stride(0)
    args.film = _ptr(film)
    args.film_group_stride = film_group_stride
    args.flags = int(flags)
    args.row_lens = lens_ptr
    check(lib.ns2_gemm(C.byref(args), _stream()), "ns2_gemm")
    return out


def wgrad(dy: torch.Tensor, x: torch.Tensor, dw: torch.Tensor, *, n: int, k: int, shift_units: int = 0,
          x_col_off: int = 0, groups: int = 1, dy_group_col_stride: int = 0, x_group_col_stride: int = 0,
          dw_group_row_stride: int = 0, dil: Optional[Sequence[int]] = None, splits: int = 0) -> torch.Tensor:
    """dw[g][:n, :k] += dy[..., g-th n columns]^T @ x[..., rows shifted by shift_units*dil[g], g-th k columns].
    dy, x: (batches, rows, cols) bf16 (strided views are fine); dw: fp32 2-D (rows >= groups' n rows, cols >= k)."""
    lib = _lib.load()
    if groups > 1 and n % 128 != 0:
        raise ValueError("wgrad: n must be a multiple of 128 for grouped weights")
    Bd, R, _ = dy.shape
    _check(("dy", dy, BF16, None, LAST), ("x", x, BF16, (Bd, R, None), LAST), ("dw", dw, F32, (None, None), LAST))
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
    check(lib.ns2_wgrad(C.byref(args), _stream()), "ns2_wgrad")
    return dw


def fold_conv_linear(w2: torch.Tensor, wc: torch.Tensor, bc: torch.Tensor, b2: torch.Tensor, i_pad: int):
    """Stacked (conv, Linear) pairs with nothing between them as one conv each (include/ns2_b200.h section 1c):
    w2 (L, O, K), wc (L, K, I, taps), bc (L, K), b2 (L, O) fp32 -> (bf16 (L, O, taps*i_pad) tap-major pack of the taps
    w2 @ wc[..., t], zero-padded from I to i_pad; fp32 (L, O) bias w2 @ bc + b2)."""
    lib = _lib.load()
    L, O, K = w2.shape
    _check(("w2", w2, F32, None, DENSE), ("wc", wc, F32, (L, K, None, None), DENSE), ("bc", bc, F32, (L, K), DENSE),
           ("b2", b2, F32, (L, O), DENSE))
    _, _, I, taps = wc.shape
    if i_pad < I:
        raise ValueError(f"fold_conv_linear: i_pad {i_pad} < {I} input channels")
    out = torch.empty(L, O, taps * i_pad, device=w2.device, dtype=torch.bfloat16)
    bias = torch.empty(L, O, device=w2.device, dtype=torch.float32)
    check(lib.ns2_fold_conv_linear(w2.data_ptr(), wc.data_ptr(), bc.data_ptr(), b2.data_ptr(), L, O, K, I, taps, i_pad,
                                   out.data_ptr(), bias.data_ptr(), _stream()), "ns2_fold_conv_linear")
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
    _check(("x", x, F32, None, DENSE, 16))
    d = _dropout_args(dropout)
    if d is not None:
        check(lib.ns2_dropout_f32(x.data_ptr(), x.numel(), C.byref(d), _stream()), "ns2_dropout_f32")
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


def _check_lens(lens: Optional[torch.Tensor], lo: int, hi: Optional[int], name: str) -> Optional[int]:
    """Check that per-sample lengths lie in [lo, hi] before a ragged launch, after `_check` has passed `lens` as an int32
    (B,) tensor on the device.  The range is read once per tensor version (one device sync) and remembered on the
    tensor; while a CUDA graph is being captured values cannot be read, and the kernels clamp them instead.  Returns the
    data pointer (None for no lengths)."""
    if lens is None:
        return None
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
    B, N, Cc = x.shape
    _check(("x", x, BF16 if x.dtype == BF16 else F32, None, LAST), ("lens", lens, I32, (B,), DENSE))
    lp = _check_lens(lens, 0, N, "lens")
    check(lib.ns2_mask_rows(x.data_ptr(), int(x.dtype == torch.float32), x.stride(1), x.stride(0), B, N, Cc, lp,
                            _stream()), "ns2_mask_rows")
    return x


def pack_rows(a: torch.Tensor, a_lens: torch.Tensor, b: torch.Tensor, b_lens: torch.Tensor,
              out: torch.Tensor) -> torch.Tensor:
    """bf16 out[s] = [a[s, :a_lens[s]] ; b[s, :b_lens[s]] ; 0]: two end-padded segments (B, Na, C), (B, Nb, C) as one
    prefix of length a_lens + b_lens of out (B, No >= Na + Nb, C).  Row- and batch-strided views are fine."""
    lib = _lib.load()
    B, Na, Cc = a.shape
    _check(("a", a, BF16, None, LAST), ("b", b, BF16, (B, None, Cc), LAST), ("out", out, BF16, (B, None, Cc), LAST),
           ("a_lens", a_lens, I32, (B,), DENSE), ("b_lens", b_lens, I32, (B,), DENSE))
    Nb, No = b.shape[1], out.shape[1]
    if No < Na + Nb:
        raise ValueError(f"out holds {No} rows, fewer than {Na} + {Nb}")
    ap = _check_lens(a_lens, 0, Na, "a_lens")
    bp = _check_lens(b_lens, 0, Nb, "b_lens")
    check(lib.ns2_pack_rows(a.data_ptr(), a.stride(1), a.stride(0), Na, ap, b.data_ptr(), b.stride(1), b.stride(0), Nb,
                            bp, B, Cc, out.data_ptr(), out.stride(1), out.stride(0), No, _stream()), "ns2_pack_rows")
    return out


# --------------------------------------------------------------------------------------------------
# attention
# --------------------------------------------------------------------------------------------------
def attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, out: torch.Tensor, *, heads: int,
              scale: Optional[float] = None, lse: Optional[torch.Tensor] = None,
              dropout: Optional[DropoutSpec] = None, kv_lens: Optional[torch.Tensor] = None,
              q_lens: Optional[torch.Tensor] = None) -> torch.Tensor:
    """q: (B, Nq, heads*64), k/v: (B, Nk, heads*64) bf16 (strided views into a fused projection are fine).
    dropout=(seed, site, p): attention dropout on the softmax probabilities (lse stays that of the undropped ones).
    kv_lens: int32 CUDA (B,) in [1, Nk]: sample b attends to its keys [0, kv_lens[b]) only (K / V rows past it must be
    finite); its output is bit-identical to the call on that sample's keys alone.  No dropout with kv_lens.
    q_lens: int32 CUDA (B,) in [1, Nq]: the 128-query tiles of sample b that start at or past q_lens[b] are skipped
    (their out rows and lse entries are left as they were); the other rows are bit-identical to the call without it.
    No dropout with q_lens."""
    lib = _lib.load()
    if (kv_lens is not None or q_lens is not None) and dropout is not None:
        raise ValueError("attention: dropout with kv_lens or q_lens is not supported")
    inner = heads * 64
    B, Nq, _ = q.shape
    _, Nk, _ = k.shape
    _check(("q", q, BF16, (B, Nq, inner), LAST), ("k", k, BF16, (B, Nk, inner), LAST), ("v", v, BF16, (B, Nk, inner), LAST),
           ("out", out, BF16, (B, Nq, inner), LAST), ("lse", lse, F32, (B, heads, Nq), DENSE),
           ("kv_lens", kv_lens, I32, (B,), DENSE), ("q_lens", q_lens, I32, (B,), DENSE))
    lens_ptr = _check_lens(kv_lens, 1, Nk, "kv_lens")
    q_lens_ptr = _check_lens(q_lens, 1, Nq, "q_lens")
    args = AttnArgs()
    args.q, args.q_row_stride, args.q_batch_stride = q.data_ptr(), q.stride(1), q.stride(0)
    args.k, args.k_row_stride, args.k_batch_stride = k.data_ptr(), k.stride(1), k.stride(0)
    args.v, args.v_row_stride, args.v_batch_stride = v.data_ptr(), v.stride(1), v.stride(0)
    args.out, args.o_row_stride, args.o_batch_stride = out.data_ptr(), out.stride(1), out.stride(0)
    args.batches, args.heads = q.shape[0], heads
    args.q_len, args.kv_len, args.dim_head = q.shape[1], k.shape[1], 64
    args.scale = float(scale if scale is not None else 64 ** -0.5)
    args.lse, args.kv_lens, args.q_lens = _ptr(lse), lens_ptr, q_lens_ptr
    d = _dropout_args(dropout)
    args.dropout = None if d is None else C.pointer(d)
    check(lib.ns2_attn_fwd(C.byref(args), _stream()), "ns2_attn_fwd")
    return out


# --------------------------------------------------------------------------------------------------
# norms, small layers, casts
# --------------------------------------------------------------------------------------------------
def rmsnorm_film(x: torch.Tensor, out: torch.Tensor, *, gamma: Optional[torch.Tensor] = None,
                 film: Optional[torch.Tensor] = None, lens: Optional[torch.Tensor] = None) -> torch.Tensor:
    """x: (B, N, D) f32 -> out (B, N, D) bf16.  film: (B, >=2D) f32 view whose row b holds [gamma_b | beta_b].
    lens: int32 CUDA (B,) in [1, N]: only rows [0, lens[b]) of sample b are normalized (bit-identical to the call without
    it); the other rows of `out` are left as they were."""
    lib = _lib.load()
    B, N, D = x.shape
    if film is not None and film.shape[-1] < 2 * D:
        raise ValueError(f"film must have >= {2 * D} columns, got {tuple(film.shape)}")
    _check(("x", x, F32, None, DENSE), ("out", out, BF16, (B, N, D), DENSE), ("gamma", gamma, F32, (D,), DENSE),
           ("film", film, F32, (B, None), LAST), ("lens", lens, I32, (B,), DENSE))
    lens_ptr = _check_lens(lens, 1, N, "lens")
    film_bs = 0 if film is None else film.stride(0)
    check(lib.ns2_rmsnorm_film(x.data_ptr(), D, B * N, D, N, _ptr(gamma), _ptr(film), film_bs,
                               out.data_ptr(), D, lens_ptr, _stream()), "ns2_rmsnorm_film")
    return out


def rmsnorm_f32(x: torch.Tensor, out: torch.Tensor, gamma: Optional[torch.Tensor]) -> torch.Tensor:
    """out (f32, x's shape) = RMSNorm(x) (* gamma) over the last dimension; x and out contiguous."""
    lib = _lib.load()
    D = x.shape[-1]
    if out.numel() != x.numel() or (gamma is not None and gamma.numel() != D):
        raise ValueError(f"out must hold x's {x.numel()} elements and gamma {D}")
    _check(("x", x, F32, None, DENSE, 16), ("out", out, F32, None, DENSE, 16), ("gamma", gamma, F32, None, DENSE, 16))
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
    B, half, n_out = times.numel(), freqs.numel(), w.shape[0]
    _check(("times", times, F32, (B,), DENSE), ("freqs", freqs, F32, (half,), DENSE),
           ("w", w, F32, (n_out, 2 * half + 1), DENSE), ("bias", bias, F32, (n_out,), DENSE),
           ("out", out, F32, (B, n_out), LAST))
    step = _small_chunk(2 * half + 1)
    for b0 in range(0, B, step):
        tb, ob = times[b0:b0 + step], out[b0:b0 + step]
        check(lib.ns2_time_cond(tb.data_ptr(), tb.shape[0], freqs.data_ptr(), half, w.data_ptr(),
                                bias.data_ptr(), n_out, ob.data_ptr(), out.stride(0), _stream()),
              "ns2_time_cond")
    return out


def small_linear(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor], out: torch.Tensor,
                 act: int = 0) -> torch.Tensor:
    lib = _lib.load()
    B, k = x.shape
    n_out = w.shape[0]
    _check(("x", x, F32, None, LAST), ("w", w, F32, (n_out, k), DENSE), ("bias", bias, F32, (n_out,), DENSE),
           ("out", out, F32, (B, n_out), LAST))
    step = _small_chunk(k)
    for b0 in range(0, B, step):
        xb, ob = x[b0:b0 + step], out[b0:b0 + step]
        check(lib.ns2_small_linear(xb.data_ptr(), x.stride(0), xb.shape[0], k, w.data_ptr(), _ptr(bias),
                                   n_out, act, ob.data_ptr(), out.stride(0), _stream()), "ns2_small_linear")
    return out


def cast_bf16(x: torch.Tensor, out: torch.Tensor, add: Optional[torch.Tensor] = None) -> torch.Tensor:
    lib = _lib.load()
    n = x.numel()
    if out.numel() != n or (add is not None and add.numel() != n):
        raise ValueError(f"out and add must hold x's {n} elements")
    _check(("x", x, F32, None, DENSE), ("out", out, BF16, None, DENSE), ("add", add, F32, None, DENSE))
    check(lib.ns2_cast_bf16(x.data_ptr(), _ptr(add), n, out.data_ptr(), _stream()),
          "ns2_cast_bf16")
    return out


def cond_inject(x: torch.Tensor, cproj: torch.Tensor, out: torch.Tensor, drop_mask: Optional[torch.Tensor] = None,
                null_cond: Optional[torch.Tensor] = None, *, cond_lens: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out (B, N, D) bf16 = x (B, N, D) f32 + [padded / curtailed, null-substituted] cproj (B, L, D) f32.
    cond_lens: int32 CUDA (B,) >= 0: sample b's condition ends at frame min(L, cond_lens[b])."""
    lib = _lib.load()
    B, N, D = x.shape
    if drop_mask is not None and (null_cond is None or drop_mask.numel() != B or null_cond.numel() != D):
        raise ValueError(f"drop_mask must hold {B} values and null_cond {D}")
    _check(("x", x, F32, None, DENSE), ("cproj", cproj, F32, (B, None, D), DENSE), ("out", out, BF16, (B, N, D), DENSE),
           ("drop_mask", drop_mask, torch.bool, None, DENSE), ("null_cond", null_cond, F32, None, DENSE),
           ("cond_lens", cond_lens, I32, (B,), DENSE))
    lp = _check_lens(cond_lens, 0, None, "cond_lens")
    check(lib.ns2_cond_inject(x.data_ptr(), cproj.data_ptr(), _ptr(drop_mask), _ptr(null_cond), B, N, cproj.shape[1], D,
                              out.data_ptr(), lp, _stream()), "ns2_cond_inject")
    return out


def select_rows(drop_mask: torch.Tensor, null_row: torch.Tensor, src: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """out[b] = null_row if drop_mask[b] else src[b]; src/out are (B, ...) with contiguous trailing dims; out may be a
    column slice of a wider f32 matrix (row stride > row length) or a bf16 tensor."""
    lib = _lib.load()
    B = src.shape[0]
    row_len = src.numel() // B
    if drop_mask.numel() != B or null_row.numel() != row_len or out.shape[0] != B or out.numel() != B * row_len:
        raise ValueError(f"drop_mask must hold {B} values, and null_row and each row of out {row_len}")
    _check(("drop_mask", drop_mask, torch.bool, None, DENSE), ("null_row", null_row, F32, None, DENSE),
           ("src", src, F32, None, DENSE),
           ("out", out, BF16 if out.dtype == BF16 else F32, None, DENSE if out.dim() > 2 else LAST))
    check(lib.ns2_select_rows(drop_mask.data_ptr(), null_row.data_ptr(), src.data_ptr(), row_len, B, row_len,
                              out.data_ptr(), out.stride(0), int(out.dtype == torch.bfloat16), _stream()),
          "ns2_select_rows")
    return out


def mean_rows(x: torch.Tensor, out: torch.Tensor, *, lens: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out (B, D) = mean over the rows of x (B, N, D) f32; lens: int32 CUDA (B,) in [1, N], the mean of sample b over
    its rows [0, lens[b])."""
    lib = _lib.load()
    B, N, D = x.shape
    _check(("x", x, F32, None, LAST), ("out", out, F32, (B, D), DENSE), ("lens", lens, I32, (B,), DENSE))
    lp = _check_lens(lens, 1, N, "lens")
    check(lib.ns2_mean_rows(x.contiguous().data_ptr(), B, N, D, out.data_ptr(), lp, _stream()), "ns2_mean_rows")
    return out


def transpose_cast(x: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """(B, C, L) f32 channel-first -> (B, L, C) bf16."""
    lib = _lib.load()
    B, Cc, L = x.shape
    _check(("x", x, F32, None, LAST), ("out", out, BF16, (B, L, Cc), DENSE))
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
    if out_f32 is None and out_bf16 is None:
        raise ValueError("groupnorm_silu needs at least one output")
    B, N, Cn = x.shape
    _check(("x", x, F32, None, DENSE), ("weight", weight, F32, (Cn,), DENSE), ("bias", bias, F32, (Cn,), DENSE),
           ("resid", resid, F32, (B, N, Cn), DENSE), ("out_f32", out_f32, F32, (B, N, Cn), DENSE),
           ("out_bf16", out_bf16, BF16, (B, N, Cn), DENSE), ("lens", lens, I32, (B,), DENSE))
    lp = _check_lens(lens, 1, N, "lens")
    check(lib.ns2_groupnorm_silu(x.data_ptr(), B, N, Cn, int(groups), weight.data_ptr(), bias.data_ptr(), float(eps),
                                 _ptr(resid), _ptr(out_f32), _ptr(out_bf16), lp, _stream()), "ns2_groupnorm_silu")
    return out_f32, out_bf16


def rowdot(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor], out: torch.Tensor, relu: bool = False):
    """out[...] = (relu)(x[..., :] . w + bias): Linear(dim, 1) heads.  x f32 contiguous, w (dim,), out one value per row."""
    lib = _lib.load()
    dim = x.shape[-1]
    if out.numel() * dim != x.numel() or w.numel() != dim or (bias is not None and bias.numel() != 1):
        raise ValueError("rowdot needs x (..., dim), w (dim,), one bias and one output per row")
    _check(("x", x, F32, None, DENSE), ("w", w, F32, None, DENSE), ("bias", bias, F32, None, DENSE),
           ("out", out, F32, None, DENSE))
    check(lib.ns2_rowdot(x.data_ptr(), out.numel(), dim, w.data_ptr(), _ptr(bias), int(relu), out.data_ptr(),
                         _stream()), "ns2_rowdot")
    return out


def expand_encodings(phon: torch.Tensor, coarse: torch.Tensor, pitch_table: torch.Tensor, idx: torch.Tensor) -> torch.Tensor:
    """(B, D, L) f32 channel-first: phon[b, idx[b, n], :] + pitch_table[coarse[b, idx[b, n]], :], 0 where idx < 0
    (expand_encodings, ns2.py:1449-1455).  phon (B, T, D) f32, coarse (B, T) int32, idx (B, L) int32."""
    lib = _lib.load()
    B, T, D = phon.shape
    _check(("phon", phon, F32, None, DENSE), ("coarse", coarse, I32, (B, T), DENSE),
           ("pitch_table", pitch_table, F32, (None, D), DENSE), ("idx", idx, I32, (B, None), DENSE))
    L = idx.shape[1]
    out = torch.empty(B, D, L, device=phon.device, dtype=torch.float32)
    check(lib.ns2_expand_encodings(phon.data_ptr(), coarse.data_ptr(), pitch_table.data_ptr(), pitch_table.shape[0],
                                   idx.data_ptr(), B, T, D, L, out.data_ptr(), _stream()), "ns2_expand_encodings")
    return out


def embedding_bf16(ids: torch.Tensor, table: torch.Tensor, out: torch.Tensor, pad_id: int) -> torch.Tensor:
    """out[..., :] = bf16(table[ids < 0 ? pad_id : ids]) — nn.Embedding + padding substitution (ns2.py:279-282)."""
    lib = _lib.load()
    rows, D = table.shape
    if out.numel() != ids.numel() * D:
        raise ValueError("out must hold one table row per id")
    _check(("ids", ids, I64, None, DENSE), ("table", table, F32, None, DENSE), ("out", out, BF16, None, DENSE))
    check(lib.ns2_embedding_bf16(ids.data_ptr(), ids.numel(), table.data_ptr(), rows, D,
                                 int(pad_id), out.data_ptr(), _stream()), "ns2_embedding_bf16")
    return out


def q_sample(x0, noise, alpha, sigma, x_t, target=None, objective: str = "v"):
    """x_t = alpha x0 + sigma noise; target of the chosen parameterisation (ns2.py:1631-1644)."""
    lib = _lib.load()
    B, n = x0.shape[0], x0.numel()
    if any(t is not None and t.numel() != n for t in (noise, x_t, target)) or alpha.numel() != B or sigma.numel() != B:
        raise ValueError(f"noise, x_t and target must hold x0's {n} elements, alpha and sigma {B}")
    _check(("x0", x0, F32, None, DENSE, 16), ("noise", noise, F32, None, DENSE, 16), ("x_t", x_t, F32, None, DENSE, 16),
           ("target", target, F32, None, DENSE, 16), ("alpha", alpha, F32, None, DENSE),
           ("sigma", sigma, F32, None, DENSE))
    check(lib.ns2_q_sample(x0.data_ptr(), noise.data_ptr(), alpha.data_ptr(), sigma.data_ptr(), B, n // B,
                           x_t.data_ptr(), _ptr(target), OBJECTIVES[objective], _stream()), "ns2_q_sample")
    return x_t, target


def mse_rows(pred, target, out, scratch=None, mean_out=None, lens=None):
    """out[b] = mean((pred[b] - target[b])^2); `mean_out` (0-d / 1-element f32) additionally receives out.mean().
    lens: int32 CUDA (B,) in [1, N] for pred (B, N, ...): out[b] is the mean over sample b's first lens[b] rows,
    bit-identical to the call on pred[b:b+1, :lens[b]]; the rest is not read."""
    lib = _lib.load()
    B, n = pred.shape[0], pred.numel()
    if scratch is None:
        scratch = torch.empty(B * NS2_MSE_SCRATCH_PER_SAMPLE, device=pred.device, dtype=torch.float32)
    if scratch.numel() < B * NS2_MSE_SCRATCH_PER_SAMPLE:
        raise ValueError(f"scratch must hold >= {B * NS2_MSE_SCRATCH_PER_SAMPLE} elements, got {scratch.numel()}")
    if mean_out is not None and mean_out.numel() != 1:
        raise ValueError(f"mean_out must hold one element, got {mean_out.numel()}")
    _check(("pred", pred, F32, None, DENSE), ("target", target, F32, tuple(pred.shape), DENSE),
           ("out", out, F32, (B,), DENSE), ("scratch", scratch, F32, None, DENSE), ("mean_out", mean_out, F32, None, DENSE),
           ("lens", lens, I32, (B,), DENSE))
    rows, lp = _rows_lens(pred, lens)
    check(lib.ns2_mse_rows(pred.data_ptr(), target.data_ptr(), B, n // B, scratch.data_ptr(),
                           out.data_ptr(), _ptr(mean_out), n // B // rows, lp, _stream()), "ns2_mse_rows")
    return out


def _rows_lens(pred: torch.Tensor, lens: Optional[torch.Tensor]) -> Tuple[int, Optional[int]]:
    """(rows per sample, checked lengths pointer) of a (B, N, ...) tensor whose samples are lens[b] rows long."""
    if lens is None:
        return 1, None
    if pred.dim() < 2:
        raise ValueError(f"pred must be (B, N, ...) with lens, got {tuple(pred.shape)}")
    rows = pred.shape[1]
    if (pred.numel() // pred.shape[0] // rows) % 4:
        raise ValueError(f"pred rows must hold a multiple of 4 elements with lens, got {tuple(pred.shape)}")
    return rows, _check_lens(lens, 1, rows, "lens")


def ddim_step(x, v, alpha, sigma, alpha_next, sigma_next, objective: str = "v"):
    """In-place DDIM update of x from the model output `v` (ns2.py:1412-1429)."""
    lib = _lib.load()
    B, n = x.shape[0], x.numel()
    if v.numel() != n or any(t.numel() != B for t in (alpha, sigma, alpha_next, sigma_next)):
        raise ValueError(f"v must hold x's {n} elements, alpha, sigma, alpha_next and sigma_next {B}")
    _check(("x", x, F32, None, DENSE, 16), ("v", v, F32, None, DENSE, 16), ("alpha", alpha, F32, None, DENSE),
           ("sigma", sigma, F32, None, DENSE), ("alpha_next", alpha_next, F32, None, DENSE),
           ("sigma_next", sigma_next, F32, None, DENSE))
    check(lib.ns2_ddim_step(x.data_ptr(), v.data_ptr(), alpha.data_ptr(), sigma.data_ptr(),
                            alpha_next.data_ptr(), sigma_next.data_ptr(), B, n // B, OBJECTIVES[objective],
                            _stream()),
          "ns2_ddim_step")
    return x


def x_start_from_pred(x, pred, alpha, sigma, out, objective: str = "v"):
    """x_start implied by the model output under the chosen parameterisation (ns2.py:1673-1680)."""
    lib = _lib.load()
    B, n = x.shape[0], x.numel()
    if pred.numel() != n or out.numel() != n or alpha.numel() != B or sigma.numel() != B:
        raise ValueError(f"pred and out must hold x's {n} elements, alpha and sigma {B}")
    _check(("x", x, F32, None, DENSE, 16), ("pred", pred, F32, None, DENSE, 16), ("out", out, F32, None, DENSE, 16),
           ("alpha", alpha, F32, None, DENSE), ("sigma", sigma, F32, None, DENSE))
    check(lib.ns2_x_start(x.data_ptr(), pred.data_ptr(), alpha.data_ptr(), sigma.data_ptr(), B, n // B, out.data_ptr(),
                          OBJECTIVES[objective], _stream()), "ns2_x_start")
    return out


def cfg_combine(cond, null, scale, out):
    """out = null + (cond - null) * scale (classifier-free guidance); out may be cond or null itself."""
    lib = _lib.load()
    n = cond.numel()
    if null.numel() != n or out.numel() != n:
        raise ValueError(f"null and out must hold cond's {n} elements")
    _check(("cond", cond, F32, None, DENSE, 16), ("null", null, F32, None, DENSE, 16), ("out", out, F32, None, DENSE, 16))
    check(lib.ns2_cfg_combine(cond.data_ptr(), null.data_ptr(), float(scale), n,
                              out.data_ptr(), _stream()), "ns2_cfg_combine")
    return out


# --------------------------------------------------------------------------------------------------
# RVQ
# --------------------------------------------------------------------------------------------------
def rvq_prepare(codebooks: torch.Tensor):
    """codebooks (Q, K, 128) f32 -> (fp16 copy, ||c||^2 (Q, K) f32, meta (Q, 2) f32)."""
    lib = _lib.load()
    _check(("codebooks", codebooks, F32, (None, None, None), LAST))
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
    cb16, cn2, meta = prepared
    cb = codebooks.contiguous()
    Q, K, D = cb.shape
    F = frames.shape[0]
    if codes is None:
        codes = torch.empty((F, Q), device=frames.device, dtype=torch.int64)
    if stats is not None and stats.numel() < _lib.NS2_RVQ_STATS_LEN:
        raise ValueError(f"stats must have >= {_lib.NS2_RVQ_STATS_LEN} elements, got {stats.numel()}")
    _check(("frames", frames, F32, (F, D), LAST), ("codebooks", cb, F32, None, DENSE),
           ("cb16", cb16, torch.float16, None, DENSE), ("cn2", cn2, F32, None, DENSE), ("meta", meta, F32, None, DENSE),
           ("codes", codes, I64, (F, Q), DENSE), ("stats", stats, I64, None, DENSE))
    fr = frames.contiguous()
    check(lib.ns2_rvq_encode(fr.data_ptr(), F, D, cb.data_ptr(), cb16.data_ptr(), cn2.data_ptr(),
                             meta.data_ptr(), Q, K, codes.data_ptr(), _ptr(stats), _stream()),
          "ns2_rvq_encode")
    return codes


def rvq_decode(codes: torch.Tensor, codebooks: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """codes (F, Q) int64 -> emb (F, 128) f32 = sum_q codebooks[q, codes[:, q]], added in order q = 0..Q-1.  Codes
    outside [0, K) are clamped to 0 / K - 1.  `out` (optional) is a contiguous (F, 128) f32 tensor."""
    lib = _lib.load()
    F, Q = codes.shape[0], codebooks.shape[0]
    if out is None:
        out = torch.empty((F, 128), device=codes.device, dtype=torch.float32)
    # codebooks and out are read / written as float4
    _check(("codes", codes, I64, (None, Q), DENSE), ("codebooks", codebooks, F32, (None, None, 128), DENSE, 16),
           ("out", out, F32, (F, 128), DENSE, 16))
    _, K, D = codebooks.shape
    check(lib.ns2_rvq_decode(codes.data_ptr(), F, Q, K, D, codebooks.data_ptr(), out.data_ptr(), _stream()),
          "ns2_rvq_decode")
    return out


def _rvq_ce_args(frames, codebooks, cn2, own_codes, target_codes):
    """What rvq_ce and rvq_ce_bwd share: (frames, codebooks) contiguous, F, Q, K and the `_check` specs of the five."""
    fr, cb = frames.contiguous(), codebooks.contiguous()
    F, Q, K = fr.shape[0], cb.shape[0], cb.shape[1]
    specs = (("frames", fr, F32, (None, 128), DENSE), ("codebooks", cb, F32, (None, None, 128), DENSE),
             ("cn2", cn2, F32, (Q, K), DENSE), ("own_codes", own_codes, I64, (F, Q), DENSE),
             ("target_codes", target_codes, I64, (F, Q), DENSE))
    return fr, cb, F, Q, K, specs


def rvq_ce(frames: torch.Tensor, codebooks: torch.Tensor, cn2: torch.Tensor, own_codes: torch.Tensor,
           target_codes: torch.Tensor) -> torch.Tensor:
    """Cross-entropy head of the residual VQ (`codec.rq`): frames (F, 128) f32, codebooks (Q, K, 128) f32, their
    squared norms cn2 (Q, K) f32, codes (F, Q) int64 -> 0-d loss."""
    lib = _lib.load()
    fr, cb, F, Q, K, specs = _rvq_ce_args(frames, codebooks, cn2, own_codes, target_codes)
    _check(*specs)
    scratch = torch.empty(F * Q, device=fr.device, dtype=torch.float32)
    loss = torch.empty((), device=fr.device, dtype=torch.float32)
    check(lib.ns2_rvq_ce(fr.data_ptr(), F, 128, cb.data_ptr(), cn2.data_ptr(), Q, K, own_codes.data_ptr(),
                         target_codes.data_ptr(), scratch.data_ptr(), loss.data_ptr(), _stream()), "ns2_rvq_ce")
    return loss


def rvq_ce_bwd(frames: torch.Tensor, codebooks: torch.Tensor, cn2: torch.Tensor, own_codes: torch.Tensor,
               target_codes: torch.Tensor, d_loss: torch.Tensor, row_scale: Optional[torch.Tensor] = None,
               rows_per_sample: int = 1, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """d loss / d frames of `rvq_ce` given d_loss (1-element f32 on the device): frames (F, 128) f32 -> (F, 128) f32.
    `row_scale` (optional, F / rows_per_sample f32) multiplies each sample's rows; `out` may be a (F, >= 128) f32 view
    with unit column stride (only its first 128 columns are written)."""
    lib = _lib.load()
    fr, cb, F, Q, K, specs = _rvq_ce_args(frames, codebooks, cn2, own_codes, target_codes)
    D = 128
    if out is None:
        out = torch.empty((F, D), device=fr.device, dtype=torch.float32)
    if d_loss.numel() != 1 or out.shape[-1] < D:
        raise ValueError(f"d_loss must hold one element and out >= {D} columns")
    if row_scale is not None and (rows_per_sample <= 0 or row_scale.numel() * rows_per_sample < F):
        raise ValueError("row_scale must hold one value per rows_per_sample rows")
    _check(*specs, ("d_loss", d_loss, F32, None, DENSE), ("row_scale", row_scale, F32, None, DENSE),
           ("out", out, F32, (F, None), LAST))
    coef = torch.empty(Q, device=fr.device, dtype=torch.float32)
    check(lib.ns2_rvq_ce_bwd(fr.data_ptr(), F, D, cb.data_ptr(), cn2.data_ptr(), Q, K, own_codes.data_ptr(),
                             target_codes.data_ptr(), d_loss.data_ptr(), _ptr(row_scale), int(rows_per_sample),
                             coef.data_ptr(), out.data_ptr(), out.stride(0), _stream()), "ns2_rvq_ce_bwd")
    return out


# --------------------------------------------------------------------------------------------------
# backward pass
# --------------------------------------------------------------------------------------------------
def attention_bwd(q, k, v, o, d_o, lse, dq_accum, dk, dv, *, heads: int, scale: Optional[float] = None,
                  delta: Optional[torch.Tensor] = None, dropout: Optional[DropoutSpec] = None,
                  kv_lens: Optional[torch.Tensor] = None):
    """(dq_accum f32 (B, Nq, inner) += dQ, dk, dv bf16) of softmax(q k^T scale) v given d_o; zero dq_accum for a plain dQ.
    dropout: the forward's (seed, site, p); the mask is regenerated, not stored.
    kv_lens: the forward's int32 CUDA (B,) key counts in [1, Nk] (see `attention`): dk / dv rows past them come out as
    exact zeros, and sample b's dk / dv are bit-identical to the call on its keys alone.  No dropout with kv_lens."""
    lib = _lib.load()
    if kv_lens is not None and dropout is not None:
        raise ValueError("attention_bwd: dropout with kv_lens is not supported")
    inner = heads * 64
    B, Nq, _ = q.shape
    _, Nk, _ = k.shape
    if delta is None:
        delta = torch.empty(B, heads, Nq, device=q.device, dtype=torch.float32)
    qs, ks = (B, Nq, inner), (B, Nk, inner)
    _check(("q", q, BF16, qs, LAST), ("k", k, BF16, ks, LAST), ("v", v, BF16, ks, LAST), ("o", o, BF16, qs, LAST),
           ("d_o", d_o, BF16, qs, LAST), ("lse", lse, F32, (B, heads, Nq), DENSE), ("dq_accum", dq_accum, F32, qs, DENSE),
           ("dk", dk, BF16, ks, LAST), ("dv", dv, BF16, ks, LAST), ("delta", delta, F32, (B, heads, Nq), DENSE),
           ("kv_lens", kv_lens, I32, (B,), DENSE))
    lens_ptr = _check_lens(kv_lens, 1, Nk, "kv_lens")
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
    a.kv_lens = lens_ptr
    check(lib.ns2_attn_bwd(C.byref(a), _stream()), "ns2_attn_bwd")
    return dq_accum, dk, dv


def rmsnorm_film_bwd(x, dh, dxr, dxr_bf, *, rows_per_batch: int, gamma=None, film=None, dfilm=None, dgamma=None):
    """dxr (f32, in place) += d/dx of rmsnorm_film(x) given dh (bf16); dxr_bf = bf16(dxr); dfilm / dgamma accumulate."""
    lib = _lib.load()
    D, n = x.shape[-1], x.numel()
    rows = n // D
    for name, t in (("dh", dh), ("dxr", dxr), ("dxr_bf", dxr_bf)):
        if t.numel() != n:
            raise ValueError(f"{name} must hold x's {n} elements, got {t.numel()}")
    for name, t in (("film", film), ("dfilm", dfilm)):   # row b holds [gamma_b | beta_b] of rows_per_batch rows
        if t is not None and (t.shape[0] * rows_per_batch < rows or t.shape[-1] < 2 * D):
            raise ValueError(f"{name} must have a row of >= {2 * D} columns per {rows_per_batch} rows of x, "
                             f"got {tuple(t.shape)}")
    _check(("x", x, F32, None, DENSE), ("dh", dh, BF16, None, DENSE), ("dxr", dxr, F32, None, DENSE),
           ("dxr_bf", dxr_bf, BF16, None, DENSE), ("gamma", gamma, F32, (D,), DENSE),
           ("film", film, F32, (None, None), LAST), ("dfilm", dfilm, F32, (None, None), LAST),
           ("dgamma", dgamma, F32, (D,), DENSE))
    film_bs = 0 if film is None else film.stride(0)
    dfilm_bs = 0 if dfilm is None else dfilm.stride(0)
    check(lib.ns2_rmsnorm_film_bwd(x.data_ptr(), dh.data_ptr(), rows, D, rows_per_batch, _ptr(gamma), _ptr(film), film_bs,
                                   _ptr(dfilm), dfilm_bs, _ptr(dgamma), dxr.data_ptr(), dxr_bf.data_ptr(), _stream()),
          "ns2_rmsnorm_film_bwd")
    return dxr


def geglu_bwd(pre, dg):
    """pre (rows, 2*Dp) bf16 packed [128 value | 128 gate] tiles -> overwritten by its gradient given dg (rows, Dp)."""
    lib = _lib.load()
    dp = dg.shape[-1]
    if pre.shape[-1] != 2 * dp or pre.numel() != 2 * dg.numel():
        raise ValueError(f"geglu_bwd: pre (.., {2 * dp}) must have dg's rows, got {tuple(pre.shape)}")
    _check(("pre", pre, BF16, None, DENSE), ("dg", dg, BF16, None, DENSE))
    check(lib.ns2_geglu_bwd(pre.data_ptr(), dg.data_ptr(), dg.numel() // dp, dp, _stream()), "ns2_geglu_bwd")
    return pre


def wavenet_gate_bwd(c, dy, dc, film, dfilm, *, dim: int, groups: int, film_group_stride: int):
    """c, dy, dc: (B, N, >= groups*dim) bf16 views (first groups*dim columns used); film/dfilm (B, ...) f32 views whose
    row b holds, for group g at g*film_group_stride, [gamma | beta]."""
    lib = _lib.load()
    B, N, _ = c.shape
    cols, film_cols = groups * dim, (groups - 1) * film_group_stride + 2 * dim
    for name, t, need in (("c", c, cols), ("dy", dy, cols), ("dc", dc, cols), ("film", film, film_cols),
                          ("dfilm", dfilm, film_cols)):
        if t.shape[-1] < need:
            raise ValueError(f"{name} must have >= {need} columns, got {tuple(t.shape)}")
    _check(("c", c, BF16, None, ROWS), ("dy", dy, BF16, (B, N, None), ROWS), ("dc", dc, BF16, (B, N, None), ROWS),
           ("film", film, F32, (B, None), LAST), ("dfilm", dfilm, F32, (B, None), LAST))
    check(lib.ns2_wavenet_gate_bwd(c.data_ptr(), c.stride(1), dy.data_ptr(), dy.stride(1), dc.data_ptr(), dc.stride(1), B,
                                   N, dim, groups, film.data_ptr(), film.stride(0), film_group_stride, dfilm.data_ptr(),
                                   dfilm.stride(0), _stream()), "ns2_wavenet_gate_bwd")
    return dc


def colsum(t, out):
    """out[c] (f32) += sum over all leading dims of t[..., c] (bf16; last dim contiguous, uniform row stride)."""
    lib = _lib.load()
    cols = t.shape[-1]
    rows = t.numel() // cols
    if out.numel() != cols:
        raise ValueError(f"out must hold {cols} elements, got {out.numel()}")
    _check(("t", t, BF16, None, ROWS), ("out", out, F32, None, DENSE))
    rs = t.stride(-2) if t.dim() >= 2 else cols
    check(lib.ns2_colsum_bf16(t.data_ptr(), rows, cols, rs, out.data_ptr(), _stream()), "ns2_colsum_bf16")
    return out


def group_sum(t, out, *, dim: int, groups: int):
    lib = _lib.load()
    if t.numel() != groups * out.numel():
        raise ValueError(f"t must hold groups * out's {groups * out.numel()} elements, got {t.numel()}")
    _check(("t", t, BF16, None, DENSE), ("out", out, BF16, None, DENSE))
    check(lib.ns2_group_sum_bf16(t.data_ptr(), out.numel() // dim, dim, groups, out.data_ptr(), _stream()),
          "ns2_group_sum_bf16")
    return out


def mse_bwd(pred, target, coef, out_bf=None, out_f32=None, lens=None):
    """coef[b] * (pred - target) as bf16 and/or f32: the seed of the backward pass.  lens: int32 CUDA (B,) in [1, N] for
    pred (B, N, ...): rows past lens[b] of sample b are written as exact zeros, the others are as without lens."""
    lib = _lib.load()
    B, n = pred.shape[0], pred.numel()
    if any(t is not None and t.numel() != n for t in (target, out_bf, out_f32)) or coef.numel() != B:
        raise ValueError(f"target, out_bf and out_f32 must hold pred's {n} elements and coef {B}")
    _check(("pred", pred, F32, None, DENSE, 16), ("target", target, F32, None, DENSE, 16), ("coef", coef, F32, None, DENSE),
           ("out_bf", out_bf, BF16, None, DENSE, 8), ("out_f32", out_f32, F32, None, DENSE, 16),
           ("lens", lens, I32, (B,), DENSE))
    rows, lp = _rows_lens(pred, lens)
    check(lib.ns2_mse_bwd(pred.data_ptr(), target.data_ptr(), coef.data_ptr(), B, n // B, _ptr(out_bf),
                          _ptr(out_f32), n // B // rows, lp, _stream()), "ns2_mse_bwd")
    return out_bf if out_bf is not None else out_f32


def film_wgrad(dfilm, t, dw, accumulate: bool = True):
    """dw (rows, cols) f32 (+)= dfilm (B, rows)^T @ t (B, cols).  accumulate=False overwrites dw (which then need not be
    initialised: one pass over the gradient buffer instead of zero-fill + read-modify-write).  `dfilm` may be a column
    window of a wider (B, total_rows) buffer (unit column stride)."""
    lib = _lib.load()
    B, rows = dfilm.shape
    cols = t.shape[-1]
    _check(("dfilm", dfilm, F32, None, LAST), ("t", t, F32, (B, cols), DENSE), ("dw", dw, F32, (rows, cols), DENSE))
    for b0 in range(0, B, 32):
        check(lib.ns2_film_wgrad(dfilm[b0:b0 + 32].data_ptr(), dfilm.stride(0), t[b0:b0 + 32].data_ptr(), min(32, B - b0),
                                 rows, cols, dw.data_ptr(), int(accumulate or b0 > 0), _stream()),
              "ns2_film_wgrad")
    return dw


def accum_bf16(acc, t, acc_bf=None):
    """acc (f32, contiguous) += t (bf16, contiguous, same numel); acc_bf (optional) = bf16(acc)."""
    lib = _lib.load()
    n = acc.numel()
    for name, o in (("t", t), ("acc_bf", acc_bf)):
        if o is not None and o.numel() != n:
            raise ValueError(f"{name} must hold acc's {n} elements, got {o.numel()}")
    _check(("acc", acc, F32, None, DENSE), ("t", t, BF16, None, DENSE), ("acc_bf", acc_bf, BF16, None, DENSE))
    check(lib.ns2_accum_bf16(acc.data_ptr(), t.data_ptr(), n, _ptr(acc_bf), _stream()), "ns2_accum_bf16")
    return acc


# --------------------------------------------------------------------------------------------------
# backward of the conditioning front end (encoders, pitch embedding, length regulation)
# --------------------------------------------------------------------------------------------------
def silu_bwd(pre: torch.Tensor, dout: torch.Tensor, dpre: Optional[torch.Tensor] = None) -> torch.Tensor:
    """d pre of out = silu(pre) given d out; pre, dout, dpre bf16 contiguous of one size.  dpre defaults to pre (in place)."""
    lib = _lib.load()
    dpre = pre if dpre is None else dpre
    n = pre.numel()
    if dout.numel() != n or dpre.numel() != n:
        raise ValueError(f"dout and dpre must hold pre's {n} elements")
    _check(("pre", pre, BF16, None, DENSE), ("dout", dout, BF16, None, DENSE), ("dpre", dpre, BF16, None, DENSE))
    check(lib.ns2_silu_bwd(pre.data_ptr(), dout.data_ptr(), n, dpre.data_ptr(), _stream()), "ns2_silu_bwd")
    return dpre


def embedding_bwd(ids: torch.Tensor, de: torch.Tensor, dtable: torch.Tensor, pad_id: int) -> torch.Tensor:
    """dtable[ids < 0 ? pad_id : ids] += de (f32, accumulated): the backward of `embedding_bf16`."""
    lib = _lib.load()
    rows, D = dtable.shape
    if de.numel() != ids.numel() * D:
        raise ValueError("de must hold one table row per id")
    _check(("ids", ids, I64, None, DENSE), ("de", de, F32, None, DENSE), ("dtable", dtable, F32, None, DENSE))
    check(lib.ns2_embedding_bwd(ids.data_ptr(), ids.numel(), de.data_ptr(), rows, D, int(pad_id),
                                dtable.data_ptr(), _stream()), "ns2_embedding_bwd")
    return dtable


def groupnorm_silu_bwd(x: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor, groups: int, dy: torch.Tensor,
                       dx: torch.Tensor, *, eps: float = 1e-5) -> Tuple[torch.Tensor, torch.Tensor]:
    """Backward of `groupnorm_silu` (without its residual): x, dy f32 (B, N, C) contiguous -> dx bf16 (B, N, C) written,
    returns (d weight, d bias) f32 (C,), reduced over the batch in a fixed order (bit-reproducible)."""
    lib = _lib.load()
    B, N, Cn = x.shape
    if weight.numel() != Cn or bias.numel() != Cn:
        raise ValueError(f"weight and bias must hold {Cn} elements")
    _check(("x", x, F32, None, DENSE), ("dy", dy, F32, (B, N, Cn), DENSE), ("dx", dx, BF16, (B, N, Cn), DENSE),
           ("weight", weight, F32, None, DENSE, 16), ("bias", bias, F32, None, DENSE, 16))
    partial = torch.empty(2 * B * Cn, device=x.device)
    dw, db = torch.empty(Cn, device=x.device), torch.empty(Cn, device=x.device)
    check(lib.ns2_groupnorm_silu_bwd(x.data_ptr(), B, N, Cn, int(groups), weight.data_ptr(), bias.data_ptr(), float(eps),
                                     dy.data_ptr(), dx.data_ptr(), partial.data_ptr(), dw.data_ptr(), db.data_ptr(),
                                     _stream()), "ns2_groupnorm_silu_bwd")
    return dw, db


def rowdot_bwd(x: torch.Tensor, w: torch.Tensor, pred: torch.Tensor, dpred: torch.Tensor,
               dx: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """Backward of `rowdot(..., relu=True)` from its output `pred`: dx (f32, x's shape) += d pre * w in place, returns
    (d w (dim,), d bias (1,)) f32, reduced in a fixed order.  d pre = d pred where pred > 0, else 0."""
    lib = _lib.load()
    dim, rows = x.shape[-1], pred.numel()
    if rows * dim != x.numel() or dpred.numel() != rows or w.numel() != dim:
        raise ValueError("rowdot_bwd needs x (..., dim), w (dim,), pred / dpred one value per row, dx of x's shape")
    _check(("x", x, F32, None, DENSE), ("w", w, F32, None, DENSE), ("pred", pred, F32, None, DENSE),
           ("dpred", dpred, F32, None, DENSE), ("dx", dx, F32, tuple(x.shape), DENSE))
    chunks = (rows + _lib.NS2_ROWDOT_BWD_ROWS - 1) // _lib.NS2_ROWDOT_BWD_ROWS
    partial = torch.empty(max(chunks, 1) * (dim + 4), device=x.device)
    dw, db = torch.empty(dim, device=x.device), torch.empty(1, device=x.device)
    check(lib.ns2_rowdot_bwd(x.data_ptr(), rows, dim, w.data_ptr(), pred.data_ptr(), dpred.data_ptr(), dx.data_ptr(),
                             partial.data_ptr(), dw.data_ptr(), db.data_ptr(), _stream()), "ns2_rowdot_bwd")
    return dw, db


def expand_encodings_bwd(dcond: torch.Tensor, coarse: torch.Tensor, idx: torch.Tensor, dphon: Optional[torch.Tensor],
                         dtable: Optional[torch.Tensor]):
    """Backward of `expand_encodings` given d cond TOKEN-MAJOR (B, L, D) f32 (unit channel stride, uniform row stride):
    dphon (B, T, D) += per-phoneme sums over its frames; dtable[coarse] += the same sums.  Both accumulate."""
    lib = _lib.load()
    B, L, D = dcond.shape
    T = coarse.shape[-1]
    _check(("dcond", dcond, F32, None, ROWS), ("coarse", coarse, I32, (B, T), DENSE), ("idx", idx, I32, (B, L), DENSE),
           ("dphon", dphon, F32, (B, T, D), DENSE), ("dtable", dtable, F32, (None, D), DENSE))
    rows = 1 if dtable is None else dtable.shape[0]
    check(lib.ns2_expand_encodings_bwd(dcond.data_ptr(), max(dcond.stride(1), D), coarse.data_ptr(), rows, idx.data_ptr(),
                                       B, T, D, L, _ptr(dphon), _ptr(dtable), _stream()), "ns2_expand_encodings_bwd")
    return dphon, dtable


def add_rows_bcast(x: torch.Tensor, v: torch.Tensor, scale: float = 1.0) -> torch.Tensor:
    """x[b, r, :] += scale * v[b, :] in place; x (B, R, D) f32 contiguous, v (B, D) f32 contiguous."""
    lib = _lib.load()
    B, R, D = x.shape
    _check(("x", x, F32, None, DENSE), ("v", v, F32, (B, D), DENSE))
    check(lib.ns2_add_rows_bcast(x.data_ptr(), B, R, D, v.data_ptr(), float(scale), _stream()), "ns2_add_rows_bcast")
    return x


# --------------------------------------------------------------------------------------------------
# Monotonic alignment search (aligner.py:88-122)
# --------------------------------------------------------------------------------------------------
def maximum_path(value: torch.Tensor, mask: torch.Tensor, neg_const: float = float("-inf"), *,
                 want_path: bool = True) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    """(idx (b, t_y) int32, path (b, t_x, t_y) f32 or None) for value/mask (b, t_x, t_y) f32 contiguous."""
    lib = _lib.load()
    _check(("value", value, F32, (None, None, None), DENSE), ("mask", mask, F32, tuple(value.shape), DENSE))
    b, t_x, t_y = value.shape
    idx = torch.empty((b, t_y), dtype=torch.int32, device=value.device)
    path = torch.empty_like(value) if want_path else None
    ws_bytes = int(lib.ns2_maximum_path_workspace_bytes(b, t_x, t_y))
    ws = torch.empty(max(ws_bytes, 16), dtype=torch.uint8, device=value.device)
    check(lib.ns2_maximum_path(value.data_ptr(), mask.data_ptr(), b, t_x, t_y, float(neg_const), ws.data_ptr(),
                               ws_bytes, idx.data_ptr(), _ptr(path), _stream()), "ns2_maximum_path")
    return idx, path


# --------------------------------------------------------------------------------------------------
# SEANet decoder and encoder (Encodec 24 kHz): LSTM recurrence, conv operand preparation, 32-channel tail and head
# --------------------------------------------------------------------------------------------------
def _row_strides(t: Optional[torch.Tensor]) -> Tuple[int, int]:
    """(row stride, batch stride) of a (B, T, C) view; (0, 0) for None."""
    return (0, 0) if t is None else (t.stride(1), t.stride(0))


def lstm_seq(xproj: torch.Tensor, w_hh: torch.Tensor, *, skip: Optional[torch.Tensor] = None,
             out: Optional[torch.Tensor] = None, out_bf16: Optional[torch.Tensor] = None) -> None:
    """One nn.LSTM(512, 512) layer over the sequence: xproj (B, T, 2048) f32 holds x W_ih^T + b_ih + b_hh in the
    kernel's gate order (see include/ns2_b200.h section 10), w_hh (2048, 512) bf16 in the same row order.
    Writes h_t (+ skip) into out (B, T, 512) f32 and/or out_bf16 (B, T, 512) bf16; all may be strided views."""
    lib = _lib.load()
    if out is None and out_bf16 is None:
        raise ValueError("lstm_seq needs out and/or out_bf16")
    B, T, _ = xproj.shape
    for name, t, cols in (("xproj", xproj, 2048), ("skip", skip, 512), ("out", out, 512), ("out_bf16", out_bf16, 512)):
        if t is not None and t.shape[-1] < cols:
            raise ValueError(f"{name} must have >= {cols} channels, got {tuple(t.shape)}")
    _check(("xproj", xproj, F32, None, LAST), ("w_hh", w_hh, BF16, (2048, 512), DENSE),
           ("skip", skip, F32, (B, T, None), LAST), ("out", out, F32, (B, T, None), LAST),
           ("out_bf16", out_bf16, BF16, (B, T, None), LAST))
    check(lib.ns2_lstm_seq(xproj.data_ptr(), *_row_strides(xproj), w_hh.data_ptr(), B, T, 512, _ptr(skip),
                           *_row_strides(skip), _ptr(out), *_row_strides(out), _ptr(out_bf16), *_row_strides(out_bf16),
                           _stream()), "ns2_lstm_seq")


def elu_pad(x: torch.Tensor, out: torch.Tensor, *, pad: int, elu: bool = True, raw: bool = False) -> torch.Tensor:
    """out[:, r, :C] = bf16(ELU(xpad[:, r - pad])) for r < pad + T (ELU only with elu=True), xpad = x reflect-padded
    on the left (Encodec's causal padding); raw=True also writes bf16(xpad) in columns [C, 2C).  x (B, T, C) f32 and
    out (B, pad + T, >= C or 2C) bf16 may be row-strided views (e.g. a GEMM output past its scratch rows)."""
    lib = _lib.load()
    B, T, Cc = x.shape
    out_cols = Cc * (2 if raw else 1)
    if out.shape[-1] < out_cols:
        raise ValueError(f"out must have >= {out_cols} channels, got {tuple(out.shape)}")
    _check(("x", x, F32, None, LAST), ("out", out, BF16, (B, pad + T, None), LAST))
    flags = (_lib.NS2_ELU_PAD_ELU if elu else 0) | (_lib.NS2_ELU_PAD_RAW if raw else 0)
    check(lib.ns2_elu_pad(x.data_ptr(), *_row_strides(x), B, T, Cc, int(pad), flags, out.data_ptr(), *_row_strides(out),
                          _stream()), "ns2_elu_pad")
    return out


def seanet_tail(x: torch.Tensor, params: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """out (B, T) f32 = conv7(ELU(ResnetBlock(x))) for x (B, T, 32) f32 (row-strided view allowed); params: the
    NS2_SEANET_TAIL_PARAMS packed f32 weights (SEANetDecoder packs them)."""
    lib = _lib.load()
    B, T, _ = x.shape
    if params.numel() != _lib.NS2_SEANET_TAIL_PARAMS:
        raise ValueError(f"params must hold {_lib.NS2_SEANET_TAIL_PARAMS} elements, got {params.numel()}")
    _check(("x", x, F32, (B, T, 32), LAST), ("params", params, F32, None, DENSE, 16), ("out", out, F32, (B, T), LAST))
    check(lib.ns2_seanet_tail(x.data_ptr(), *_row_strides(x), B, T, params.data_ptr(), out.data_ptr(), out.stride(0),
                              _stream()), "ns2_seanet_tail")
    return out


def seanet_head(x: torch.Tensor, params: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """out (B, T + 2, 32) bf16 = elu_pad(ResnetBlock(conv7(x)), pad=2) for audio x (B, T) f32 (unit time stride,
    any batch stride): the encoder's full-rate stage, ready as the first strided conv's A operand.  params: the
    NS2_SEANET_HEAD_PARAMS packed f32 weights (SEANetEncoder packs them).  out may be a row-strided view."""
    lib = _lib.load()
    B, T = x.shape
    if params.numel() != _lib.NS2_SEANET_HEAD_PARAMS:
        raise ValueError(f"params must hold {_lib.NS2_SEANET_HEAD_PARAMS} elements, got {params.numel()}")
    _check(("x", x, F32, None, LAST), ("params", params, F32, None, DENSE, 16), ("out", out, BF16, (B, T + 2, 32), LAST))
    check(lib.ns2_seanet_head(x.data_ptr(), x.stride(0), B, T, params.data_ptr(), out.data_ptr(), *_row_strides(out),
                              _stream()), "ns2_seanet_head")
    return out
