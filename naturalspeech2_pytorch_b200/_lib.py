"""ctypes binding of libns2b200.so (declarations mirror include/ns2_b200.h one to one).

The library is the product: if it is missing or fails to load, importing the ops raises — there is no
PyTorch/CPU fallback for any op on the hot path.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

_LIB_PATH = Path(__file__).resolve().parent / "lib" / "libns2b200.so"

NS2_EPI_BF16, NS2_EPI_F32, NS2_EPI_GEGLU, NS2_EPI_WAVENET = 0, 1, 2, 3
NS2_GEMM_MAX_SEGS = 12
NS2_GEMM_MAX_GROUPS = 8
NS2_MSE_SCRATCH_PER_SAMPLE = 64
NS2_RVQ_STATS_LEN = 4
NS2_OBJ_V, NS2_OBJ_EPS, NS2_OBJ_X0 = 0, 1, 2
NS2_GEMM_FLAG_SKIP_EPILOGUE, NS2_GEMM_FLAG_SILU = 1, 4
NS2_ELU_PAD_ELU, NS2_ELU_PAD_RAW = 1, 2
NS2_SEANET_TAIL_PARAMS = 3348
NS2_SEANET_HEAD_PARAMS = 3376
NS2_ROWDOT_BWD_ROWS = 32
NS2_GEMM_ROW_LENS_MAX_BATCHES = 64
NS2_ABI_VERSION = 9


class GemmSeg(C.Structure):
    _fields_ = [("a_col_off", C.c_int32), ("b_col_off", C.c_int32), ("k_len", C.c_int32),
                ("shift_units", C.c_int32), ("acc", C.c_int32)]


class GemmArgs(C.Structure):
    _fields_ = [
        ("A", C.c_void_p), ("a_row_stride", C.c_int64), ("a_batch_stride", C.c_int64),
        ("a_batches", C.c_int32), ("a_rows", C.c_int32), ("a_cols", C.c_int32),
        ("B", C.c_void_p), ("b_row_stride", C.c_int64), ("b_rows", C.c_int32), ("b_cols", C.c_int32),
        ("n", C.c_int32), ("groups", C.c_int32), ("a_group_col_stride", C.c_int32),
        ("b_group_row_stride", C.c_int32), ("out_group_col_stride", C.c_int32),
        ("dil", C.c_int32 * NS2_GEMM_MAX_GROUPS),
        ("num_segs", C.c_int32), ("segs", GemmSeg * NS2_GEMM_MAX_SEGS),
        ("epilogue", C.c_int32), ("bias", C.c_void_p), ("bias1_off", C.c_int32),
        ("out", C.c_void_p), ("out_row_stride", C.c_int64),
        ("resid", C.c_void_p), ("resid_row_stride", C.c_int64),
        ("film", C.c_void_p), ("film_batch_stride", C.c_int64), ("film_group_stride", C.c_int32),
        ("flags", C.c_int32), ("row_lens", C.c_void_p),
    ]


class WgradArgs(C.Structure):
    _fields_ = [
        ("dY", C.c_void_p), ("dy_row_stride", C.c_int64), ("dy_batch_stride", C.c_int64), ("dy_cols", C.c_int32),
        ("X", C.c_void_p), ("x_row_stride", C.c_int64), ("x_batch_stride", C.c_int64), ("x_cols", C.c_int32),
        ("batches", C.c_int32), ("rows", C.c_int32), ("n", C.c_int32), ("k", C.c_int32),
        ("groups", C.c_int32), ("dy_group_col_stride", C.c_int32), ("x_group_col_stride", C.c_int32),
        ("x_col_off", C.c_int32), ("dil", C.c_int32 * NS2_GEMM_MAX_GROUPS), ("shift_units", C.c_int32),
        ("dW", C.c_void_p), ("dw_row_stride", C.c_int64), ("dw_group_row_stride", C.c_int32), ("splits", C.c_int32),
    ]


class Dropout(C.Structure):
    _fields_ = [("seed", C.c_uint64), ("site", C.c_uint32), ("p", C.c_float)]


class AttnArgs(C.Structure):
    _fields_ = [
        ("q", C.c_void_p), ("q_row_stride", C.c_int64), ("q_batch_stride", C.c_int64),
        ("k", C.c_void_p), ("k_row_stride", C.c_int64), ("k_batch_stride", C.c_int64),
        ("v", C.c_void_p), ("v_row_stride", C.c_int64), ("v_batch_stride", C.c_int64),
        ("out", C.c_void_p), ("o_row_stride", C.c_int64), ("o_batch_stride", C.c_int64),
        ("batches", C.c_int32), ("heads", C.c_int32), ("q_len", C.c_int32), ("kv_len", C.c_int32),
        ("dim_head", C.c_int32), ("scale", C.c_float), ("lse", C.c_void_p),
        ("kv_lens", C.c_void_p), ("dropout", C.POINTER(Dropout)), ("q_lens", C.c_void_p),
    ]


class AttnBwdArgs(C.Structure):
    _fields_ = [
        ("q", C.c_void_p), ("q_row_stride", C.c_int64), ("q_batch_stride", C.c_int64),
        ("k", C.c_void_p), ("k_row_stride", C.c_int64), ("k_batch_stride", C.c_int64),
        ("v", C.c_void_p), ("v_row_stride", C.c_int64), ("v_batch_stride", C.c_int64),
        ("o", C.c_void_p), ("o_row_stride", C.c_int64), ("o_batch_stride", C.c_int64),
        ("d_o", C.c_void_p), ("do_row_stride", C.c_int64), ("do_batch_stride", C.c_int64),
        ("lse", C.c_void_p), ("delta", C.c_void_p), ("dq_accum", C.c_void_p),
        ("dk", C.c_void_p), ("dk_row_stride", C.c_int64), ("dk_batch_stride", C.c_int64),
        ("dv", C.c_void_p), ("dv_row_stride", C.c_int64), ("dv_batch_stride", C.c_int64),
        ("batches", C.c_int32), ("heads", C.c_int32), ("q_len", C.c_int32), ("kv_len", C.c_int32),
        ("dim_head", C.c_int32), ("scale", C.c_float), ("dropout", C.POINTER(Dropout)), ("kv_lens", C.c_void_p),
    ]


_P, _I32, _I64, _F = C.c_void_p, C.c_int32, C.c_int64, C.c_float

# name -> (restype, argtypes); every symbol include/ns2_b200.h declares
SIGNATURES = {
    "ns2_last_error": (C.c_char_p, []),
    "ns2_abi_version": (C.c_int, []),
    "ns2_set_sm_limit": (C.c_int, [C.c_int]),
    "ns2_launch_count": (C.c_int64, []),
    "ns2_gemm": (C.c_int, [C.POINTER(GemmArgs), _P]),
    "ns2_wgrad": (C.c_int, [C.POINTER(WgradArgs), _P]),
    "ns2_fold_conv_linear": (C.c_int, [_P, _P, _P, _P, _I32, _I32, _I32, _I32, _I32, _I32, _P, _P, _P]),
    "ns2_attn_fwd": (C.c_int, [C.POINTER(AttnArgs), _P]),
    "ns2_attn_bwd": (C.c_int, [C.POINTER(AttnBwdArgs), _P]),
    "ns2_dropout_f32": (C.c_int, [_P, _I64, C.POINTER(Dropout), _P]),
    "ns2_rmsnorm_film": (C.c_int, [_P, _I64, _I64, _I32, _I32, _P, _P, _I64, _P, _I64, _P, _P]),
    "ns2_rmsnorm_f32": (C.c_int, [_P, _I64, _I64, _I32, _P, _P, _I64, _P]),
    "ns2_time_cond": (C.c_int, [_P, _I32, _P, _I32, _P, _P, _I32, _P, _I64, _P]),
    "ns2_small_linear": (C.c_int, [_P, _I64, _I32, _I32, _P, _P, _I32, _I32, _P, _I64, _P]),
    "ns2_cast_bf16": (C.c_int, [_P, _P, _I64, _P, _P]),
    "ns2_mean_rows": (C.c_int, [_P, _I32, _I32, _I32, _P, _P, _P]),
    "ns2_mask_rows": (C.c_int, [_P, _I32, _I64, _I64, _I32, _I32, _I32, _P, _P]),
    "ns2_pack_rows": (C.c_int, [_P, _I64, _I64, _I32, _P, _P, _I64, _I64, _I32, _P, _I32, _I32, _P, _I64, _I64, _I32,
                                _P]),
    "ns2_transpose_cast": (C.c_int, [_P, _I32, _I32, _I32, _P, _P]),
    "ns2_groupnorm_silu": (C.c_int, [_P, _I32, _I32, _I32, _I32, _P, _P, _F, _P, _P, _P, _P, _P]),
    "ns2_rowdot": (C.c_int, [_P, _I64, _I32, _P, _P, _I32, _P, _P]),
    "ns2_expand_encodings": (C.c_int, [_P, _P, _P, _I32, _P, _I32, _I32, _I32, _I32, _P, _P]),
    "ns2_embedding_bf16": (C.c_int, [_P, _I64, _P, _I32, _I32, _I32, _P, _P]),
    "ns2_cond_inject": (C.c_int, [_P, _P, _P, _P, _I32, _I32, _I32, _I32, _P, _P, _P]),
    "ns2_select_rows": (C.c_int, [_P, _P, _P, _I64, _I32, _I32, _P, _I64, _I32, _P]),
    "ns2_q_sample": (C.c_int, [_P, _P, _P, _P, _I32, _I64, _P, _P, _I32, _P]),
    "ns2_mse_rows": (C.c_int, [_P, _P, _I32, _I64, _P, _P, _P, _I64, _P, _P]),
    "ns2_ddim_step": (C.c_int, [_P, _P, _P, _P, _P, _P, _I32, _I64, _I32, _P]),
    "ns2_cfg_combine": (C.c_int, [_P, _P, _F, _I64, _P, _P]),
    "ns2_x_start": (C.c_int, [_P, _P, _P, _P, _I32, _I64, _P, _I32, _P]),
    "ns2_rmsnorm_film_bwd": (C.c_int, [_P, _P, _I64, _I32, _I32, _P, _P, _I64, _P, _I64, _P, _P, _P, _P]),
    "ns2_geglu_bwd": (C.c_int, [_P, _P, _I64, _I32, _P]),
    "ns2_wavenet_gate_bwd": (C.c_int, [_P, _I64, _P, _I64, _P, _I64, _I32, _I32, _I32, _I32, _P, _I64, _I32, _P, _I64, _P]),
    "ns2_colsum_bf16": (C.c_int, [_P, _I64, _I32, _I64, _P, _P]),
    "ns2_group_sum_bf16": (C.c_int, [_P, _I64, _I32, _I32, _P, _P]),
    "ns2_mse_bwd": (C.c_int, [_P, _P, _P, _I32, _I64, _P, _P, _I64, _P, _P]),
    "ns2_film_wgrad": (C.c_int, [_P, _I64, _P, _I32, _I64, _I32, _P, _I32, _P]),
    "ns2_accum_bf16": (C.c_int, [_P, _P, _I64, _P, _P]),
    "ns2_silu_bwd": (C.c_int, [_P, _P, _I64, _P, _P]),
    "ns2_embedding_bwd": (C.c_int, [_P, _I64, _P, _I32, _I32, _I32, _P, _P]),
    "ns2_expand_encodings_bwd": (C.c_int, [_P, _I64, _P, _I32, _P, _I32, _I32, _I32, _I32, _P, _P, _P]),
    "ns2_add_rows_bcast": (C.c_int, [_P, _I32, _I32, _I32, _P, _F, _P]),
    "ns2_groupnorm_silu_bwd": (C.c_int, [_P, _I32, _I32, _I32, _I32, _P, _P, _F, _P, _P, _P, _P, _P, _P]),
    "ns2_rowdot_bwd": (C.c_int, [_P, _I64, _I32, _P, _P, _P, _P, _P, _P, _P, _P]),
    "ns2_rvq_prepare": (C.c_int, [_P, _I32, _I32, _I32, _P, _P, _P, _P]),
    "ns2_rvq_encode": (C.c_int, [_P, _I64, _I32, _P, _P, _P, _P, _I32, _I32, _P, _P, _P]),
    "ns2_rvq_decode": (C.c_int, [_P, _I64, _I32, _I32, _I32, _P, _P, _P]),
    "ns2_maximum_path_workspace_bytes": (C.c_int64, [_I32, _I32, _I32]),
    "ns2_maximum_path": (C.c_int, [_P, _P, _I32, _I32, _I32, _F, _P, _I64, _P, _P, _P]),
    "ns2_rvq_ce": (C.c_int, [_P, _I64, _I32, _P, _P, _I32, _I32, _P, _P, _P, _P, _P]),
    "ns2_rvq_ce_bwd": (C.c_int, [_P, _I64, _I32, _P, _P, _I32, _I32, _P, _P, _P, _P, _I64, _P, _P, _I64, _P]),
    "ns2_lstm_seq": (C.c_int, [_P, _I64, _I64, _P, _I32, _I32, _I32, _P, _I64, _I64, _P, _I64, _I64, _P, _I64, _I64,
                               _P]),
    "ns2_elu_pad": (C.c_int, [_P, _I64, _I64, _I32, _I32, _I32, _I32, _I32, _P, _I64, _I64, _P]),
    "ns2_seanet_tail": (C.c_int, [_P, _I64, _I64, _I32, _I32, _P, _P, _I64, _P]),
    "ns2_seanet_head": (C.c_int, [_P, _I64, _I32, _I32, _P, _P, _I64, _I64, _P]),
}

_lib = None


class Ns2Error(RuntimeError):
    pass


def lib_path() -> Path:
    return _LIB_PATH


def load() -> C.CDLL:
    """Load the shared library (once) and attach the prototypes.  Raises if it is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not _LIB_PATH.exists():
        raise Ns2Error(
            f"{_LIB_PATH} not found: the CUDA extension is not built. Run "
            "`python -c 'import __graft_entry__ as g; g.build()'` (needs nvcc). There is no fallback path.")
    lib = C.CDLL(str(_LIB_PATH))
    for name, (res, args) in SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError:
            raise Ns2Error(f"ABI mismatch: {_LIB_PATH} does not export {name} (a library built from older sources); "
                           "rebuild it with `python -m naturalspeech2_pytorch_b200.build --force`") from None
        fn.restype = res
        fn.argtypes = args
    if lib.ns2_abi_version() != NS2_ABI_VERSION:
        raise Ns2Error(f"ABI mismatch: library {lib.ns2_abi_version()} vs binding {NS2_ABI_VERSION}")
    _lib = lib
    return lib


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = load().ns2_last_error()
        raise Ns2Error(f"{what} failed (code {rc}): {msg.decode() if msg else '?'}")
