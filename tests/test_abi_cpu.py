"""CPU: the C-ABI library builds, loads without a GPU driver, and exports every symbol include/ns2_b200.h declares."""
import ctypes
import re
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent


@pytest.fixture(scope="module")
def lib():
    from naturalspeech2_pytorch_b200 import _lib, build
    build.build()
    return _lib.load()


def test_header_symbols_are_exported(lib):
    header = (ROOT / "include" / "ns2_b200.h").read_text()
    declared = set(re.findall(r"\b(ns2_[a-z0-9_]+)\s*\(", header))
    assert len(declared) >= 18, declared
    from naturalspeech2_pytorch_b200 import _lib
    assert declared == set(_lib.SIGNATURES), declared ^ set(_lib.SIGNATURES)
    raw = ctypes.CDLL(str(_lib.lib_path()))
    for name in declared:
        assert hasattr(raw, name), f"{name} is declared in the header but not exported"


def test_abi_version_and_error_string(lib):
    from naturalspeech2_pytorch_b200 import _lib
    assert lib.ns2_abi_version() == _lib.NS2_ABI_VERSION
    assert isinstance(lib.ns2_last_error(), (bytes, type(None)))
    assert lib.ns2_launch_count() >= 0


def test_argument_validation_without_gpu(lib):
    """Host-side validation runs before any CUDA call, so bad arguments are reported even on a CPU box."""
    from naturalspeech2_pytorch_b200._lib import GemmArgs, AttnArgs
    a = GemmArgs()
    assert lib.ns2_gemm(ctypes.byref(a), None) < 0
    assert b"non-NULL" in lib.ns2_last_error()
    # an otherwise valid call (dummy pointers, never dereferenced) with a flag bit the library does not define
    a.A, a.B, a.out = 256, 512, 1024
    a.a_batches, a.a_rows, a.a_cols, a.a_row_stride, a.a_batch_stride = 1, 128, 64, 64, 128 * 64
    a.b_rows, a.b_cols, a.b_row_stride = 128, 64, 64
    a.n, a.groups, a.num_segs, a.out_row_stride = 128, 1, 1, 128
    a.segs[0].k_len = 64
    before = lib.ns2_launch_count()
    for flags in (2, 8):
        a.flags = flags
        assert lib.ns2_gemm(ctypes.byref(a), None) < 0
        assert f"unknown flags 0x{flags:x}".encode() in lib.ns2_last_error()
    assert lib.ns2_launch_count() == before
    t = AttnArgs()
    assert lib.ns2_attn_fwd(ctypes.byref(t), None) < 0
    assert lib.ns2_rvq_encode(None, 0, 128, None, None, None, None, 8, 1024, None, None, None) < 0
    # round-2 entry points (aligner / conditioning encoders): size checks come before any CUDA call too
    assert lib.ns2_maximum_path_workspace_bytes(32, 100, 1024) == 32 * 1024 * 128
    assert lib.ns2_maximum_path(1, 1, 2, 2000, 16, float("-inf"), 1, 1 << 20, 1, None, None) < 0
    assert b"1024" in lib.ns2_last_error()
    assert lib.ns2_maximum_path(None, None, 0, 10, 10, float("-inf"), None, 0, None, None, None) == 0   # empty batch
    assert lib.ns2_groupnorm_silu(None, 2, 8, 100, 8, None, None, 1e-5, None, None, None, None, None) < 0  # 100 % 8 != 0
    assert lib.ns2_rowdot(None, 4, 10, None, None, 0, None, None) < 0                                     # dim % 4 != 0
    assert lib.ns2_embedding_bf16(None, 4, None, 10, 128, 10, None, None) < 0                             # pad_id outside
    assert lib.ns2_film_wgrad(None, 8, None, 33, 8, 8, None, 0, None) < 0


@pytest.mark.parametrize("k", [
    4096,   # above MAX_K = 2048, the 11-bit code index of the encoder's packed keys
    192,    # not a multiple of the 128-code chunk
])
def test_rvq_rejects_unsupported_codebook_size_before_launch(lib, k):
    """The codebook-size checks are host-side: a clean error and no kernel launch (dummy non-NULL device pointers are
    never dereferenced)."""
    before = lib.ns2_launch_count()
    assert lib.ns2_rvq_encode(16, 4, 128, 16, 16, 16, 16, 1, k, 16, None, None) < 0
    assert b"codebook size" in lib.ns2_last_error()
    if k % 128:
        assert lib.ns2_rvq_prepare(16, 1, k, 128, 16, 16, 16, None) < 0
        assert b"codebook size" in lib.ns2_last_error()
    assert lib.ns2_launch_count() == before


def test_struct_layout_matches_header():
    """ctypes mirrors of the C structs: sizes, and the offsets of the optional pointer fields, are what a C compiler
    produces for include/ns2_b200.h (equal sizes alone would not catch two pointers swapped)."""
    import subprocess, tempfile, textwrap
    from naturalspeech2_pytorch_b200._lib import GemmArgs, AttnArgs, AttnBwdArgs, GemmSeg
    src = textwrap.dedent('''
        #include <stddef.h>
        #include <stdio.h>
        #include "ns2_b200.h"
        int main(void) {
          printf("%zu %zu %zu %zu\\n", sizeof(ns2_gemm_seg), sizeof(ns2_gemm_args), sizeof(ns2_attn_args),
                 sizeof(ns2_attn_bwd_args));
          printf("%zu %zu %zu %zu %zu %zu\\n", offsetof(ns2_gemm_args, row_lens), offsetof(ns2_attn_args, kv_lens),
                 offsetof(ns2_attn_args, dropout), offsetof(ns2_attn_args, q_lens),
                 offsetof(ns2_attn_bwd_args, dropout), offsetof(ns2_attn_bwd_args, kv_lens));
          return 0;
        }
    ''')
    with tempfile.TemporaryDirectory() as d:
        c = Path(d) / "t.c"
        c.write_text(src)
        exe = Path(d) / "t"
        subprocess.run(["gcc", "-I", str(ROOT / "include"), str(c), "-o", str(exe)], check=True)
        out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    assert [int(v) for v in out] == [ctypes.sizeof(GemmSeg), ctypes.sizeof(GemmArgs), ctypes.sizeof(AttnArgs),
                                     ctypes.sizeof(AttnBwdArgs),
                                     GemmArgs.row_lens.offset, AttnArgs.kv_lens.offset, AttnArgs.dropout.offset,
                                     AttnArgs.q_lens.offset, AttnBwdArgs.dropout.offset, AttnBwdArgs.kv_lens.offset]


def test_ops_reject_cpu_tensors():
    import torch
    from naturalspeech2_pytorch_b200 import ops
    with pytest.raises(ValueError):
        ops.cast_bf16(torch.zeros(8), torch.zeros(8, dtype=torch.bfloat16))


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    from naturalspeech2_pytorch_b200 import _lib
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "_LIB_PATH", tmp_path / "nope.so")
    with pytest.raises(_lib.Ns2Error):
        _lib.load()
