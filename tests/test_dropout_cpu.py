"""CPU: the dropout random numbers (tests/dropout_oracle.py restates csrc/philox.cuh), the keep rule, the C ABI of the
dropout entry points, the encoders' dropout plumbing, and what ptxas makes of the dropout attention backward."""
import ctypes
import re
import subprocess
import tempfile
import textwrap
from pathlib import Path

import numpy as np
import pytest

import dropout_oracle as do

ROOT = Path(__file__).resolve().parent.parent


@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), "6627e8d5 e169c58d bc57ac4c 9b00dbd8"),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, "408f276d 41c83b0e a20bc7c6 6d5451fd"),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0), "d16cfe09 94fdcceb 5001e420 24126ea1"),
])
def test_philox_known_answers(ctr, key, want):
    """The Random123 known-answer vectors of Philox4x32-10."""
    got = " ".join(f"{int(w):08x}" for w in do.philox4x32_10(*ctr, *key))
    assert got == want


def test_keep_rule():
    assert do.keep_threshold(0.0) == 0 and do.keep_scale(0.0) == np.float32(1.0)
    assert do.attention_mask(2 ** 40 + 3, 1, 0.0, 2, 3, 70, 40).all()
    assert do.elementwise_mask(2 ** 40 + 3, 0, 0.0, 1001).all()
    assert do.keep_threshold(0.5) == 2 ** 31
    assert do.keep_threshold(np.nextafter(np.float32(1), np.float32(0))) == 2 ** 32 - 2 ** 8
    assert do.keep_scale(0.2) == np.float32(1 / (1 - float(np.float32(0.2))))
    for bad in (-0.1, 1.0, 1.5, float("nan")):
        with pytest.raises(ValueError):
            do.keep_threshold(bad)


def test_attention_mask_layout():
    """Element (b, h, q, k) is word 2 q[3] + k[3] of the block (idx(k & ~8), idx(q & ~8), b heads + h, site)."""
    seed, site, p, B, H, Nq, Nk = 0x1234_5678_9ABC_DEF1, 7, 0.5, 2, 3, 45, 37
    m = do.attention_mask(seed, site, p, B, H, Nq, Nk)
    t = do.keep_threshold(p)
    for b, h, q, k in [(0, 0, 0, 0), (1, 2, 9, 8), (1, 1, 44, 36), (0, 2, 25, 17)]:
        idx = lambda x: ((x & ~8) >> 4) * 8 + ((x & ~8) & 7)   # noqa: E731
        w = do.philox4x32_10(idx(k), idx(q), b * H + h, site, seed & 0xFFFFFFFF, seed >> 32)
        assert m[b, h, q, k] == (int(w[2 * ((q >> 3) & 1) + ((k >> 3) & 1)]) >= t)
    e = do.elementwise_mask(seed, site, p, 11)
    w = do.philox4x32_10(2, 0, 0xFFFFFFFF, site, seed & 0xFFFFFFFF, seed >> 32)
    assert list(e[8:11]) == [int(v) >= t for v in w[:3]]


def test_ops_reject_bad_p():
    """ops validates p before anything reaches the library (no tensor is touched)."""
    from naturalspeech2_pytorch_b200 import ops
    for bad in (-0.1, 1.0, 2.0, float("nan")):
        with pytest.raises(ValueError):
            ops._dropout_args((1, 0, bad))
    assert ops._dropout_args(None) is None and ops._dropout_args((5, 1, 0.0)) is None
    d = ops._dropout_args((2 ** 63 + 5, 3, 0.25))
    assert (d.seed, d.site, d.p) == (2 ** 63 + 5, 3, 0.25)


@pytest.fixture(scope="module")
def lib():
    from naturalspeech2_pytorch_b200 import _lib, build
    build.build()
    return _lib.load()


def test_entry_points_reject_bad_p_before_launch(lib):
    from naturalspeech2_pytorch_b200._lib import AttnArgs, AttnBwdArgs, Dropout
    before = lib.ns2_launch_count()
    for p in (-0.5, 1.0, float("nan")):
        d = Dropout(1, 0, p)
        assert lib.ns2_attn_fwd(ctypes.byref(AttnArgs(dropout=ctypes.pointer(d))), None) < 0
        assert b"[0, 1)" in lib.ns2_last_error()
        assert lib.ns2_attn_bwd(ctypes.byref(AttnBwdArgs(dropout=ctypes.pointer(d))), None) < 0
        assert b"[0, 1)" in lib.ns2_last_error()
        assert lib.ns2_dropout_f32(16, 4, ctypes.byref(d), None) < 0
        assert b"[0, 1)" in lib.ns2_last_error()
    assert lib.ns2_dropout_f32(16, 4, None, None) < 0
    assert lib.ns2_dropout_f32(None, 0, ctypes.byref(Dropout(1, 0, 0.5)), None) == 0   # empty: nothing to do
    assert lib.ns2_launch_count() == before


def test_dropout_struct_and_abi_version_match_header():
    from naturalspeech2_pytorch_b200._lib import Dropout
    src = textwrap.dedent('''
        #include <stddef.h>
        #include <stdio.h>
        #include "ns2_b200.h"
        int main(void) {
          printf("%zu %zu %zu %zu %d\\n", sizeof(ns2_dropout), offsetof(ns2_dropout, seed), offsetof(ns2_dropout, site),
                 offsetof(ns2_dropout, p), NS2_ABI_VERSION);
          return 0;
        }
    ''')
    with tempfile.TemporaryDirectory() as d:
        c = Path(d) / "t.c"
        c.write_text(src)
        exe = Path(d) / "t"
        subprocess.run(["gcc", "-I", str(ROOT / "include"), str(c), "-o", str(exe)], check=True)
        out = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert out[:4] == [ctypes.sizeof(Dropout), Dropout.seed.offset, Dropout.site.offset, Dropout.p.offset]
    assert out[4] == 9


def test_train_dropout_defaults_off_and_conditioner_plumbs_it():
    from naturalspeech2_pytorch_b200.encoders import Conditioner, PhonemeEncoder, SpeechPromptEncoder
    spe = SpeechPromptEncoder(dim_codebook=128, dims=(256,), depth=1, heads=2, dropout=0.3)
    pe = PhonemeEncoder(num_tokens=10, dim=128, dim_hidden=128, depth=1, heads=2, conv_dropout=0.25, attn_dropout=0.1)
    assert not spe.train_dropout and not pe.train_dropout
    assert spe.attn_dropout == 0.3 and (pe.conv_dropout, pe.attn_dropout) == (0.25, 0.1)
    spe.train()
    assert spe._dropout_seed() is None                  # off by default: nothing drawn
    spe.train_dropout = True
    import torch
    torch.manual_seed(3)
    s1 = spe._dropout_seed()
    torch.manual_seed(3)
    assert s1 == spe._dropout_seed() and 0 <= s1 < 2 ** 63
    spe.eval()
    assert spe._dropout_seed() is None
    assert not Conditioner(num_phoneme_tokens=10).prompt_enc.train_dropout
    c = Conditioner(num_phoneme_tokens=10, train_dropout=True)
    assert c.prompt_enc.train_dropout and c.phoneme_enc.train_dropout
    assert c.prompt_enc.attn_dropout == 0.2 and c.phoneme_enc.conv_dropout == 0.2   # the reference's defaults


def test_dropout_attention_backward_spills_no_more_than_the_plain_one():
    from naturalspeech2_pytorch_b200 import build
    try:
        nvcc = build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not found")
    with tempfile.TemporaryDirectory() as d:
        res = subprocess.run([nvcc, *build.NVCC_FLAGS, "-I", str(build.INCLUDE), "-Xptxas", "-v", "-cubin", "-o",
                              str(Path(d) / "a.cubin"), str(build.CSRC / "attn_bwd.cu")], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    spills, cur = {}, None
    for line in (res.stdout + res.stderr).splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", line)
        if m:
            cur = m.group(1)
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur and "attn_bwd_kernel" in cur:
            spills["ILb1E" in cur] = (int(m.group(1)), int(m.group(2)))
    assert set(spills) == {False, True}, spills
    assert spills[True][0] <= spills[False][0] and spills[True][1] <= spills[False][1], spills
