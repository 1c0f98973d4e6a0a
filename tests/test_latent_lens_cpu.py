"""CPU: the C entry points and Python front ends of per-sample latent lengths refuse malformed calls before any launch,
and the length-aware GEMM instantiations keep the epilogue's load discipline.

- include/ns2_b200.h declares the lengths where the other optional inputs live: `row_lens` in ns2_gemm_args, `q_lens`
  in ns2_attn_args and a trailing `lens` argument of ns2_rmsnorm_film, ns2_mse_rows and ns2_mse_bwd; no `_lens` twin
  of an entry point is declared, bound or exported.  NULL arguments, a batch over NS2_GEMM_ROW_LENS_MAX_BATCHES and
  q_lens with dropout are refused with nothing launched.
- `ops.gemm(row_lens=)`, `ops.attention(q_lens=)`, `ops.rmsnorm_film(lens=)`, `ops.mse_rows(lens=)` and
  `ops.mse_bwd(lens=)` reject lengths of the wrong dtype or shape before the device check, `Model.forward(lengths=)`
  rejects batches over the cap, and `NaturalSpeech2.forward(latent_lens=)` refuses raw audio and the RVQ
  cross-entropy term.
- SASS (`cuobjdump -sass` of gemm.cu built for sm_90a): the length-aware BF16 / GEGLU / WAVENET kernels contain no
  global load, the F32 ones only the per-row residual read LDG.E.64, and every one stages the lengths through LDGSTS.
"""
import ctypes
import re
import subprocess
from pathlib import Path

import pytest
import torch

from naturalspeech2_pytorch_b200 import _lib, build as _build, ops

ROOT = Path(__file__).resolve().parent.parent
# the entry points' former length-taking twins (entry point + suffix)
TWINS = [entry + suffix for entry, suffix in [("ns2_gemm", "_row_lens"), ("ns2_attn_fwd", "_q_lens"),
                                              ("ns2_attn_bwd", "_kv_lens"), ("ns2_rmsnorm_film", "_lens"),
                                              ("ns2_mse_rows", "_lens"), ("ns2_mse_bwd", "_lens")]]


@pytest.fixture(scope="module")
def lib():
    _build.build()
    return _lib.load()


def _struct(header, name):
    return re.search(rf"typedef struct {name} \{{([^}}]*)\}} {name};", header).group(1)


def test_lengths_are_fields_or_trailing_arguments_of_the_entry_points(lib):
    header = (ROOT / "include" / "ns2_b200.h").read_text()
    assert re.search(r"\bconst int32_t\* row_lens;", _struct(header, "ns2_gemm_args"))
    assert re.search(r"\bconst int32_t\* q_lens;", _struct(header, "ns2_attn_args"))
    assert "row_lens" in dict(_lib.GemmArgs._fields_) and "q_lens" in dict(_lib.AttnArgs._fields_)
    for name, tail in [("ns2_rmsnorm_film", r"const int32_t\* lens"),
                       ("ns2_mse_rows", r"int64_t row_elems, const int32_t\* lens"),
                       ("ns2_mse_bwd", r"int64_t row_elems, const int32_t\* lens")]:
        assert re.search(rf"\bint {name}\([^;]*{tail},\s+ns2_stream_t stream\);", header), name
        params = re.sub(r"/\*.*?\*/", "", re.search(rf"\bint {name}\(([^;]*)\);", header).group(1), flags=re.S)
        assert len(_lib.SIGNATURES[name][1]) == len(params.split(",")), name
        assert getattr(lib, name) is not None
    assert not re.findall(r"\b(ns2_\w+_lens)\s*\(", header)
    assert not [name for name in _lib.SIGNATURES if name.endswith("_lens")]
    for name in TWINS:
        assert not re.search(rf"\b{name}\b", header), name
        assert name not in _lib.SIGNATURES, name
        assert not hasattr(lib, name), name
    assert re.search(rf"#define NS2_GEMM_ROW_LENS_MAX_BATCHES {_lib.NS2_GEMM_ROW_LENS_MAX_BATCHES}\b", header)


def test_length_calls_refuse_null_and_malformed_arguments(lib):
    before = lib.ns2_launch_count()
    lens = (ctypes.c_int32 * 4)(1, 2, 3, 4)
    lens_ptr = ctypes.addressof(lens)
    assert lib.ns2_gemm(None, None) < 0
    a = _lib.GemmArgs(a_batches=1, row_lens=lens_ptr)
    assert lib.ns2_gemm(ctypes.byref(a), None) < 0                              # NULL A / B / out
    assert b"non-NULL" in lib.ns2_last_error()
    a.A = a.B = a.out = 16
    a.a_batches = _lib.NS2_GEMM_ROW_LENS_MAX_BATCHES + 1
    assert lib.ns2_gemm(ctypes.byref(a), None) < 0
    assert b"batches" in lib.ns2_last_error()
    assert lib.ns2_attn_fwd(None, None) < 0
    assert lib.ns2_attn_fwd(ctypes.byref(_lib.AttnArgs(q_lens=lens_ptr)), None) < 0   # NULL q / k / v / out
    d = _lib.Dropout(1, 0, 0.5)
    t = _lib.AttnArgs(q=16, k=16, v=16, out=16, batches=1, heads=1, q_len=8, kv_len=8, dim_head=64,
                      dropout=ctypes.pointer(d), q_lens=lens_ptr)
    assert lib.ns2_attn_fwd(ctypes.byref(t), None) < 0
    assert b"q_lens" in lib.ns2_last_error()
    assert lib.ns2_rmsnorm_film(None, 128, 8, 128, 4, None, None, 0, None, 128, lens, None) < 0
    assert lib.ns2_rmsnorm_film(16, 128, 9, 128, 4, None, None, 0, 16, 128, lens, None) < 0   # 9 rows, 4 per batch
    assert lib.ns2_mse_rows(None, 16, 2, 64, 16, 16, None, 32, lens, None) < 0
    assert lib.ns2_mse_rows(16, 16, 2, 64, 16, 16, None, 24, lens, None) < 0     # 24 does not divide 64
    assert lib.ns2_mse_bwd(16, 16, 16, 2, 64, None, None, 32, lens, None) < 0    # no output
    assert lib.ns2_mse_bwd(16, 16, 16, 2, 64, None, 16, 6, lens, None) < 0       # row not a multiple of 4
    assert lib.ns2_launch_count() == before


def _f(*s, dtype=torch.float32):
    return torch.zeros(*s, dtype=dtype)


@pytest.mark.parametrize("bad, match", [(_f(2, dtype=torch.int64), "int32"), (_f(3, dtype=torch.int32), r"\(2\)"),
                                        (_f(2, dtype=torch.float32), "int32")])
def test_ops_reject_bad_lengths_before_the_device_check(lib, bad, match):
    bf = torch.bfloat16
    calls = [
        lambda: ops.gemm(_f(2, 8, 64, dtype=bf), _f(64, 64, dtype=bf), _f(2, 8, 64, dtype=bf), n=64,
                         epilogue=ops.EPI_BF16, row_lens=bad),
        lambda: ops.attention(_f(2, 8, 64, dtype=bf), _f(2, 8, 64, dtype=bf), _f(2, 8, 64, dtype=bf),
                              _f(2, 8, 64, dtype=bf), heads=1, q_lens=bad),
        lambda: ops.rmsnorm_film(_f(2, 8, 128), _f(2, 8, 128, dtype=bf), lens=bad),
        lambda: ops.mse_rows(_f(2, 8, 64), _f(2, 8, 64), _f(2), lens=bad),
        lambda: ops.mse_bwd(_f(2, 8, 64), _f(2, 8, 64), _f(2), out_f32=_f(2, 8, 64), lens=bad),
    ]
    before = lib.ns2_launch_count()
    for call in calls:
        with pytest.raises(ValueError, match=match) as e:
            call()
        assert "CUDA" not in str(e.value)
    assert lib.ns2_launch_count() == before


def test_gemm_refuses_batches_over_the_cap(lib):
    Bb = _lib.NS2_GEMM_ROW_LENS_MAX_BATCHES + 1
    bf = torch.bfloat16
    with pytest.raises(ValueError, match="at most"):
        ops.gemm(_f(Bb, 8, 64, dtype=bf), _f(64, 64, dtype=bf), _f(Bb, 8, 64, dtype=bf), n=64, epilogue=ops.EPI_BF16,
                 row_lens=_f(Bb, dtype=torch.int32))


def test_attention_refuses_q_lens_with_dropout(lib):
    bf = torch.bfloat16
    with pytest.raises(ValueError, match="dropout"):
        ops.attention(_f(2, 8, 64, dtype=bf), _f(2, 8, 64, dtype=bf), _f(2, 8, 64, dtype=bf), _f(2, 8, 64, dtype=bf),
                      heads=1, q_lens=_f(2, dtype=torch.int32), dropout=(1, 0, 0.1))


def test_model_refuses_batches_over_the_cap():
    from naturalspeech2_pytorch_b200 import Model
    model = Model(dim=128, depth=1, heads=2, wavenet_layers=1, wavenet_stacks=1).eval()
    Bb = _lib.NS2_GEMM_ROW_LENS_MAX_BATCHES + 1
    with pytest.raises(ValueError, match="at most"):
        model(torch.zeros(Bb, 8, 128), torch.zeros(Bb), lengths=[8] * Bb)


# ---- SASS of the length-aware GEMM instantiations ----
EPI = {0: "BF16", 1: "F32", 2: "GEGLU", 3: "WAVENET"}
KERNEL = re.compile(r"gemm_kernelILi(\d+)ELi(\d+)ELi(\d+)ELb([01])E")
OPCODE = re.compile(r"/\*[0-9a-f]{4}\*/\s+(?:@!?U?P[T0-9]+\s+)?([A-Z][A-Z0-9_.]*)")


@pytest.fixture(scope="module")
def gemm_sass(tmp_path_factory):
    try:
        nvcc = Path(_build._nvcc())
    except RuntimeError:
        pytest.skip("nvcc not found")
    cuobjdump = nvcc.parent / "cuobjdump"
    if not cuobjdump.exists():
        pytest.skip("cuobjdump not found")
    cubin = tmp_path_factory.mktemp("sass") / "gemm.cubin"
    res = subprocess.run([str(nvcc), *_build.NVCC_FLAGS, "-I", str(_build.INCLUDE), "-cubin", "-o", str(cubin),
                          str(_build.CSRC / "gemm.cu")], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    res = subprocess.run([str(cuobjdump), "-sass", str(cubin)], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr
    kernels = {}
    for block in re.split(r"\n\s*Function : ", res.stdout)[1:]:
        m = KERNEL.search(block.split("\n", 1)[0])
        if m:
            bn, nacc, epi, lens = (int(x) for x in m.groups())
            kernels[(bn, nacc, EPI[epi], bool(lens))] = OPCODE.findall(block)
    return kernels


def test_length_aware_instantiations_exist(gemm_sass):
    plain = {k[:3] for k in gemm_sass if not k[3]}
    aware = {k[:3] for k in gemm_sass if k[3]}
    assert plain == aware == {(256, 1, "BF16"), (128, 1, "BF16"), (256, 1, "F32"), (128, 1, "F32"), (256, 1, "GEGLU"),
                              (128, 2, "WAVENET")}


def test_length_aware_kernels_load_nothing_through_registers(gemm_sass):
    for key, code in gemm_sass.items():
        if not key[3]:
            continue
        loads = {o for o in code if o == "LDG" or o.startswith("LDG.")}
        allowed = {"LDG.E.64"} if key[2] == "F32" else set()
        assert loads <= allowed, f"gemm_kernel{key}: global loads {sorted(loads)}"
        # the lengths (and the column vectors) arrive by cp.async; the plain kernel of the same shape has fewer LDGSTS
        plain = gemm_sass[key[:3] + (False,)]
        n_aware = sum(o.startswith("LDGSTS") for o in code)
        n_plain = sum(o.startswith("LDGSTS") for o in plain)
        assert n_aware > n_plain, f"gemm_kernel{key}: lengths not staged by LDGSTS ({n_aware} vs {n_plain})"


def test_training_refusals_before_any_launch(lib):
    """NaturalSpeech2.forward(latent_lens=) refuses raw audio and the RVQ cross-entropy term before anything runs."""
    from naturalspeech2_pytorch_b200 import Model, NaturalSpeech2
    ns = NaturalSpeech2(Model(dim=128, depth=1, heads=2, wavenet_layers=1, wavenet_stacks=1), target_sample_hz=24000,
                        timesteps=3)
    before = lib.ns2_launch_count()
    with pytest.raises(ValueError, match="encoded latents"):
        ns(torch.zeros(2, 3200), latent_lens=[8, 10])
    ns.rvq_cross_entropy_loss_weight = 0.5
    with pytest.raises(NotImplementedError, match="cross-entropy"):
        ns(torch.zeros(2, 10, 128), codes=torch.zeros(2, 10, 8, dtype=torch.long), latent_lens=[8, 10])
    assert lib.ns2_launch_count() == before
