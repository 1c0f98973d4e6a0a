"""CPU: the GEMM epilogue reads its column vectors from shared memory, not from global memory.

gemm.cu is compiled for sm_90a (no GPU needed) and the SASS of every `gemm_kernel<BN, NACC, EPI>` instantiation is read
with `cuobjdump -sass`.  The tile's bias, GEGLU value / gate bias and WAVENET bias / FiLM slices are copied into shared
memory by cp.async (LDGSTS) under the tile's mainloop, so the epilogue does not wait out one global-load round trip per
column group.  The BF16, GEGLU and WAVENET kernels therefore contain no global load at all; the F32 kernel keeps only the
read of a residual that is not `out` itself, which is per row (a plain LDG.E.64, not a read-only cached one).
"""
import re
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from naturalspeech2_pytorch_b200 import build as _build  # noqa: E402


def _tools():
    try:
        nvcc = Path(_build._nvcc())
    except RuntimeError:
        return None, None
    cuobjdump = nvcc.parent / "cuobjdump"
    return nvcc, (cuobjdump if cuobjdump.exists() else None)


NVCC, CUOBJDUMP = _tools()
pytestmark = pytest.mark.skipif(CUOBJDUMP is None, reason="nvcc / cuobjdump not found")

EPI = {0: "BF16", 1: "F32", 2: "GEGLU", 3: "WAVENET"}   # NS2_EPI_* in include/ns2_b200.h
KERNEL = re.compile(r"gemm_kernelILi(\d+)ELi(\d+)ELi(\d+)E")
OPCODE = re.compile(r"/\*[0-9a-f]{4}\*/\s+(?:@!?U?P[T0-9]+\s+)?([A-Z][A-Z0-9_.]*)")


@pytest.fixture(scope="module")
def gemm_sass(tmp_path_factory):
    """{(BN, NACC, epilogue name): [SASS opcodes]} for every gemm_kernel instantiation."""
    cubin = tmp_path_factory.mktemp("sass") / "gemm.cubin"
    cmd = [str(NVCC), *_build.NVCC_FLAGS, "-I", str(_build.INCLUDE), "-cubin", "-o", str(cubin),
           str(_build.CSRC / "gemm.cu")]
    res = subprocess.run(cmd, capture_output=True, text=True)
    assert res.returncode == 0, f"nvcc failed for gemm.cu:\n{res.stderr}"
    res = subprocess.run([str(CUOBJDUMP), "-sass", str(cubin)], capture_output=True, text=True)
    assert res.returncode == 0, f"cuobjdump failed:\n{res.stderr}"
    kernels = {}
    for block in re.split(r"\n\s*Function : ", res.stdout)[1:]:
        m = KERNEL.search(block.split("\n", 1)[0])
        if m:
            bn, nacc, epi = (int(x) for x in m.groups())
            kernels[(bn, nacc, EPI[epi])] = OPCODE.findall(block)
    return kernels


def _global_loads(ops):
    return [o for o in ops if o == "LDG" or o.startswith("LDG.")]   # not LDGSTS / LDGDEPBAR


def test_every_instantiation_is_found(gemm_sass):
    assert set(gemm_sass) == {(256, 1, "BF16"), (128, 1, "BF16"), (256, 1, "F32"), (128, 1, "F32"),
                              (256, 1, "GEGLU"), (128, 2, "WAVENET")}
    for key, ops in gemm_sass.items():
        assert any(o.startswith("HGMMA") for o in ops), f"{key}: no wgmma in the parsed SASS"


@pytest.mark.parametrize("epi", ["BF16", "GEGLU", "WAVENET"])
def test_no_global_loads(gemm_sass, epi):
    for key, ops in gemm_sass.items():
        if key[2] != epi:
            continue
        assert not _global_loads(ops), f"gemm_kernel{key}: global loads {sorted(set(_global_loads(ops)))}"
        assert any(o.startswith("LDGSTS") for o in ops), f"gemm_kernel{key}: column vectors not copied by cp.async"


def test_f32_keeps_only_the_residual_read(gemm_sass):
    for key, ops in gemm_sass.items():
        if key[2] != "F32":
            continue
        loads = set(_global_loads(ops))
        assert loads <= {"LDG.E.64"}, f"gemm_kernel{key}: global loads besides the residual read: {sorted(loads)}"
        assert any(o.startswith("LDGSTS") for o in ops), f"gemm_kernel{key}: bias not copied by cp.async"
