"""CPU: what ptxas makes of the sm_90a kernels.

Every csrc/*.cu is compiled for sm_90a with `-Xptxas -v` (no GPU needed).  The test fails when ptxas reports that it
serialized a kernel's wgmma.mma_async instructions (advisories C7510 / C7520: one MMA at a time, each waited for
before the next is issued, e.g. because a function call such as printf sits inside the kernel), and when a GEMM or
attention-forward instantiation spills registers to local memory.
"""
import os
import re
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
from naturalspeech2_pytorch_b200 import build as _build  # noqa: E402


def _nvcc():
    try:
        return _build._nvcc()
    except RuntimeError:
        return None


NVCC = _nvcc()
pytestmark = pytest.mark.skipif(NVCC is None, reason="nvcc not found")
SOURCES = sorted(p.name for p in _build.CSRC.glob("*.cu"))
NO_SPILL = re.compile(r"gemm_kernel|attn_fwd_kernel")


@pytest.fixture(scope="module")
def ptxas_logs(tmp_path_factory):
    out = tmp_path_factory.mktemp("cubin")

    def one(src):
        cmd = [NVCC, *_build.NVCC_FLAGS, "-I", str(_build.INCLUDE), "-Xptxas", "-v", "-cubin",
               "-o", str(out / (Path(src).stem + ".cubin")), str(_build.CSRC / src)]
        res = subprocess.run(cmd, capture_output=True, text=True)
        assert res.returncode == 0, f"nvcc failed for {src}:\n{res.stderr}"
        return src, res.stdout + res.stderr

    with ThreadPoolExecutor(max_workers=min(len(SOURCES), os.cpu_count() or 4)) as ex:
        return dict(ex.map(one, SOURCES))


def _per_kernel(log):
    """{mangled kernel name: [ptxas lines about it]}: the lines after each 'Compiling entry function' header, plus
    advisories that name the function."""
    kernels, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", line)
        if m:
            cur = m.group(1)
            kernels.setdefault(cur, [])
            continue
        m = re.search(r"in (?:the )?function '([^']+)'", line)
        if m:
            kernels.setdefault(m.group(1), []).append(line)
        elif cur is not None:
            kernels[cur].append(line)
    return kernels


@pytest.mark.parametrize("src", SOURCES)
def test_no_serialized_wgmma(ptxas_logs, src):
    bad = [l for l in ptxas_logs[src].splitlines() if re.search(r"C75(10|20)\b", l)]
    assert not bad, f"{src}: ptxas serialized wgmma:\n" + "\n".join(bad)


@pytest.mark.parametrize("src", ["gemm.cu", "attn.cu"])
def test_hot_kernels_do_not_spill(ptxas_logs, src):
    kernels = {k: v for k, v in _per_kernel(ptxas_logs[src]).items() if NO_SPILL.search(k)}
    assert kernels, f"{src}: no gemm_kernel / attn_fwd_kernel instantiation found in the ptxas output"
    for name, lines in kernels.items():
        for line in lines:
            m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
            if m:
                assert m.group(1) == "0" and m.group(2) == "0", f"{name} spills: {line.strip()}"


def test_every_source_is_checked():
    assert set(SOURCES) >= {"gemm.cu", "attn.cu", "attn_bwd.cu", "wgrad.cu", "rvq.cu"}
    assert shutil.which(NVCC) or Path(NVCC).exists()
