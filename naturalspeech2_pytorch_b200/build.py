"""Build libns2b200.so (the sm_90a kernels + C ABI) in-tree with nvcc.

`nvcc` cross-compiles for sm_90a without a GPU, so the library can be built on a machine without one.  The build
products (`lib/`, `build/`) are git-ignored.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

PKG_DIR = Path(__file__).resolve().parent
CSRC = PKG_DIR / "csrc"
INCLUDE = PKG_DIR.parent / "include"
LIB_DIR = PKG_DIR / "lib"
LIB_PATH = LIB_DIR / "libns2b200.so"
OBJ_DIR = PKG_DIR / "build" / "obj"

SOURCES = ["host_common.cu", "elementwise.cu", "gemm.cu", "attn.cu", "rvq.cu", "rvq_ce.cu", "wgrad.cu", "backward.cu", "attn_bwd.cu", "align.cu",
           "encoder_bwd.cu", "seanet.cu", "fold.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and Path(cand).exists():
            return cand
    raise RuntimeError("nvcc not found (set NVCC=/path/to/nvcc)")


def _fingerprint() -> str:
    h = hashlib.sha256()
    for p in sorted(list(CSRC.glob("*.cu")) + list(CSRC.glob("*.cuh")) + list(CSRC.glob("*.h"))
                    + list(INCLUDE.glob("*.h"))):
        h.update(p.name.encode())
        h.update(p.read_bytes())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def is_fresh() -> bool:
    stamp = LIB_DIR / "libns2b200.stamp"
    return LIB_PATH.exists() and stamp.exists() and stamp.read_text().strip() == _fingerprint()


def build(force: bool = False, verbose: bool = False) -> Path:
    """Compile every CUDA source for sm_90a and link the shared library.  Returns its path."""
    if not force and is_fresh():
        return LIB_PATH
    nvcc = _nvcc()
    OBJ_DIR.mkdir(parents=True, exist_ok=True)
    LIB_DIR.mkdir(parents=True, exist_ok=True)

    def compile_one(src: str) -> Path:
        obj = OBJ_DIR / (Path(src).stem + ".o")
        cmd = [nvcc, *NVCC_FLAGS, "-I", str(INCLUDE), "-c", str(CSRC / src), "-o", str(obj)]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{res.stdout}\n{res.stderr}")
        if verbose:
            sys.stderr.write(res.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=min(len(SOURCES), os.cpu_count() or 4)) as ex:
        objs = list(ex.map(compile_one, SOURCES))

    link = [nvcc, "-shared", "-o", str(LIB_PATH), *map(str, objs),
            "-gencode", "arch=compute_90a,code=sm_90a", "-cudart", "static"]
    res = subprocess.run(link, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError(f"link failed:\n{res.stdout}\n{res.stderr}")
    (LIB_DIR / "libns2b200.stamp").write_text(_fingerprint())
    return LIB_PATH


if __name__ == "__main__":
    path = build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(path)
