"""Recipe for oracle/_ref: the UNMODIFIED reference package (lucidrains/naturalspeech2-pytorch), pip-installed from a
source checkout without its dependencies.  The reference arm of bench.py (`--impl reference`, the in-run parity leg)
and tests/test_dropin_cpu.py import it from there; without it they fall back to the oracle port or skip.

The source checkout is taken from $NS2_REFERENCE_SRC (default /root/reference).  oracle/_ref is a build product:
git-ignored, created once, never edited by hand."""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
import tempfile
from pathlib import Path

DST = Path(__file__).resolve().parent / "_ref"


def install() -> None:
    src = Path(os.environ.get("NS2_REFERENCE_SRC", "/root/reference"))
    try:
        have_src = os.access(src / "setup.py", os.R_OK)
    except OSError:
        have_src = False
    if (DST / "naturalspeech2_pytorch").exists() or not have_src:
        return
    with tempfile.TemporaryDirectory() as tmp:
        copy = Path(tmp) / "reference"
        # the source may be read-only and setuptools writes build files next to it
        shutil.copytree(src, copy, ignore=shutil.ignore_patterns("__pycache__", "*.egg-info", "build"))
        cmd = [sys.executable, "-m", "pip", "install", "--no-index", "--no-build-isolation", "--no-deps",
               "--target", str(DST), str(copy)]
        env = dict(os.environ, PIP_CACHE_DIR=str(Path(tmp) / "pip-cache"))
        res = subprocess.run(cmd, capture_output=True, text=True, cwd=tmp, env=env)
    if res.returncode != 0:
        shutil.rmtree(DST, ignore_errors=True)
        print(f"reference install into {DST} failed (the reference arm will use the oracle port):\n{res.stderr[-400:]}")
    else:
        print(f"installed the reference into {DST}")


if __name__ == "__main__":
    install()
