"""In-tree build of the sm_90a (H100) shared library (C ABI declared in include/controllora_b200.h).

`python -m controllora_b200.build` compiles every csrc/*.cu with nvcc for sm_90a and links
`controllora_b200/libcontrollora_b200.so`.  Objects are rebuilt only when a source or header is newer.
"""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
OBJ = PKG / "build"
LIB = PKG / "libcontrollora_b200.so"

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
    "-Xptxas", "-v" if os.environ.get("CLB_PTXAS_V") else "-O3",
] + os.environ.get("CLB_EXTRA_NVCC", "").split()


def _newer(a: Path, b: Path) -> bool:
    return (not b.exists()) or a.stat().st_mtime > b.stat().st_mtime


def build(verbose: bool = False, force: bool = False) -> Path:
    OBJ.mkdir(exist_ok=True)
    sources = sorted(CSRC.glob("*.cu"))
    headers = list(CSRC.glob("*.cuh")) + list(CSRC.glob("*.h")) + list((PKG.parent / "include").glob("*.h"))
    newest_hdr = max((h.stat().st_mtime for h in headers), default=0.0)
    jobs = []
    for src in sources:
        obj = OBJ / (src.stem + ".o")
        if force or _newer(src, obj) or newest_hdr > obj.stat().st_mtime:
            jobs.append((src, obj))

    def compile_one(job):
        src, obj = job
        cmd = [NVCC, *FLAGS, "-c", str(src), "-o", str(obj)]
        r = subprocess.run(cmd, capture_output=True, text=True)
        return src, r

    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            for src, r in ex.map(compile_one, jobs):
                if verbose or r.returncode != 0:
                    sys.stderr.write(f"[nvcc] {src.name}\n{r.stdout}{r.stderr}\n")
                if r.returncode != 0:
                    raise RuntimeError(f"nvcc failed on {src}")
    objs = [OBJ / (s.stem + ".o") for s in sources]
    if jobs or not LIB.exists():
        cmd = [NVCC, "-shared", "-o", str(LIB), *map(str, objs), "-lcudart"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("link failed")
    return LIB


if __name__ == "__main__":
    p = build(verbose="-v" in sys.argv, force="-f" in sys.argv)
    print(p)
