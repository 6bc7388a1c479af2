"""In-tree build of libneutts_b200.so (sm_90a only) with plain nvcc.

The shared object and the object files are build products (git-ignored), written next to the sources.
``python -m neutts_air_b200.build`` rebuilds them; ``__graft_entry__.build()`` calls ``build()``.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
LIB = PKG / "libneutts_b200.so"
SOURCES = ["lm_api.cu", "lm_kernels.cu", "lm_decode_tc.cu", "gemm_tc.cu", "codec.cu", "resample.cu", "stretch.cu", "loudness.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC",
    "-Xcompiler", "-Wall",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: the sm_90a kernels cannot be built")


def _stamp() -> str:
    h = hashlib.sha256()
    for p in sorted(CSRC.glob("*")) + [PKG.parent / "include" / "neutts_b200.h"]:
        h.update(p.name.encode())
        h.update(p.read_bytes())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> Path:
    stamp_file = PKG / ".build_stamp"
    stamp = _stamp()
    if not force and LIB.exists() and stamp_file.exists() and stamp_file.read_text() == stamp:
        return LIB
    nvcc = _nvcc()
    objdir = PKG / "build"
    objdir.mkdir(exist_ok=True)
    procs = []
    for src in SOURCES:
        obj = objdir / (src + ".o")
        cmd = [nvcc, *NVCC_FLAGS, "-c", str(CSRC / src), "-o", str(obj)]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        procs.append((src, obj, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    objs = []
    for src, obj, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src}:\n{out}")
        if verbose and out:
            print(out)
        objs.append(str(obj))
    cmd = [nvcc, "-shared", "-o", str(LIB), *objs, "-gencode", "arch=compute_90a,code=sm_90a"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}")
    stamp_file.write_text(stamp)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
