"""In-tree build of the sm_90a (H100) CUDA library (libtooncrafter_b200.so) with plain nvcc.

The .so and the object files are build products (git-ignored).  nvcc cross-compiles without a GPU, so the
library can be built on a machine that has none.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from pathlib import Path

PKG_DIR = Path(__file__).resolve().parent
CSRC = PKG_DIR / "csrc"
LIB_PATH = PKG_DIR / "libtooncrafter_b200.so"
STAMP = PKG_DIR / ".build_stamp"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "-Xptxas", "-v",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and Path(cand).exists():
            return cand
    raise RuntimeError("nvcc not found (needed to build tooncrafter_b200's CUDA library)")


def _sources() -> list[Path]:
    return sorted(list(CSRC.glob("*.cu")) + list(CSRC.glob("*.cpp")))


def _digest() -> str:
    h = hashlib.sha256()
    files = _sources() + sorted(CSRC.glob("*.cuh")) + sorted(CSRC.glob("*.h"))
    files.append(PKG_DIR.parent / "include" / "tooncrafter_b200.h")
    for f in files:
        h.update(f.name.encode())
        h.update(f.read_bytes())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> Path:
    """Compile csrc/*.cu + *.cpp into libtooncrafter_b200.so (no-op when sources are unchanged)."""
    digest = _digest()
    if not force and LIB_PATH.exists() and STAMP.exists() and STAMP.read_text().strip() == digest:
        return LIB_PATH
    nvcc = _nvcc()
    objdir = PKG_DIR / "build"
    objdir.mkdir(exist_ok=True)
    objs = []
    procs = []
    for src in _sources():
        obj = objdir / (src.stem + ".o")
        cmd = [nvcc, *NVCC_FLAGS, "-x", "cu", "-c", str(src), "-o", str(obj)]
        procs.append((src, obj, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    log = []
    failed = False
    for src, obj, pr in procs:
        out, _ = pr.communicate()
        log.append(f"== {src.name}\n{out}")
        if pr.returncode != 0:
            failed = True
        objs.append(str(obj))
    (objdir / "build.log").write_text("\n".join(log))
    if failed:
        sys.stderr.write("\n".join(log))
        raise RuntimeError("nvcc failed; see tooncrafter_b200/build/build.log")
    if verbose:
        print("\n".join(log))
    link = [nvcc, "-shared", "-o", str(LIB_PATH), *objs, "-lcudart"]
    r = subprocess.run(link, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError("link failed")
    STAMP.write_text(digest)
    return LIB_PATH


if __name__ == "__main__":
    p = build(force="--force" in sys.argv, verbose=True)
    print("built", p)
