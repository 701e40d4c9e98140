"""In-tree build of libv3d_b200.so (sm_90a, H100) with plain nvcc; no torch, no CMake.

`python -m v3d_b200.build` compiles every csrc/*.cu that changed into build/obj and links
v3d_b200/_lib/libv3d_b200.so.  Both are build products and stay out of git.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

ROOT = Path(__file__).resolve().parent
REPO = ROOT.parent
CSRC = ROOT / "csrc"
INCLUDE = REPO / "include"
OBJ_DIR = REPO / "build" / "obj"
LIB_DIR = ROOT / "_lib"
LIB_PATH = LIB_DIR / "libv3d_b200.so"

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = [
    *ARCH,
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
    # keep the embedded cubin uncompressed (nvcc compresses large fat binaries by default): no decompression at load
    "--no-compress",
    "-I", str(INCLUDE), "-I", str(CSRC),
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and Path(cand).exists():
            return cand
    raise RuntimeError("nvcc not found; cannot build libv3d_b200.so")


def _digest(src: Path) -> str:
    h = hashlib.sha256()
    h.update(" ".join(NVCC_FLAGS).encode())
    h.update(src.read_bytes())
    for hdr in sorted(list(CSRC.glob("*.cuh")) + list(INCLUDE.glob("*.h"))):
        h.update(hdr.read_bytes())
    return h.hexdigest()


def _compile_one(nvcc: str, src: Path, verbose: bool) -> Path:
    obj = OBJ_DIR / (src.stem + ".o")
    stamp = OBJ_DIR / (src.stem + ".sha")
    dig = _digest(src)
    if obj.exists() and stamp.exists() and stamp.read_text() == dig:
        return obj
    cmd = [nvcc, *NVCC_FLAGS, "-c", str(src), "-o", str(obj)]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src.name}:\n{res.stdout}\n{res.stderr}")
    if verbose:
        sys.stderr.write(res.stderr)
    stamp.write_text(dig)
    return obj


def build(verbose: bool = False, force: bool = False) -> Path:
    nvcc = _nvcc()
    OBJ_DIR.mkdir(parents=True, exist_ok=True)
    LIB_DIR.mkdir(parents=True, exist_ok=True)
    if force:
        for f in OBJ_DIR.glob("*.sha"):
            f.unlink()
    srcs = sorted(CSRC.glob("*.cu"))
    if not srcs:
        raise RuntimeError("no CUDA sources found")
    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(lambda s: _compile_one(nvcc, s, verbose), srcs))
    newest = max(o.stat().st_mtime for o in objs)
    if force or not LIB_PATH.exists() or LIB_PATH.stat().st_mtime < newest:
        cmd = [nvcc, "-shared", *ARCH, "-Xcompiler", "-fPIC", "--no-compress",
               "-o", str(LIB_PATH), *map(str, objs)]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError(f"link failed:\n{res.stdout}\n{res.stderr}")
    return LIB_PATH


if __name__ == "__main__":
    p = build(verbose="-v" in sys.argv, force="-f" in sys.argv)
    print(p)
