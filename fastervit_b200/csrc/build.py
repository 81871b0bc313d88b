"""Build libfvit_sm100.so (the C-ABI CUDA library) in-tree with nvcc for sm_90a (H100).

Usage: python -m fastervit_b200.csrc.build [--force] [--verbose]
The .so is written next to the Python package (fastervit_b200/libfvit_sm100.so), where lib.py loads it from;
objects go to fastervit_b200/csrc/build/.
"""
from __future__ import annotations

import hashlib
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

CSRC = Path(__file__).resolve().parent
PKG = CSRC.parent
ROOT = PKG.parent
LIB_PATH = PKG / "libfvit_sm100.so"
OBJ_DIR = CSRC / "build"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
    "-I", str(ROOT / "include"),
]


def _nvcc() -> str:
    cand = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not Path(cand).exists():
        raise RuntimeError("nvcc not found; cannot build libfvit_sm100.so")
    return cand


def sources() -> list[Path]:
    return sorted(CSRC.glob("*.cu"))


def _digest(src: Path) -> str:
    h = hashlib.sha256()
    h.update(" ".join(NVCC_FLAGS).encode())
    h.update(src.read_bytes())
    for hdr in sorted(list(CSRC.glob("*.cuh")) + list(CSRC.glob("*.h")) + list((ROOT / "include").glob("*.h"))):
        h.update(hdr.read_bytes())
    return h.hexdigest()


def _compile(src: Path, verbose: bool) -> Path:
    obj = OBJ_DIR / (src.stem + ".o")
    stamp = OBJ_DIR / (src.stem + ".sha")
    dig = _digest(src)
    if obj.exists() and stamp.exists() and stamp.read_text() == dig:
        return obj
    cmd = [_nvcc(), *NVCC_FLAGS, "-c", str(src), "-o", str(obj)]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
        print(" ".join(cmd), flush=True)
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src.name}:\n{res.stdout}\n{res.stderr}")
    if verbose and res.stderr:
        print(res.stderr, flush=True)
    stamp.write_text(dig)
    return obj


def build(force: bool = False, verbose: bool = False) -> Path:
    OBJ_DIR.mkdir(exist_ok=True)
    if force:
        for f in OBJ_DIR.glob("*"):
            f.unlink()
    srcs = sources()
    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(lambda s: _compile(s, verbose), srcs))
    newest = max(o.stat().st_mtime for o in objs)
    if force or not LIB_PATH.exists() or LIB_PATH.stat().st_mtime < newest:
        cmd = [_nvcc(), "-shared", "-o", str(LIB_PATH), *map(str, objs),
               "-gencode", "arch=compute_90a,code=sm_90a"]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError(f"link failed:\n{res.stdout}\n{res.stderr}")
    return LIB_PATH


if __name__ == "__main__":
    p = build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
    print(p)
