"""Builds ``libartdeco_b200.so`` (the C-ABI CUDA library) in-tree with nvcc for sm_90a (H100).

The library has no torch/pybind dependency: it is plain CUDA runtime + CUB headers, so it can be
bound from ctypes, cgo, JNI or anything else (see INTEGRATION.md).  Objects are cached by source
mtime so an incremental rebuild only recompiles what changed.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

PKG_DIR = Path(__file__).resolve().parent
CSRC = PKG_DIR / "csrc"
BUILD = PKG_DIR / "build"
LIB_PATH = PKG_DIR / "libartdeco_b200.so"

ARCH_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON_FLAGS = [
    "-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden",
    "--expt-relaxed-constexpr", "-I", str(CSRC), "-I", str(PKG_DIR.parent / "include"),
]
# Per-file extra flags.  raster_project.cu is compiled without FMA contraction so that the values
# feeding the integer tile keys (depth bits, tile bounds) are bit-identical to the C oracle.
PER_FILE_FLAGS = {
    "raster_project.cu": ["-fmad=false"],
    "raster_isect.cu": ["-fmad=false"],
}


def nvcc() -> str:
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(exe):
        raise RuntimeError("nvcc not found; artdeco_b200 needs the CUDA 12.9 toolkit to build")
    return exe


def sources() -> list[Path]:
    return sorted(CSRC.glob("*.cu"))


def _needs_rebuild(obj: Path, src: Path) -> bool:
    if not obj.exists():
        return True
    newest_dep = max([src.stat().st_mtime] + [h.stat().st_mtime for h in CSRC.glob("*.cuh")]
                     + [h.stat().st_mtime for h in (PKG_DIR.parent / "include").glob("*.h")]
                     + [Path(__file__).stat().st_mtime])
    return obj.stat().st_mtime < newest_dep


def _compile(src: Path, verbose: bool) -> Path:
    obj = BUILD / (src.stem + ".o")
    if _needs_rebuild(obj, src):
        cmd = [nvcc(), *ARCH_FLAGS, *COMMON_FLAGS, *PER_FILE_FLAGS.get(src.name, []), "-c", str(src), "-o", str(obj)]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src.name}:\n{res.stdout}\n{res.stderr}")
        if verbose:
            sys.stderr.write(res.stderr)
    return obj


def build(verbose: bool = False, force: bool = False) -> Path:
    BUILD.mkdir(exist_ok=True)
    if force:
        for o in BUILD.glob("*.o"):
            o.unlink()
    srcs = sources()
    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(lambda s: _compile(s, verbose), srcs))
    if (not LIB_PATH.exists()) or any(o.stat().st_mtime > LIB_PATH.stat().st_mtime for o in objs):
        cmd = [nvcc(), *ARCH_FLAGS, "-shared", "-o", str(LIB_PATH), *map(str, objs), "-cudart", "static"]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError(f"link failed:\n{res.stdout}\n{res.stderr}")
    return LIB_PATH


if __name__ == "__main__":
    p = build(verbose="-v" in sys.argv, force="-f" in sys.argv)
    print(p)
