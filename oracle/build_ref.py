"""TEST INFRASTRUCTURE ONLY.  Builds the REFERENCE's own CUDA extensions from the sources where they lie under
/root/reference into oracle/_ref/ (git-ignored, travels to the GPU box with the snapshot), for sm_90:
  fused_ssim_ref   <- Reconstruct/submodules/fused-ssim/{ssim.cu,ext.cpp}      (flags of its setup.py:13-23)
  simple_knn_ref   <- Reconstruct/submodules/simple-knn/{simple_knn.cu,spatial.cu,ext.cpp}
  mast3r_matching_ref <- VSLAM/backend/src/matching_kernels.cu + oracle/matching_bind.cpp (our binding; gn.cpp needs Eigen)
No reference source is copied into the repo.  The built modules are used only by tests (bit/tolerance comparison of
our kernels against the real reference on the GPU) and by bench tooling ("reference CUDA build on the same box")."""
from __future__ import annotations

import os
import sys
from pathlib import Path

REF = Path("/root/reference/Reconstruct/submodules")
REF_ROOT = Path("/root/reference")
HERE = Path(__file__).resolve().parent
OUT = Path(__file__).resolve().parent / "_ref"

EXTS = {
    "fused_ssim_ref": dict(sources=["fused-ssim/ssim.cu", "fused-ssim/ext.cpp"],
                           cuda_flags=["-O3", "--maxrregcount=32", "--use_fast_math"]),
    "simple_knn_ref": dict(sources=["simple-knn/simple_knn.cu", "simple-knn/spatial.cu", "simple-knn/ext.cpp"],
                           cuda_flags=["-O3"]),
    # the reference's matching kernels (flags of VSLAM/setup.py:62-67) behind our own two-function binding
    "mast3r_matching_ref": dict(sources=["@VSLAM/backend/src/matching_kernels.cu", "#matching_bind.cpp"],
                                cuda_flags=["-O3", "--use_fast_math", "-include", str(HERE / "ref_compat.h")]),
}


def _src(s: str) -> str:
    if s.startswith("@"):
        return str(REF_ROOT / s[1:])     # relative to the reference root
    if s.startswith("#"):
        return str(HERE / s[1:])         # our own file under oracle/
    return str(REF / s)


def _so(name: str) -> Path:
    return OUT / name / f"{name}.so"


def build_all(verbose: bool = False) -> None:
    if not REF.exists():
        print("[build_ref] /root/reference absent: using prebuilt oracle/_ref if present")
        return
    from torch.utils import cpp_extension
    os.environ["TORCH_CUDA_ARCH_LIST"] = "10.0"
    for name, cfg in EXTS.items():
        if _so(name).exists():
            continue
        bdir = OUT / name
        bdir.mkdir(parents=True, exist_ok=True)
        cpp_extension.load(name=name, sources=[_src(s) for s in cfg["sources"]],
                           extra_cuda_cflags=cfg["cuda_flags"] + ["-gencode", "arch=compute_90,code=sm_90"],
                           extra_cflags=["-O3"], build_directory=str(bdir), verbose=verbose, is_python_module=False)
        print(f"[build_ref] built {_so(name)}")


def load(name: str):
    """Imports a prebuilt reference extension (needs torch; CUDA only when its functions are called)."""
    import importlib.util
    import torch  # noqa: F401
    so = _so(name)
    if not so.exists():
        raise FileNotFoundError(f"{so} not built (run oracle/build_ref.py where /root/reference exists)")
    spec = importlib.util.spec_from_file_location(name, so)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


if __name__ == "__main__":
    build_all(verbose="-v" in sys.argv)
