"""TEST INFRASTRUCTURE ONLY.  Compiles the reference's ASMK Hamming module where it lies
(/root/reference/VSLAM/thirdparty/mast3r/asmk/asmk/cython/hamming.pyx, cythonized as its cython/build.sh does) into
oracle/_ref/hamming/ (git-ignored).  Nothing is copied into the repository: Cython's C output and the extension are build
products.  Used by tests/golden/make_retrieval_golden.py and the CPU retrieval tests."""
from __future__ import annotations

import subprocess
import sys
import sysconfig
from pathlib import Path

PYX = Path("/root/reference/VSLAM/thirdparty/mast3r/asmk/cython/hamming.pyx")
OUT = Path(__file__).resolve().parent / "_ref" / "hamming"
SO = OUT / ("hamming" + sysconfig.get_config_var("EXT_SUFFIX"))


def build() -> None:
    if SO.exists():
        return
    if not PYX.exists():
        print("[build_hamming] reference asmk absent: skipped")
        return
    import numpy as np
    OUT.mkdir(parents=True, exist_ok=True)
    c_file = OUT / "hamming.c"
    subprocess.run([sys.executable, "-m", "cython", "-3", str(PYX), "-o", str(c_file)], check=True)
    cc = sysconfig.get_config_var("CC") or "gcc"
    subprocess.run(cc.split() + ["-O2", "-shared", "-fPIC", f"-I{sysconfig.get_paths()['include']}",
                                 f"-I{np.get_include()}", str(c_file), "-o", str(SO)], check=True)
    print(f"[build_hamming] built {SO}")


def load():
    """The compiled reference module; FileNotFoundError when it was not built."""
    import importlib.util
    if not SO.exists():
        raise FileNotFoundError(f"{SO} not built")
    spec = importlib.util.spec_from_file_location("hamming", SO)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


if __name__ == "__main__":
    build()
