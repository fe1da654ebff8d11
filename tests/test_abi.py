"""The C-ABI shared library loads and exports exactly the symbols include/artdeco_b200.h declares
(no compute calls: runs without a GPU)."""
import ctypes
import re
import subprocess
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]


def header_symbols():
    text = (ROOT / "include" / "artdeco_b200.h").read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(adb_[a-z0-9_]+)\s*\(", text)))


def test_library_builds_and_exports_header_symbols():
    from artdeco_b200 import build
    lib_path = build.build()
    lib = ctypes.CDLL(str(lib_path))
    syms = header_symbols()
    assert len(syms) >= 10
    missing = [s for s in syms if not hasattr(lib, s)]
    assert not missing, f"declared in the header but not exported: {missing}"
    out = subprocess.run(["nm", "-D", "--defined-only", str(lib_path)], capture_output=True, text=True).stdout
    exported = sorted(set(re.findall(r"\bT (adb_[a-z0-9_]+)", out)))
    undeclared = [s for s in exported if s not in syms]
    assert not undeclared, f"exported but not declared in the header: {undeclared}"
    assert lib.adb_version() >= 100


def test_python_binding_table_matches_header():
    from artdeco_b200 import _lib
    import artdeco_b200  # registers every sub-module's signatures
    syms = set(header_symbols()) - {"adb_last_error"}
    assert syms == set(_lib._SIGS), (sorted(syms - set(_lib._SIGS)), sorted(set(_lib._SIGS) - syms))


def test_product_path_never_imports_oracle():
    for py in (ROOT / "artdeco_b200").rglob("*.py"):
        src = py.read_text()
        assert not re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M), f"{py} imports the oracle"
    for py in list((ROOT / "shims").rglob("*.py")) + list((ROOT / "tools").rglob("*.py")):
        src = py.read_text()
        assert not re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M), f"{py} imports the oracle"
    # the two sanctioned users outside tests/: smoke() and the bench's CPU legs -- and only inside those functions
    import ast
    allowed = {"__graft_entry__.py": {"build", "smoke", "_smoke_mast3r"}, "bench.py": {"cpu_oracle_leg", "cpu_mast3r_leg", "bench_mast3r", "bench_ops"}}
    for name, funcs in allowed.items():
        tree = ast.parse((ROOT / name).read_text())
        for node in tree.body:
            inner = [n for n in ast.walk(node) if isinstance(n, (ast.Import, ast.ImportFrom))]
            for imp in inner:
                mods = [a.name for a in imp.names] if isinstance(imp, ast.Import) else [imp.module or ""]
                if any(m == "oracle" or m.startswith("oracle.") for m in mods):
                    assert isinstance(node, ast.FunctionDef) and node.name in funcs, f"{name}: oracle imported outside {funcs}"


def test_no_cpu_fallback_without_gpu():
    import pytest
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from artdeco_b200 import _lib
    from artdeco_b200.ssim import fused_ssim
    with pytest.raises(_lib.ArtdecoB200Error):
        fused_ssim(torch.rand(1, 3, 32, 32), torch.rand(1, 3, 32, 32))


def test_header_is_plain_c_and_cpp(tmp_path):
    """The boundary is a C ABI: include/artdeco_b200.h must compile as C99 and as C++17 with no CUDA or torch headers."""
    import shutil
    inc = ROOT / "include"
    for comp, std, ext in (("gcc", "-std=c99", "c"), ("g++", "-std=c++17", "cpp")):
        exe = shutil.which(comp, path="/usr/bin:/bin") or shutil.which(comp)
        if exe is None:
            continue
        src = tmp_path / f"hdr.{ext}"
        src.write_text('#include "artdeco_b200.h"\nint main(void) { return 0; }\n')
        r = subprocess.run([exe, std, "-Wall", "-Wextra", "-pedantic", "-fsyntax-only", f"-I{inc}", str(src)],
                           capture_output=True, text=True)
        assert r.returncode == 0 and not r.stderr.strip(), r.stderr
    text = (inc / "artdeco_b200.h").read_text()
    assert "torch" not in re.sub(r"/\*.*?\*/", "", text, flags=re.S).lower() and "#include <cuda" not in text


def test_blend_and_split_sh_entry_points_refuse_bad_arguments_before_touching_the_device():
    """Error behaviour of the boundary (status 1 + adb_last_error, no exception, no CUDA call): checked on CPU for the
    shared-culling blend pair and the split SH backward."""
    from artdeco_b200 import _lib
    import artdeco_b200  # noqa: F401  (registers every signature)
    L = _lib.lib()

    def refused(rc, needle):
        msg = L.adb_last_error()
        return rc == 1 and msg is not None and needle in msg.decode()

    hm = ctypes.c_void_p(256)                                                                  # never dereferenced
    for mask in (None, hm):
        assert refused(L.adb_raster_blend_fwd(0, 16, 4, None, None, None, None, None, None, mask, None),
                       "adb_raster_blend_fwd: bad sizes")
        assert refused(L.adb_raster_blend_fwd(16, 16, 4, None, None, None, None, None, None, mask, None),
                       "adb_raster_blend_fwd: null pointer")
        assert refused(L.adb_raster_blend_bwd(16, 16, -1, None, None, None, None, None, None, None, None, mask, None),
                       "adb_raster_blend_bwd: bad sizes")
        assert refused(L.adb_raster_blend_bwd(16, 16, 4, None, None, None, None, None, None, None, None, mask, None),
                       "adb_raster_blend_bwd: null pointer")
        assert refused(L.adb_raster_blend_bwd(16, 16, 4, None, None, hm, hm, hm, hm, hm, None, mask, None),
                       "adb_raster_blend_bwd: null v_splats")
    assert refused(L.adb_raster_sh_expand_multi(4, 0, None, 3, None, None, None, None), "adb_raster_sh_expand_multi")
    assert refused(L.adb_raster_sh_expand_multi(4, 1, None, 4, None, None, None, None), "adb_raster_sh_expand_multi")  # degree > 3
    assert refused(L.adb_raster_sh_dir_bwd_multi(4, 1, None, None, 3, None, None, None, None, None, None),
                   "adb_raster_sh_dir_bwd_multi")
    # empty problems are accepted without a launch
    assert L.adb_raster_sh_expand_multi(0, 1, None, 3, None, None, None, None) == 0
