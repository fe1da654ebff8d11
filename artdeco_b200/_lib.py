"""ctypes binding of ``libartdeco_b200.so`` — the only way Python reaches the CUDA kernels.

There is deliberately no CPU fallback anywhere in the package: if the shared library is missing and
cannot be built, or a tensor is not a contiguous CUDA tensor of the expected dtype, we raise.
"""
from __future__ import annotations

import ctypes as C
import os
import threading
from pathlib import Path

import torch

_PKG = Path(__file__).resolve().parent
LIB_PATH = _PKG / "libartdeco_b200.so"

_lib = None
_lock = threading.Lock()

vp, i32, i64, f32 = C.c_void_p, C.c_int, C.c_longlong, C.c_float

# name -> argtypes; every function returns int status (0 = ok) unless noted in _RESTYPES.
# Must list exactly the symbols include/artdeco_b200.h declares (tests/test_abi.py checks this).
_SIGS = {
    "adb_version": [],
    "adb_check_device": [],
    "adb_ssim_forward": [i32, i32, i32, i32, f32, f32, vp, vp, i32, vp, vp, vp, vp, vp, vp],
    "adb_ssim_backward": [i32, i32, i32, i32, f32, f32, vp, vp, vp, vp, f32, vp, vp, vp, vp, vp],
}
_RESTYPES = {"adb_last_error": C.c_char_p}


class ArtdecoB200Error(RuntimeError):
    pass


def register(name: str, argtypes: list) -> None:
    """Sub-modules register their C signatures here (keeps each binding next to its wrapper)."""
    _SIGS[name] = argtypes
    if _lib is not None:
        fn = getattr(_lib, name)
        fn.argtypes = argtypes
        fn.restype = C.c_int


def lib() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not LIB_PATH.exists() or os.environ.get("ADB_REBUILD") == "1":
            from . import build as _build  # needs nvcc; raises loudly if it cannot build
            _build.build()
        try:
            handle = C.CDLL(str(LIB_PATH))
        except OSError as e:  # pragma: no cover
            raise ArtdecoB200Error(f"cannot load {LIB_PATH}: {e}") from e
        handle.adb_last_error.restype = C.c_char_p
        handle.adb_last_error.argtypes = []
        for name, argtypes in _SIGS.items():
            try:
                fn = getattr(handle, name)
            except AttributeError as e:
                raise ArtdecoB200Error(f"{LIB_PATH} does not export {name}; rebuild with "
                                       f"`python -m artdeco_b200.build -f`") from e
            fn.argtypes = argtypes
            fn.restype = C.c_int
        _lib = handle
    return _lib


# Kernel launches issued by one call of each entry point.
LAUNCHES = {
    "adb_ssim_forward": 1, "adb_ssim_backward": 1, "adb_raster_project_fwd": 1, "adb_raster_blend_fwd": 1,
    "adb_raster_blend_bwd": 1, "adb_raster_project_bwd": 1,
    "adb_raster_project_fwd_legacy": 1, "adb_raster_blend_fwd_legacy": 1,
    "adb_raster_blend_bwd_legacy": 1, "adb_raster_tile_count_scan": 2,
    "adb_raster_project_bwd_multi": 1, "adb_raster_sh_bwd_multi": 1, "adb_raster_sh_dir_bwd_multi": 1,
    "adb_raster_sh_expand_multi": 1, "adb_raster_project_fwd_counts": 1, "adb_raster_tile_scan": 1,
    "adb_raster_project_fwd_multi": 1, "adb_raster_tile_scan_multi": 1,
    "adb_raster_blend_fwd_multi": 1, "adb_raster_blend_bwd_multi": 1,
    "adb_raster_tile_band_scatter_sort": 3, "adb_raster_tile_band_scatter_sort_multi": 3,
}


class StageTimer:
    """Optional per-entry-point device timing (CUDA events on the launching stream) and launch counting, used by
    bench.py to report the dominant kernel's live duration.  Off by default: zero overhead on the product path."""

    def __init__(self):
        self.events: dict[str, list] = {}
        self.launches = 0

    def reset(self):
        self.events.clear()
        self.launches = 0

    def totals_ms(self) -> dict[str, tuple[float, int]]:
        out = {}
        for k, evs in self.events.items():
            out[k] = (sum(a.elapsed_time(b) for a, b in evs), len(evs))
        return out


TIMER: StageTimer | None = None


def call(name: str, *args) -> None:
    if TIMER is not None and name in LAUNCHES:
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        rc = getattr(lib(), name)(*args)
        b.record()
        TIMER.events.setdefault(name, []).append((a, b))
        TIMER.launches += LAUNCHES[name]
    else:
        rc = getattr(lib(), name)(*args)
    if rc != 0:
        msg = lib().adb_last_error()
        raise ArtdecoB200Error(f"{name} failed (status {rc}): {msg.decode() if msg else '?'}")


_checked_devices: set[int] = set()


def require_cuda(t: torch.Tensor | None = None) -> None:
    """Fail loudly when there is no sm_90 device: the product path has no CPU implementation."""
    if not torch.cuda.is_available():
        raise ArtdecoB200Error("artdeco_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback")
    if t is not None and not t.is_cuda:
        raise ArtdecoB200Error("expected a CUDA tensor: artdeco_b200 has no CPU implementation")
    dev =t.device.index if (t is not None and t.is_cuda) else torch.cuda.current_device()
    if dev not in _checked_devices:
        with torch.cuda.device(dev):
            call("adb_check_device")
        _checked_devices.add(dev)


def ptr(t: torch.Tensor | None, dtype: torch.dtype | None = None) -> C.c_void_p:
    if t is None:
        return C.c_void_p(0)
    if not t.is_cuda:
        raise ArtdecoB200Error("expected a CUDA tensor (no CPU fallback in artdeco_b200)")
    if not t.is_contiguous():
        raise ArtdecoB200Error("expected a contiguous tensor")
    if dtype is not None and t.dtype != dtype:
        raise ArtdecoB200Error(f"expected dtype {dtype}, got {t.dtype}")
    return C.c_void_p(t.data_ptr())


def stream() -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)
