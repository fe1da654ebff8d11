"""Gradient exchange of the multi-view optimiser step through NVLink peer memory (csrc/peer_exchange.cu).

Same interface and same result as ``parallel.MultiViewExchange`` (all-gather of the 12 B/view colour gradients + all-reduce of
the 11 geometry floats per Gaussian), but the data moves by this library's own kernels storing straight into the other GPUs'
memory through the NVSwitch, ordered by release/acquire step counters — no NCCL call on the data path:

  * gather:  ``adb_peer_push_rgb`` fuses the SH-clamp mask of the colour gradient with the broadcast of the view's row into
    every rank's table (the NCCL path runs a mask kernel, then ``all_gather_into_tensor``);
  * reduce:  ``adb_peer_scatter`` (reduce-scatter by push) + ``adb_peer_reduce_bcast`` (the shard owner sums the ranks'
    slots in rank order — every rank gets bit-identical sums — and writes the result to every rank).

``torch.distributed`` is only the plumbing: it carries the 64-byte CUDA IPC handles at construction.  One process per GPU,
all GPUs on one NVSwitch domain (world <= 8), N a multiple of 4.
"""
from __future__ import annotations

import ctypes as C

import torch
import torch.distributed as dist

from . import _lib
from .parallel import GEOM_FIELDS, GEOM_FLOATS

vp, i32, u32, sz = C.c_void_p, C.c_int, C.c_uint, C.c_size_t
_lib.register("adb_peer_warmup", [])
_lib.register("adb_peer_alloc", [sz, C.POINTER(vp)])
_lib.register("adb_peer_free", [vp])
_lib.register("adb_peer_export", [vp, C.c_char_p])
_lib.register("adb_peer_import", [C.c_char_p, C.POINTER(vp)])
_lib.register("adb_peer_close", [vp])
_lib.register("adb_peer_signal", [C.POINTER(vp), i32, i32, i32, u32, vp])
_lib.register("adb_peer_wait", [vp, i32, i32, i32, u32, C.c_double, vp, vp])
_lib.register("adb_peer_push_rgb", [i32, vp, vp, C.POINTER(vp), i32, sz, vp, C.POINTER(vp), sz, vp])
_lib.register("adb_peer_bcast", [sz, vp, C.POINTER(vp), i32, sz, vp, C.POINTER(vp), sz, vp])
_lib.register("adb_peer_scatter", [sz, sz, vp, C.POINTER(vp), i32, i32, vp])
_lib.register("adb_peer_reduce_bcast", [sz, sz, vp, C.POINTER(vp), i32, i32, vp])

MAXW = 8
SLOT_X, SLOT_Y, SLOT_G = 0, 1, 2          # flag slots: scatter done, result written, colour row of local view c (SLOT_G + c)
N_SLOTS = 64


class _DeviceMemory:
    """Lets torch alias a raw device allocation (``torch.as_tensor`` understands ``__cuda_array_interface__``)."""

    def __init__(self, ptr: int, n_elems: int, typestr: str):
        self.__cuda_array_interface__ = {"shape": (n_elems,), "typestr": typestr, "data": (ptr, False), "version": 2}


def _align(n: int, a: int = 64) -> int:
    return (n + a - 1) // a * a


class PeerRegion:
    """Layout (in 4-byte words) of one rank's peer-visible region."""

    def __init__(self, n_gaussians: int, views_local: int, world: int):
        self.row = n_gaussians * 3                               # one view's colour-gradient row
        self.n4 = (n_gaussians * GEOM_FLOATS + 3) // 4           # float4 count of the geometry block
        self.per4 = (self.n4 + world - 1) // world               # shard size (float4)
        rows = views_local * world
        self.off_flags = 0
        self.off_cam = _align(N_SLOTS * MAXW)
        self.cam_stride = _align(rows * 3)
        self.off_g = self.off_cam + 2 * self.cam_stride
        self.g_stride = _align(rows * self.row)
        self.off_stage = self.off_g + 2 * self.g_stride
        self.off_y = self.off_stage + _align(world * self.per4 * 4)
        self.words = self.off_y + _align(world * self.per4 * 4)


class PeerExchange:
    """Drop-in for ``parallel.MultiViewExchange`` on CUDA (see module docstring).

    ``views_in``: where the geometry backward writes this rank's partial sums; ``views``: the reduced gradients (valid after
    ``wait_reduce``).  ``peers``: optional list of ``world`` base pointers of already-mapped regions (tests drive several
    "ranks" inside one process); by default the regions are exchanged through CUDA IPC over ``torch.distributed``."""

    fused_mask = True           # push_view() applies the SH-clamp mask itself

    def __init__(self, n_gaussians: int, views_local: int, device, group=None, rank: int | None = None,
                 world: int | None = None, base: int | None = None, peers: list[int] | None = None, timeout_s: float = 5.0):
        if n_gaussians % 4:
            raise _lib.ArtdecoB200Error("PeerExchange needs a Gaussian count that is a multiple of 4")
        self.n, self.views_local, self.group = n_gaussians, views_local, group
        self.dev = torch.device(device)
        self.world = world if world is not None else dist.get_world_size(group)
        self.rank = rank if rank is not None else dist.get_rank(group)
        if not 1 <= self.world <= MAXW or views_local > N_SLOTS - SLOT_G:
            raise _lib.ArtdecoB200Error(f"PeerExchange supports at most {MAXW} ranks")
        self.timeout_s = timeout_s
        L = self.layout = PeerRegion(n_gaussians, views_local, self.world)
        with torch.cuda.device(self.dev):
            _lib.require_cuda()
            _lib.call("adb_peer_warmup")
            self._owned = base is None
            self._imported = []
            self.base = base or 0
            if peers is None:
                peers = self._allocate_and_map()      # collective: every rank succeeds or every rank raises
            elif base is None:
                raise _lib.ArtdecoB200Error("PeerExchange: `peers` given without `base`")
            base = self.base
            self.peers = list(peers)
            self.comm = torch.cuda.Stream(device=self.dev)
            self.err = torch.zeros(1, dtype=torch.int32, device=self.dev)
        self._mem = _DeviceMemory(base, L.words, "<f4")
        region = torch.as_tensor(self._mem, device=self.dev)
        assert region.data_ptr() == base
        self.region = region
        self.flags_ptr = base + L.off_flags * 4
        # double-buffered (step parity) colour table and camera centres, view-major like MultiViewExchange.g_all
        self.g_all = [region[L.off_g + k * L.g_stride:][:views_local * self.world * L.row].view(views_local * self.world,
                                                                                                 n_gaussians, 3) for k in (0, 1)]
        self.campos_all = [region[L.off_cam + k * L.cam_stride:][:views_local * self.world * 3].view(-1, 3) for k in (0, 1)]
        self.stage_ptr = base + L.off_stage * 4
        y = region[L.off_y:][:L.n4 * 4]
        self.geom_in = torch.zeros(L.n4 * 4, dtype=torch.float32, device=self.dev)
        self.views, self.views_in = {}, {}
        o = 0
        for name, m in GEOM_FIELDS:
            for buf, d in ((y, self.views), (self.geom_in, self.views_in)):
                v = buf[o:o + n_gaussians * m]
                d[name] = v.view(n_gaussians, m) if m > 1 else v
            o += n_gaussians * m
        self.step_g = self.step_r = 0
        self._views_started = 0
        self._campos = None
        self._pushed = torch.cuda.Event()
        self.bytes_per_step = {"all_gather_recv": (self.world - 1) * views_local * n_gaussians * 12,
                               "all_reduce_payload": n_gaussians * GEOM_FLOATS * 4,
                               "dense_all_reduce_payload_replaced": n_gaussians * 59 * 4}

    # ---- setup ------------------------------------------------------------------------------------------------------
    def _allocate_and_map(self) -> list[int]:
        """Allocates this rank's region and maps everyone else's through CUDA IPC.  Every rank runs the same collectives whatever
        fails locally, and all of them raise together if any rank could not finish."""
        ok, why = 1, ""
        h = C.create_string_buffer(64)
        try:
            p = vp()
            _lib.call("adb_peer_alloc", self.layout.words * 4, C.byref(p))
            self.base = p.value
            _lib.call("adb_peer_export", vp(self.base), h)
        except Exception as e:  # noqa: BLE001
            ok, why = 0, repr(e)
        mine = torch.tensor(list(h.raw), dtype=torch.uint8, device=self.dev)
        table = torch.empty(self.world, 64, dtype=torch.uint8, device=self.dev)
        dist.all_gather_into_tensor(table, mine, group=self.group)
        table = table.cpu()
        peers = []
        for r in range(self.world):
            if r == self.rank:
                peers.append(self.base)
                continue
            p = vp()
            try:
                if ok:
                    _lib.call("adb_peer_import", bytes(table[r].tolist()), C.byref(p))
                    self._imported.append(p.value)
            except Exception as e:  # noqa: BLE001
                ok, why = 0, repr(e)
            peers.append(p.value or 0)
        torch.cuda.synchronize(self.dev)
        # doubles as the barrier: every region is zeroed and mapped everywhere before the first signal
        flag = torch.tensor([ok], dtype=torch.int32, device=self.dev)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=self.group)
        if not int(flag):
            self.close()
            raise _lib.ArtdecoB200Error(f"peer-memory exchange unavailable on this node ({why or 'another rank failed'})")
        return peers

    def _ptrs(self, off_words: int):
        return (vp * self.world)(*[p + off_words * 4 for p in self.peers])

    def close(self):
        """Unmaps the peers' regions and frees this rank's.  Collective: every rank must have finished its last step."""
        with torch.cuda.device(self.dev):
            torch.cuda.synchronize(self.dev)
            for p in self._imported:
                _lib.call("adb_peer_close", vp(p))
            self._imported = []
            if self._owned and self.base:
                self.region = self.g_all = self.campos_all = self.views = None
                _lib.call("adb_peer_free", vp(self.base))
                self.base = 0

    # ---- ordering ---------------------------------------------------------------------------------------------------
    def _signal(self, slot: int, value: int):
        _lib.call("adb_peer_signal", self._ptrs(self.layout.off_flags), self.world, slot, self.rank, value, _lib.stream())

    def _wait(self, slot_lo: int, n_slots: int, value: int):
        _lib.call("adb_peer_wait", vp(self.flags_ptr), self.world, slot_lo, n_slots, value, float(self.timeout_s),
                  _lib.ptr(self.err), _lib.stream())

    def check(self):
        """Host sync.  Raises if a wait timed out (a rank died or fell out of step)."""
        e = int(self.err)
        if e:
            raise _lib.ArtdecoB200Error(f"peer exchange: rank {self.rank} timed out waiting on flag slot {e - 1}")

    # ---- gather -----------------------------------------------------------------------------------------------------
    def _begin_view(self, campos):
        if self._views_started == 0:
            self.step_g += 1
        if campos is not None:
            self._campos = campos
        self._views_started += 1
        return self.step_g & 1

    def _push(self, c: int, launch):
        L = self.layout
        par = self.step_g & 1
        row = (c * self.world + self.rank)
        cur = torch.cuda.current_stream(self.dev)
        self.comm.wait_stream(cur)
        with torch.cuda.stream(self.comm):
            cam = self._campos[c] if self._campos is not None else None
            launch(self._ptrs(L.off_g + par * L.g_stride), row * L.row, cam,
                   self._ptrs(L.off_cam + par * L.cam_stride), row * 3)
            self._signal(SLOT_G + c, self.step_g)
            self._pushed.record(self.comm)

    def push_view(self, c: int, splats: torch.Tensor, v_splats: torch.Tensor, campos: torch.Tensor | None = None):
        """Local view c: mask the colour gradient (SH clamp) and write it into every rank's table.  ``campos [C_local,3]``
        with the first view of the step."""
        if tuple(splats.shape) != (self.n, 12) or tuple(v_splats.shape) != (self.n, 12) or not 0 <= c < self.views_local:
            raise ValueError(f"push_view: expected splats / v_splats of shape ({self.n}, 12) and 0 <= c < {self.views_local}")
        self._begin_view(campos)
        n = self.n
        self._push(c, lambda dst, off, cam, camp, camoff: _lib.call(
            "adb_peer_push_rgb", n, _lib.ptr(splats), _lib.ptr(v_splats), dst, self.world, off,
            _lib.ptr(cam) if cam is not None else None, camp, camoff, _lib.stream()))

    def start_gather_view(self, c: int, g_view: torch.Tensor, campos: torch.Tensor | None = None):
        """Same, for an already masked gradient row [N,3]."""
        assert g_view.shape == (self.n, 3)
        self._begin_view(campos)
        g_view = g_view.contiguous()
        g_view.record_stream(self.comm)
        self._push(c, lambda dst, off, cam, camp, camoff: _lib.call(
            "adb_peer_bcast", self.n * 3, _lib.ptr(g_view), dst, self.world, off,
            _lib.ptr(cam) if cam is not None else None, camp, camoff, _lib.stream()))

    def start_gather(self, g_rgb: torch.Tensor, campos: torch.Tensor):
        assert g_rgb.shape == (self.views_local, self.n, 3) and campos.shape == (self.views_local, 3)
        campos = campos.contiguous()
        for c in range(self.views_local):
            self.start_gather_view(c, g_rgb[c], campos if c == 0 else None)

    @property
    def gather_started(self) -> bool:
        return self._views_started > 0

    def wait_gather(self):
        """Returns (g_all [C_local*world, N, 3], campos_all [C_local*world, 3]), view-major (entry c*world + r = view c of rank r)."""
        par = self.step_g & 1
        torch.cuda.current_stream(self.dev).wait_event(self._pushed)
        self._wait(SLOT_G, self.views_local, self.step_g)
        self._views_started = 0
        return self.g_all[par], self.campos_all[par]

    # ---- reduce -----------------------------------------------------------------------------------------------------
    def start_reduce(self):
        """Sums ``views_in`` over the ranks into ``views`` (asynchronously, on the exchange's own stream)."""
        L = self.layout
        self.step_r += 1
        cur = torch.cuda.current_stream(self.dev)
        self.comm.wait_stream(cur)
        with torch.cuda.stream(self.comm):
            _lib.call("adb_peer_scatter", L.n4, L.per4, _lib.ptr(self.geom_in), self._ptrs(L.off_stage), self.world, self.rank,
                      _lib.stream())
            self._signal(SLOT_X, self.step_r)
            self._wait(SLOT_X, 1, self.step_r)
            _lib.call("adb_peer_reduce_bcast", L.n4, L.per4, vp(self.stage_ptr), self._ptrs(L.off_y), self.world, self.rank,
                      _lib.stream())
            self._signal(SLOT_Y, self.step_r)

    def wait_reduce(self):
        torch.cuda.current_stream(self.dev).wait_stream(self.comm)
        self._wait(SLOT_Y, 1, self.step_r)


def make_exchange(n_gaussians: int, views_local: int, device, group=None, kind: str | None = None):
    """The multi-GPU gradient exchange for ``multiview.MultiViewStep`` / ``rasterization(grad_exchange=)``.

    ``kind`` (default: ``$ADB_EXCHANGE``, else "nccl"):
      * "nccl" — ``parallel.MultiViewExchange``, the library collectives;
      * "peer" — ``PeerExchange``, this library's kernels over NVLink peer memory (falls back to "nccl", with a warning, when the
        ranks cannot map each other's memory).
    The peer exchange's stores from every SM can slow the backward kernels running beside it, and capping its grids
    (``ADB_PEER_CTAS=32``) trades that for slower copies; until the grid size is tuned on H100 the library collectives stay the
    default."""
    import os

    from .parallel import MultiViewExchange
    kind = kind or os.environ.get("ADB_EXCHANGE", "nccl")
    if kind not in ("nccl", "peer"):
        raise ValueError(f"exchange kind must be 'nccl' or 'peer', got {kind!r}")
    dev = torch.device(device)
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    if kind == "peer" and dev.type == "cuda" and 1 < world <= MAXW and n_gaussians % 4 == 0:
        try:
            return PeerExchange(n_gaussians, views_local, dev, group=group)      # raises on every rank or on none
        except _lib.ArtdecoB200Error as e:
            import warnings
            warnings.warn(f"{e}; using the NCCL exchange")
    return MultiViewExchange(n_gaussians, views_local, device, group=group)
