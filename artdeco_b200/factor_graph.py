"""The Backend's factor graph on the device: a drop-in ``FactorGraph`` for ``VSLAM/mast3r_slam/global_opt.py``'s, with the
methods ``Backend`` calls (``add_factors``, ``solve_GN_calib``, ``solve_GN_rays``) and the ``ii`` / ``jj`` attributes.

``frames`` is the reference's ``SharedKeyframes``, read through its stacked tensors (``T_WC [buf,1,8]``, ``X [buf,n,3]``,
``C [buf,n,1]``, ``N``, ``N_updates``, ``dataset_idx``, ``h``, ``w``, ``lock``), on the host or on this graph's device.

What runs differently from the reference (csrc/factor_graph.cu):
  * the edges live in a two-way table (edge e = rows 2e (i -> j) and 2e+1 (j -> i)) that grows by doubling, so the
    reference's eight ``torch.cat``'s per key frame and ``prep_two_way_edges``' copy per solve are gone: the first 2E rows
    are what the solve reads.  Edge order inside the solve changes nothing but rounding (its sums are atomics);
  * gating is three launches, with integer match counts; ``add_matches`` reads the device once, for the accepted flags;
  * the solve's point maps and confidences come from a device mirror indexed by key-frame id, refreshed only for key
    frames whose ``(dataset_idx, N_updates)`` changed since the last refresh, instead of copying every key frame of the
    graph to the device on every solve.  The poses are gathered and written back by one launch each;
  * the edge list is kept on the host as well (``ii_list`` / ``jj_list``), so the key-frame ranks the solve needs cost no
    ``torch.unique`` and, with device-resident frames, a solve reads nothing back from the device;
  * a match index outside ``[0, n)`` (the reference faults in the gather) is not read: its pixel is an invalid match and
    is counted in ``n_bad``, a device int32.
Quirks kept: ``C / N`` is evaluated as C times the fp32 reciprocal of N, as PyTorch does on CUDA for a Python-int divisor;
``match_frac`` is the fp32 count times the fp32 reciprocal of n; thresholds compare in fp32."""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib, gn
from ._lib import f32, i32, i64, vp
from .mast3r.wrappers import mast3r_match_symmetric

_lib.register("adb_fg_gate_workspace_bytes", [i32, i32, C.POINTER(C.c_size_t)])
_lib.register("adb_fg_gate", [i32, i32, i64, i64, vp, vp, vp, vp, vp, vp, vp, vp, vp, f32, f32, i32, vp, vp, vp, vp, vp, vp, vp,
                              vp, vp, C.c_size_t, vp])
_lib.register("adb_fg_mirror_refresh", [i32, i32, i32, i32, i32, vp, i32, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp])
_lib.register("adb_fg_pose_gather", [i32, i32, vp, vp, vp, vp])
_lib.register("adb_fg_pose_scatter", [i32, i32, i32, vp, vp, vp, vp])

RAYS, CALIB = 0, 1
_NEVER = -(2 ** 31)        # stamp of a mirror row never refreshed


def _upload(values, dev) -> torch.Tensor:
    """int64 host list -> device without blocking the host (pinned staging)."""
    return torch.tensor(values, dtype=torch.int64).pin_memory().to(dev, non_blocking=True)


class FactorGraph:
    def __init__(self, config, model, frames, K=None, device="cuda"):
        _lib.require_cuda()
        dev = torch.device(device)
        if dev.type != "cuda":
            raise ValueError("FactorGraph runs on a CUDA device")
        self.device = torch.device("cuda", dev.index if dev.index is not None else torch.cuda.current_device())
        self.model = model
        self.frames = frames
        self.config = config
        self.cfg = config["local_opt"]
        self.window_size = self.cfg["window_size"]
        self.K = K
        self._K = K.detach().to(self.device, torch.float32).reshape(3, 3).contiguous() if K is not None else None
        self.h, self.w = int(frames.h), int(frames.w)
        self.n = self.h * self.w
        if frames.X.device.type == "cuda" and frames.X.device != self.device:
            raise ValueError(f"frames live on {frames.X.device}, the graph on {self.device}")
        self.frames_on_device = frames.X.device.type == "cuda"
        for name, t, dt in (("T_WC", frames.T_WC, torch.float32), ("X", frames.X, torch.float32),
                            ("C", frames.C, torch.float32), ("N", frames.N, torch.int32),
                            ("N_updates", frames.N_updates, torch.int32), ("dataset_idx", frames.dataset_idx, torch.int32)):
            if t.dtype != dt or not t.is_contiguous():
                raise ValueError(f"frames.{name} must be a contiguous {dt} tensor")
        if frames.X.shape[1:] != (self.n, 3) or frames.C.numel() != frames.C.shape[0] * self.n:
            raise ValueError(f"frames.X must be [buf,{self.n},3] and frames.C [buf,{self.n},1]")
        self.n_bad = torch.zeros(1, dtype=torch.int32, device=self.device)
        self.last_accepted = self.last_counts = None
        # two-way edge table
        self.E = 0
        self._cap = 0
        self._edges: list[tuple[int, int]] = []
        self._rows_i = torch.empty(0, dtype=torch.int64, device=self.device)
        self._rows_j = torch.empty(0, dtype=torch.int64, device=self.device)
        self._idx = torch.empty(0, self.n, dtype=torch.int64, device=self.device)
        self._valid = torch.empty(0, self.n, dtype=torch.bool, device=self.device)
        self._Q = torch.empty(0, self.n, dtype=torch.float32, device=self.device)
        # key-frame mirror
        self._mode = None
        self._mir_rows = 0
        self._Xm = self._Cm = None
        self._seen = None            # device frames: two int32 [rows,2] stamp buffers, read one, write the other
        self._stamps = None          # host frames: the stamps, on the host

    # ---------------------------------------------------------------- edges
    @property
    def ii(self) -> torch.Tensor:
        return self._rows_i[0:2 * self.E:2]

    @property
    def jj(self) -> torch.Tensor:
        return self._rows_j[0:2 * self.E:2]

    @property
    def ii_list(self) -> list:
        """``ii.cpu().tolist()`` without reading the device."""
        return [e[0] for e in self._edges]

    @property
    def jj_list(self) -> list:
        return [e[1] for e in self._edges]

    def two_way_edges(self):
        """The solve's edge arrays, rows interleaved (2e: i -> j, 2e+1: j -> i): ``(ii, jj, idx_ii2jj, valid_match, Q)``,
        views of the table."""
        r = 2 * self.E
        return self._rows_i[:r], self._rows_j[:r], self._idx[:r], self._valid[:r], self._Q[:r]

    def _reserve(self, edges: int) -> None:
        if edges <= self._cap:
            return
        cap = max(edges, 2 * self._cap, 4)
        r, dev, n = 2 * self.E, self.device, self.n
        rows_i = torch.empty(2 * cap, dtype=torch.int64, device=dev)
        rows_j = torch.empty(2 * cap, dtype=torch.int64, device=dev)
        idx = torch.empty(2 * cap, n, dtype=torch.int64, device=dev)
        valid = torch.empty(2 * cap, n, dtype=torch.bool, device=dev)
        Q = torch.empty(2 * cap, n, dtype=torch.float32, device=dev)
        for new, old in ((rows_i, self._rows_i), (rows_j, self._rows_j), (idx, self._idx), (valid, self._valid),
                         (Q, self._Q)):
            new[:r].copy_(old[:r])
        self._rows_i, self._rows_j, self._idx, self._valid, self._Q = rows_i, rows_j, idx, valid, Q
        self._cap = cap

    def add_factors(self, ii, jj, min_match_frac, embeddings, is_reloc=False):
        """global_opt.py:40-110: match the candidate edges with MASt3R, then ``add_matches``."""
        feat_i = torch.cat([embeddings[idx][0] for idx in ii])
        feat_j = torch.cat([embeddings[idx][0] for idx in jj])
        pos_i = torch.cat([embeddings[idx][1] for idx in ii])
        pos_j = torch.cat([embeddings[idx][1] for idx in jj])
        shape = torch.tensor([[self.h, self.w]])
        matches = mast3r_match_symmetric(self.config, self.model, feat_i, pos_i, feat_j, pos_j, [shape] * len(ii),
                                         [shape] * len(jj))
        return self.add_matches(ii, jj, min_match_frac, *matches, is_reloc=is_reloc)

    @torch.no_grad()
    def add_matches(self, ii, jj, min_match_frac, idx_i2j, idx_j2i, valid_j, valid_i, Qii, Qjj, Qji, Qij, is_reloc=False):
        """Gate B candidate edges (i = ``ii[b]``, j = ``jj[b]``) on ``mast3r_match_symmetric``'s outputs and append the
        accepted ones.  Returns True when edges were added; False when none were, or when ``is_reloc`` and one edge
        failed (then nothing is added).  Reads the device once (the B accepted flags); ``last_counts`` keeps the
        per-edge ``(valid_j, valid_i)`` counts on the device."""
        ii, jj = [int(x) for x in ii], [int(x) for x in jj]
        B, n, dev = len(ii), self.n, self.device
        if B == 0 or len(jj) != B:
            raise ValueError("ii and jj must list the same, non-zero number of candidate edges")
        if min(ii + jj) < 0:
            raise ValueError("key-frame ids must be >= 0")

        def arg(name, t, dtype):
            if not isinstance(t, torch.Tensor) or t.dtype != dtype or t.numel() != B * n:
                raise ValueError(f"{name} must be a {dtype} tensor of B*n = {B}*{n} elements")
            if t.device != dev:
                raise ValueError(f"{name} is on {t.device}, expected {dev}")
            return t.detach().reshape(B, n).contiguous()

        a = [arg("idx_i2j", idx_i2j, torch.int64), arg("idx_j2i", idx_j2i, torch.int64),
             arg("valid_j", valid_j, torch.bool), arg("valid_i", valid_i, torch.bool)]
        a += [arg(k, t, torch.float32) for k, t in (("Qii", Qii), ("Qjj", Qjj), ("Qji", Qji), ("Qij", Qij))]
        nb = C.c_size_t(0)
        _lib.call("adb_fg_gate_workspace_bytes", B, n, C.byref(nb))
        self._reserve(self.E + B)
        cand = _upload([v for e in zip(ii, jj) for v in e], dev)
        ws = torch.empty(nb.value, dtype=torch.uint8, device=dev)
        accepted = torch.empty(B, dtype=torch.int32, device=dev)
        counts = torch.empty(B, 2, dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            _lib.call("adb_fg_gate", B, n, self.E, self._cap, _lib.ptr(cand), *[_lib.ptr(t) for t in a],
                      float(self.cfg["Q_conf"]), float(min_match_frac), int(bool(is_reloc)), _lib.ptr(self._rows_i),
                      _lib.ptr(self._rows_j), _lib.ptr(self._idx), _lib.ptr(self._valid), _lib.ptr(self._Q),
                      _lib.ptr(accepted), _lib.ptr(counts), _lib.ptr(self.n_bad), _lib.ptr(ws), ws.numel(), _lib.stream())
        flags = accepted.cpu().tolist()
        self.last_accepted, self.last_counts = accepted, counts
        new = [(ii[b], jj[b]) for b in range(B) if flags[b]]
        self._edges += new
        self.E += len(new)
        return len(new) > 0

    # ---------------------------------------------------------------- key-frame mirror
    def _grow_mirror(self, rows: int) -> None:
        if rows <= self._mir_rows:
            return
        cap = max(rows, 2 * self._mir_rows)
        old = self._mir_rows
        Xm = torch.empty(cap, self.n, 3, dtype=torch.float32, device=self.device)
        Cm = torch.empty(cap, self.n, dtype=torch.float32, device=self.device)
        if old:
            Xm[:old].copy_(self._Xm[:old])
            Cm[:old].copy_(self._Cm[:old])
        self._Xm, self._Cm = Xm, Cm
        if self.frames_on_device:
            seen = [torch.full((cap, 2), _NEVER, dtype=torch.int32, device=self.device) for _ in range(2)]
            if old:
                for s, o in zip(seen, self._seen):
                    s[:old].copy_(o[:old])
            self._seen = seen
        else:
            stamps = torch.full((cap, 2), _NEVER, dtype=torch.int32)
            if old:
                stamps[:old] = self._stamps[:old]
            self._stamps = stamps
        self._mir_rows = cap

    def refresh_mirror(self, mode: int, n_ids: int) -> None:
        """Mirror rows ``0..n_ids-1``: the key frames' points (on their rays in calib mode) and average confidences."""
        if mode != self._mode:          # the rows of the other mode are no use
            self._mir_rows, self._Xm, self._Cm, self._seen, self._stamps = 0, None, None, None, None
            self._mode = mode
        self._grow_mirror(n_ids)
        f, dev = self.frames, self.device
        Kp = _lib.ptr(self._K) if mode == CALIB else None
        if mode == CALIB and self._K is None:
            raise ValueError("solve_GN_calib needs the intrinsics K")
        if self.frames_on_device:
            seen, seen_next = self._seen
            with f.lock, torch.cuda.device(dev):
                _lib.call("adb_fg_mirror_refresh", mode, n_ids, self.h, self.w, self._mir_rows, None, 0, _lib.ptr(f.X),
                          _lib.ptr(f.C), _lib.ptr(f.N), _lib.ptr(f.dataset_idx), _lib.ptr(f.N_updates), _lib.ptr(seen),
                          _lib.ptr(seen_next), Kp, _lib.ptr(self._Xm), _lib.ptr(self._Cm), _lib.stream())
            self._seen = [seen_next, seen]
            return
        with f.lock:
            now = torch.stack([f.dataset_idx[:n_ids], f.N_updates[:n_ids]], 1)
            changed = (now != self._stamps[:n_ids]).any(1).nonzero()[:, 0]
            R = int(changed.numel())
            if R == 0:
                return
            X = torch.empty(R, self.n, 3, dtype=torch.float32, pin_memory=True)
            Cc = torch.empty(R, self.n, 1, dtype=torch.float32, pin_memory=True)
            torch.index_select(f.X, 0, changed, out=X)
            torch.index_select(f.C, 0, changed, out=Cc)
            N = f.N.index_select(0, changed).pin_memory()
            self._stamps[changed] = now[changed]
        ids = changed.pin_memory().to(dev, non_blocking=True)
        X, Cc, N = (t.to(dev, non_blocking=True) for t in (X, Cc, N))
        with torch.cuda.device(dev):
            _lib.call("adb_fg_mirror_refresh", mode, R, self.h, self.w, self._mir_rows, _lib.ptr(ids), 1, _lib.ptr(X),
                      _lib.ptr(Cc), _lib.ptr(N), None, None, None, None, Kp, _lib.ptr(self._Xm), _lib.ptr(self._Cm),
                      _lib.stream())

    def mirror(self):
        """``(Xm [rows,n,3], Cm [rows,n])`` as the last refresh left them."""
        return self._Xm, self._Cm

    # ---------------------------------------------------------------- solve
    def _solve(self, mode: int) -> None:
        cfg, f, dev = self.cfg, self.frames, self.device
        pin = int(cfg["pin"])
        unique = sorted({k for e in self._edges for k in e})
        U = len(unique)
        if U <= pin:
            return
        n_ids = unique[-1] + 1
        dense = n_ids == U            # the graph names key frames 0..U-1: ranks are ids
        self.refresh_mirror(mode, n_ids)
        ids = None if dense else _upload(unique, dev)
        poses = torch.empty(U, 8, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            if self.frames_on_device:
                with f.lock:
                    _lib.call("adb_fg_pose_gather", U, int(f.T_WC.shape[0]), _lib.ptr(ids), _lib.ptr(f.T_WC),
                              _lib.ptr(poses), _lib.stream())
            else:
                with f.lock:
                    T = f.T_WC.reshape(-1, 8).index_select(0, torch.tensor(unique)).pin_memory()
                T = T.to(dev, non_blocking=True)
                _lib.call("adb_fg_pose_gather", U, U, None, _lib.ptr(T), _lib.ptr(poses), _lib.stream())
        ii, jj, idx, valid, Q = self.two_way_edges()
        Xs, Cs = self._Xm[:U], self._Cm[:U]
        if not dense:
            rank = {k: r for r, k in enumerate(unique)}
            ii = _upload([rank[k] for e in self._edges for k in e], dev)
            jj = _upload([rank[k] for e in self._edges for k in e[::-1]], dev)
            Xs, Cs = self._Xm.index_select(0, ids), self._Cm.index_select(0, ids)
        common = (cfg["C_conf"], cfg["Q_conf"], cfg["max_iters"], cfg["delta_norm"])
        if mode == CALIB:
            gn.solve_positions(1, poses, Xs, Cs, self._K, ii, jj, idx, valid, Q, self.h, self.w, cfg["pixel_border"],
                               cfg["depth_eps"], cfg["sigma_pixel"], cfg["sigma_depth"], *common)
        else:
            gn.solve_positions(0, poses, Xs, Cs, None, ii, jj, idx, valid, Q, 0, 0, 0, 0.0, cfg["sigma_ray"],
                               cfg["sigma_dist"], *common)
        # update_T_WCs(T_WCs[pin:], unique[pin:])
        if self.frames_on_device:
            with f.lock, torch.cuda.device(dev):
                _lib.call("adb_fg_pose_scatter", U, pin, int(f.T_WC.shape[0]), _lib.ptr(ids), _lib.ptr(poses),
                          _lib.ptr(f.T_WC), _lib.stream())
        else:
            out = poses[pin:].cpu()
            with f.lock:
                f.T_WC.view(-1, 8)[torch.tensor(unique[pin:])] = out

    @torch.no_grad()
    def solve_GN_calib(self):
        """global_opt.py:174-220."""
        self._solve(CALIB)

    @torch.no_grad()
    def solve_GN_rays(self):
        """global_opt.py:138-172."""
        self._solve(RAYS)
