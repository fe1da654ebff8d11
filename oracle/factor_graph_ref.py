"""TEST INFRASTRUCTURE ONLY.  Oracle for the factor graph (csrc/factor_graph.cu, artdeco_b200/factor_graph.py):
``FactorGraph`` (VSLAM/mast3r_slam/global_opt.py) restated in PyTorch on any device, after matching (``add_matches`` takes
``mast3r_match_symmetric``'s outputs), with ``oracle/track_ref.py``'s pypose stand-in, ``constrain_points_to_ray`` and
``quat2unit``.  The solve goes to ``backend`` (an object with ``gauss_newton_rays`` / ``gauss_newton_calib`` taking the
reference's positional arguments); ``GnRefBackend`` runs ``oracle/gn_ref.py``'s.

``Keyframes`` is a stand-in for the reference's ``SharedKeyframes`` (VSLAM/SharedKeyframes.py) with the stacked tensors
the factor graph reads, a ``threading.RLock`` for the manager's lock, and ``update_pointmap`` (ImageFrame.py:35-46)."""
import threading

import torch

from oracle import gn_ref, track_ref


class Frame:
    """What ``FactorGraph`` reads of an ``ImageFrame``."""

    def __init__(self, img, T_WC, X_canon, C, N):
        self.img, self.T_WC, self.X_canon, self.C, self.N = img, T_WC, X_canon, C, N

    def to(self, device):
        return Frame(self.img.to(device), self.T_WC.to(device), self.X_canon.to(device), self.C.to(device), self.N)

    def get_average_conf(self):
        return self.C / self.N


class Keyframes:
    def __init__(self, h, w, buffer=16, device="cpu"):
        self.h, self.w, self.buffer, self.device = h, w, buffer, device
        self.lock = threading.RLock()
        self.n_size = 0
        n = h * w
        self.dataset_idx = torch.zeros(buffer, dtype=torch.int32, device=device)
        self.T_WC = torch.zeros(buffer, 1, 8, device=device)
        self.T_WC[:, 0, 6:8] = 1.0
        self.X = torch.zeros(buffer, n, 3, device=device)
        self.C = torch.zeros(buffer, n, 1, device=device)
        self.N = torch.zeros(buffer, dtype=torch.int32, device=device)
        self.N_updates = torch.zeros(buffer, dtype=torch.int32, device=device)

    def __len__(self):
        return self.n_size

    def __getitem__(self, idx):
        idx = int(idx)
        return Frame(torch.zeros(3, self.h, self.w, device=self.device), self.T_WC[idx].clone(), self.X[idx], self.C[idx],
                     int(self.N[idx]))

    def append(self, dataset_idx, T_WC, X, C, N=1, N_updates=1):
        k = self.n_size
        self.dataset_idx[k] = int(dataset_idx)
        self.T_WC[k, 0] = T_WC.to(self.device)
        self.X[k] = X.to(self.device)
        self.C[k] = C.reshape(-1, 1).to(self.device)
        self.N[k], self.N_updates[k] = int(N), int(N_updates)
        self.n_size = k + 1
        return k

    def pop_last(self):
        self.n_size -= 1

    def update_pointmap(self, idx, X, C):
        """ImageFrame.update_pointmap on a stored key frame (N > 0)."""
        Cs = self.C[idx]
        C = C.reshape(-1, 1).to(self.device)
        self.X[idx] = ((Cs * self.X[idx]) + (C * X.to(self.device))) / (Cs + C)
        self.C[idx] = Cs + C
        self.N[idx] += 1
        self.N_updates[idx] += 1

    def update_T_WCs(self, T_WCs, idx):
        self.T_WC[idx] = T_WCs.to(self.device)

    def to(self, device):
        out = Keyframes(self.h, self.w, self.buffer, device)
        for k in ("dataset_idx", "T_WC", "X", "C", "N", "N_updates"):
            setattr(out, k, getattr(self, k).to(device).clone())
        out.n_size = self.n_size
        return out


class GnRefBackend:
    """``mast3r_slam_backends`` through oracle/gn_ref.py."""

    @staticmethod
    def gauss_newton_rays(Twc, Xs, Cs, ii, jj, idx, valid, Q, sigma_ray, sigma_dist, C_thresh, Q_thresh, max_iter, delta):
        gn_ref.gauss_newton("rays", Twc, Xs, Cs, ii, jj, idx, valid, Q, sigma_ray, sigma_dist, C_thresh, Q_thresh, max_iter,
                            delta)

    @staticmethod
    def gauss_newton_calib(Twc, Xs, Cs, K, ii, jj, idx, valid, Q, height, width, pixel_border, z_eps, sigma_pixel,
                           sigma_depth, C_thresh, Q_thresh, max_iter, delta):
        gn_ref.gauss_newton("calib", Twc, Xs, Cs, ii, jj, idx, valid, Q, sigma_pixel, sigma_depth, C_thresh, Q_thresh,
                            max_iter, delta, K=K, height=height, width=width, pixel_border=pixel_border, z_eps=z_eps)


class FactorGraphRef:
    def __init__(self, config, frames, K=None, device="cpu", backend=GnRefBackend):
        self.frames, self.device, self.cfg, self.K, self.backend = frames, device, config["local_opt"], K, backend
        self.ii = torch.as_tensor([], dtype=torch.long, device=device)
        self.jj = torch.as_tensor([], dtype=torch.long, device=device)
        self.idx_ii2jj = torch.as_tensor([], dtype=torch.long, device=device)
        self.idx_jj2ii = torch.as_tensor([], dtype=torch.long, device=device)
        self.valid_match_j = torch.as_tensor([], dtype=torch.bool, device=device)
        self.valid_match_i = torch.as_tensor([], dtype=torch.bool, device=device)
        self.Q_ii2jj = torch.as_tensor([], dtype=torch.float32, device=device)
        self.Q_jj2ii = torch.as_tensor([], dtype=torch.float32, device=device)
        self.last_counts = None

    def add_matches(self, ii, jj, min_match_frac, idx_i2j, idx_j2i, valid_match_j, valid_match_i, Qii, Qjj, Qji, Qij,
                    is_reloc=False):
        """global_opt.py:65-110.  ``last_counts`` [B,2] = (valid_j, valid_i) counts."""
        b = torch.arange(idx_i2j.shape[0], device=idx_i2j.device)[:, None].repeat(1, idx_i2j.shape[1])
        Qj = torch.sqrt(Qii[b, idx_i2j] * Qji)
        Qi = torch.sqrt(Qjj[b, idx_j2i] * Qij)
        valid_j = valid_match_j & (Qj > self.cfg["Q_conf"])
        valid_i = valid_match_i & (Qi > self.cfg["Q_conf"])
        nj = valid_j.shape[1] * valid_j.shape[2]
        ni = valid_i.shape[1] * valid_i.shape[2]
        self.last_counts = torch.stack([valid_j.sum(dim=(1, 2)), valid_i.sum(dim=(1, 2))], 1)
        match_frac_j = valid_j.sum(dim=(1, 2)) / nj
        match_frac_i = valid_i.sum(dim=(1, 2)) / ni
        ii_t = torch.as_tensor(ii, device=self.device)
        jj_t = torch.as_tensor(jj, device=self.device)
        invalid = torch.minimum(match_frac_j, match_frac_i) < min_match_frac
        invalid = (~(ii_t == (jj_t - 1))) & invalid
        if invalid.any() and is_reloc:
            return False
        ok = ~invalid
        self.ii = torch.cat([self.ii, ii_t[ok]])
        self.jj = torch.cat([self.jj, jj_t[ok]])
        self.idx_ii2jj = torch.cat([self.idx_ii2jj, idx_i2j[ok]])
        self.idx_jj2ii = torch.cat([self.idx_jj2ii, idx_j2i[ok]])
        self.valid_match_j = torch.cat([self.valid_match_j, valid_match_j[ok]])
        self.valid_match_i = torch.cat([self.valid_match_i, valid_match_i[ok]])
        self.Q_ii2jj = torch.cat([self.Q_ii2jj, Qj[ok]])
        self.Q_jj2ii = torch.cat([self.Q_jj2ii, Qi[ok]])
        return bool(ok.sum() > 0)

    def get_unique_kf_idx(self):
        return torch.unique(torch.cat([self.ii, self.jj]), sorted=True)

    def get_poses_points(self, unique_kf_idx):
        kfs = [self.frames[idx].to(self.device) for idx in unique_kf_idx]
        Xs = torch.stack([kf.X_canon for kf in kfs])
        T_WCs = track_ref.quat2unit(torch.stack([kf.T_WC for kf in kfs]))
        Cs = torch.stack([kf.get_average_conf() for kf in kfs])
        return Xs, T_WCs, Cs

    def prep_two_way_edges(self):
        return (torch.cat((self.ii, self.jj)), torch.cat((self.jj, self.ii)), torch.cat((self.idx_ii2jj, self.idx_jj2ii)),
                torch.cat((self.valid_match_j, self.valid_match_i)), torch.cat((self.Q_ii2jj, self.Q_jj2ii)))

    def solve_inputs(self, calib):
        """``(unique, Xs, T_WCs [U,1,8], Cs)`` as the solve receives them (Xs on their rays in calib mode)."""
        unique = self.get_unique_kf_idx()
        Xs, T_WCs, Cs = self.get_poses_points(unique)
        if calib:
            n = Xs.shape[1]
            Xs = torch.stack([track_ref.constrain_points_to_ray(Xs[k], self.frames.h, self.frames.w, self.K.to(Xs.device))
                              for k in range(Xs.shape[0])]) if n else Xs
        return unique, Xs, T_WCs, Cs

    def _solve(self, calib):
        pin = self.cfg["pin"]
        if self.get_unique_kf_idx().numel() <= pin:
            return
        unique, Xs, T_WCs, Cs = self.solve_inputs(calib)
        ii, jj, idx, valid, Q = self.prep_two_way_edges()
        c = self.cfg
        pose_data = T_WCs[:, 0, :]
        if calib:
            self.backend.gauss_newton_calib(pose_data, Xs, Cs, self.K, ii, jj, idx, valid, Q, self.frames.h, self.frames.w,
                                            c["pixel_border"], c["depth_eps"], c["sigma_pixel"], c["sigma_depth"],
                                            c["C_conf"], c["Q_conf"], c["max_iters"], c["delta_norm"])
        else:
            self.backend.gauss_newton_rays(pose_data, Xs, Cs, ii, jj, idx, valid, Q, c["sigma_ray"], c["sigma_dist"],
                                           c["C_conf"], c["Q_conf"], c["max_iters"], c["delta_norm"])
        self.frames.update_T_WCs(T_WCs[pin:], unique[pin:].to(self.frames.T_WC.device))

    def solve_GN_calib(self):
        self._solve(True)

    def solve_GN_rays(self):
        self._solve(False)
