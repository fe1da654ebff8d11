"""TEST INFRASTRUCTURE ONLY.  The map update that run_system.py runs on every SLAM key frame, restated op for op in PyTorch:
the mapper key-frame pose loop (run_system.py:194-226, with Keyframe.get_Rt / set_Rt of Reconstruct/scene/keyframe.py and
sixD2mtx of Reconstruct/utils.py:223-229), SceneModel.rigid_transform_gs (Reconstruct/scene/scene_models/h3dgsv3.py:955-966)
and update_gaussians (Reconstruct/utils.py:28-60).  Runs on the CPU or the device.

pypose is the ``track_ref`` stand-in on [8] tensors (an SE3 is an [8] tensor with s = 1); kornia's
``quaternion_to_rotation_matrix`` and ``rotation_matrix_to_quaternion`` are restated below (``quat2mat``, ``mat2quat``).
tests/golden/make_reanchor_golden.py pins this module to the reference's own statements; parity of the stand-ins with
pypose and kornia themselves is unpinned (neither is vendored or installable)."""
import torch

from oracle import track_ref as pp
from oracle.mapper_loss_ref import sixD2mtx

MAT2QUAT_EPS = 1e-8


# ---- kornia.geometry.conversions ----
def quat2mat(q):
    """quaternion_to_rotation_matrix: q [...,4] wxyz, normalised with F.normalize(eps=1e-12) -> [...,3,3]."""
    q = q / q.norm(p=2, dim=-1, keepdim=True).clamp_min(1e-12)
    w, x, y, z = torch.chunk(q, chunks=4, dim=-1)
    tx, ty, tz = 2.0 * x, 2.0 * y, 2.0 * z
    twx, twy, twz = tx * w, ty * w, tz * w
    txx, txy, txz = tx * x, ty * x, tz * x
    tyy, tyz, tzz = ty * y, tz * y, tz * z
    one = torch.tensor(1.0, dtype=q.dtype, device=q.device)
    m = torch.stack((one - (tyy + tzz), txy - twz, txz + twy,
                     txy + twz, one - (txx + tzz), tyz - twx,
                     txz - twy, tyz + twx, one - (txx + tyy)), dim=-1)
    return m.reshape(*q.shape[:-1], 3, 3)


def _safe_div(num, den):
    return num / torch.clamp(den, min=torch.finfo(num.dtype).tiny)


def mat2quat(m, eps=MAT2QUAT_EPS):
    """rotation_matrix_to_quaternion: m [...,3,3] -> q [...,4] wxyz; all four branches evaluated, chosen by torch.where."""
    m00, m01, m02, m10, m11, m12, m20, m21, m22 = torch.chunk(m.reshape(*m.shape[:-2], 9), chunks=9, dim=-1)
    trace = m00 + m11 + m22

    sq = torch.sqrt(trace + 1.0 + eps) * 2.0
    q0 = torch.cat((0.25 * sq, _safe_div(m21 - m12, sq), _safe_div(m02 - m20, sq), _safe_div(m10 - m01, sq)), dim=-1)
    sq = torch.sqrt(1.0 + m00 - m11 - m22 + eps) * 2.0
    q1 = torch.cat((_safe_div(m21 - m12, sq), 0.25 * sq, _safe_div(m01 + m10, sq), _safe_div(m02 + m20, sq)), dim=-1)
    sq = torch.sqrt(1.0 + m11 - m00 - m22 + eps) * 2.0
    q2 = torch.cat((_safe_div(m02 - m20, sq), _safe_div(m01 + m10, sq), 0.25 * sq, _safe_div(m12 + m21, sq)), dim=-1)
    sq = torch.sqrt(1.0 + m22 - m00 - m11 + eps) * 2.0
    q3 = torch.cat((_safe_div(m10 - m01, sq), _safe_div(m02 + m20, sq), _safe_div(m12 + m21, sq), 0.25 * sq), dim=-1)

    where_2 = torch.where(m11 > m22, q2, q3)
    where_1 = torch.where((m00 > m11) & (m00 > m22), q1, where_2)
    return torch.where(trace > 0.0, q0, where_1)


def mat2quat_branch(m):
    """(branch [...] in 0..3 as mat2quat picks it, the smallest |difference| that decided it)."""
    d = m.reshape(*m.shape[:-2], 9)
    m00, m11, m22 = d[..., 0], d[..., 4], d[..., 8]
    trace = m00 + m11 + m22
    b = torch.where(trace > 0, 0, torch.where((m00 > m11) & (m00 > m22), 1, torch.where(m11 > m22, 2, 3)))
    diag = torch.stack([(m00 - m11).abs(), (m00 - m22).abs(), (m11 - m22).abs()], -1).amin(-1)
    margin = torch.where(trace > 0, trace.abs(), torch.minimum(trace.abs(), diag))
    return b, margin


# ---- the reference's statements ----
def SE3(x7):
    return torch.cat([x7, torch.ones(1, dtype=x7.dtype, device=x7.device)])


def get_Rt(r, t):
    """Keyframe.get_Rt: [4,4] world-to-camera from the 6-D rotation r [3,2] and t [3]."""
    Rt = torch.eye(4, dtype=r.dtype, device=r.device)
    Rt[:3, :3] = sixD2mtx(r)
    Rt[:3, 3] = t
    return Rt


def keyframe_poses(rW2C, tW2C, slam_T_WC, last_keyframe_index, is_slam_keyframe, T_CkCf):
    """run_system.py:198-226 for every mapper key frame, in order.  Returns the updated (rW2C, tW2C) and old_c2ws,
    new_c2ws [K,4,4], cam_centres, approx_centres [K,3].  Every last_keyframe_index must be in range (the reference
    indexes the Backend's list with it)."""
    rW2C, tW2C = rW2C.clone(), tW2C.clone()
    K = rW2C.shape[0]
    dt, dev = rW2C.dtype, rW2C.device
    old_c2ws = torch.zeros(K, 4, 4, dtype=dt, device=dev)
    new_c2ws = torch.zeros(K, 4, 4, dtype=dt, device=dev)
    cam_centres = torch.zeros(K, 3, dtype=dt, device=dev)
    approx_centres = torch.zeros(K, 3, dtype=dt, device=dev)
    for k in range(K):
        T_WC = slam_T_WC[int(last_keyframe_index[k])]
        if bool(is_slam_keyframe[k]):
            T_WCk = pp.quat2unit(SE3(T_WC[:7]))
            T_WCf = T_WCk
        else:
            T_WCk = T_WC
            T_WCf = pp.mul(T_WCk, T_CkCf[k])
            T_WCf = SE3(pp.quat2unit(T_WCf)[:7])
        new_Rt = pp.matrix(pp.inv(T_WCf))
        old_Rt = get_Rt(rW2C[k], tW2C[k])
        # set_Rt
        rW2C[k] = new_Rt[:3, :2]
        tW2C[k] = new_Rt[:3, 3]
        approx_centres[k] = -new_Rt[:3, :3].T @ new_Rt[:3, 3]
        view_matrix = get_Rt(rW2C[k], tW2C[k]).transpose(0, 1)
        cam_centres[k] = view_matrix.inverse()[3, :3]
        old_c2ws[k] = torch.linalg.inv(old_Rt)
        new_c2ws[k] = torch.linalg.inv(new_Rt)
    return dict(rW2C=rW2C, tW2C=tW2C, old_c2ws=old_c2ws, new_c2ws=new_c2ws, cam_centres=cam_centres,
                approx_centres=approx_centres)


def update_gaussians(old_c2ws, new_c2ws, gaussians_positions, gaussians_quaternions):
    """Reconstruct/utils.py:28-60: per-row [N,4,4] tables."""
    delta_T = torch.bmm(new_c2ws, torch.inverse(old_c2ws))
    R = delta_T[:, :3, :3]
    t = delta_T[:, :3, 3]
    rot_mats_orig = quat2mat(gaussians_quaternions)
    new_positions = torch.einsum('bij,bj->bi', R, gaussians_positions) + t
    new_rot_mats = torch.bmm(R, rot_mats_orig)
    return new_positions, mat2quat(new_rot_mats), new_rot_mats


def rigid_transform_gs(ids, xyz, rotation, old_c2ws, new_c2ws):
    """SceneModel.rigid_transform_gs on (id [N,1], xyz [N,3], rotation [N,4]) -> (xyz, rotation, the rotated matrices)."""
    old = old_c2ws[ids.squeeze(-1)]
    new = new_c2ws[ids.squeeze(-1)]
    return update_gaussians(old, new, xyz, rotation)
