"""TEST INFRASTRUCTURE ONLY.  ``SceneModel.add_new_gaussians`` oracle (/root/reference Reconstruct/scene/scene_models/
h3dgsv3.py:766-940 with the helpers of Reconstruct/utils.py:93-108, :119-130, :188-216 and the disc / uv block of __init__,
:209-225) restated op for op in PyTorch, on the CPU or on CUDA.  Substitutions, all at the object boundary:
  * the scene is a dict of the reference's ``gaussian_params`` values (raw opacity / scaling) and the optimiser's
    ``add_and_prune`` is ``add_and_prune`` below (cat(t[mask], ext) per key; global_feat is appended unmasked);
  * the render is a callable ``render(cls_id) -> [3,H,W]`` raw RGB (``render_from_id`` applies the exposure here);
  * ``update_voxel`` defaults to ``oracle.voxel_ref.update_voxel`` (run on the CPU) and may be replaced;
  * ``weed_out_gaussians`` takes the key frames' centres ``keyframe.get_Rt().T.inverse()[3, :3]``.
PARITY: pinned against the reference's own code by tests/golden/make_densify_golden.py (tests/golden/densify_small.pt)."""
import numpy as np
import torch
import torch.nn.functional as F

from . import voxel_ref

LODS = (1, 2, 4, 8)
C0 = 0.28209479177387814


def disc_kernel(device="cpu"):
    radius = 3
    k = torch.zeros(1, 1, 2 * radius + 1, 2 * radius + 1, device=device)
    y, x = torch.meshgrid(torch.arange(-radius, radius + 1), torch.arange(-radius, radius + 1), indexing="ij")
    k[0, 0, (torch.sqrt(x.to(device) ** 2 + y.to(device) ** 2) <= radius + 0.5)] = 1
    return k / k.sum()


def uvs(width, height, lod, device="cpu"):
    return torch.stack(torch.meshgrid(torch.arange(0, width // lod), torch.arange(0, height // lod), indexing="xy"),
                       dim=-1).float().to(device)


def get_lapla_norm(img, kernel):
    lap = torch.tensor([[0, 1, 0], [1, -4, 1], [0, 1, 0]], device=img.device, dtype=torch.float32)[None, None]
    lap = lap.repeat(1, img.shape[0], 1, 1)
    laplacian = F.conv2d(img[None], lap, padding="same")
    n = torch.linalg.vector_norm(laplacian, ord=1, dim=1, keepdim=True)
    n[..., :, 0] = 0
    n[..., :, -1] = 0
    n[..., 0, :] = 0
    n[..., -1, :] = 0
    return F.conv2d(n, kernel, padding="same")[0, 0].clamp(0, 1)


def sample(map, uv, width, height):
    s = uv.clone()
    s[..., 0] = s[..., 0] * (2.0 / (width - 1)) - 1.0
    s[..., 1] = s[..., 1] * (2.0 / (height - 1)) - 1.0
    return F.grid_sample(map, s, mode="bilinear", align_corners=True)


def depth2points(uv, depth, f, centre):
    return depth * torch.cat([(uv[..., :2] - centre) / f, torch.ones_like(uv[..., 0:1])], dim=-1)


def inverse_sigmoid(x):
    return torch.log(x / (1 - x))


def exposed(raw, exposure):
    """``render_from_id``'s exposure and clamp (h3dgsv3.py:611-614)."""
    _, H, W = raw.shape
    out = exposure[:3, :3] @ raw.reshape(3, -1) + exposure[:3, 3, None]
    return out.clamp(0, 1).view(3, H, W)


def depth_threshold(point_map):
    """``min(1e-2, torch.quantile(point_map[:, 2], 0.02).item())`` (a NaN quantile gives 1e-2)."""
    return min(1e-2, torch.quantile(point_map[:, 2], 0.02).item())


def prune_mask(params, approx_centre, f, width):
    xyz = params["xyz"]
    if xyz.shape[0] == 0:
        return torch.ones(0, device=xyz.device, dtype=torch.bool)
    valid = torch.sigmoid(params["opacity"])[:, 0] > 0.05
    dist = torch.linalg.vector_norm(xyz - approx_centre[None], dim=-1)
    screen = f * torch.exp(params["scaling"]).max(dim=-1)[0] / dist
    valid *= screen < 0.5 * width
    return valid


def sample_lod(image, render, point_map, conf, R, t, approx_centre, exposure, *, lod, f, init_proba_scaler, gs_add_ratio,
               uniforms, qmin, disc=None):
    """Lines 779-891 of one LoD up to the voxel step; ``render`` is the raw RGB (None for an empty scene) and ``uniforms`` the
    draw.  Returns the maps and the rows, like ``artdeco_b200.densify.sample_lod``."""
    dev = image.device
    H, W = image.shape[-2:]
    disc = disc_kernel(dev) if disc is None else disc
    cur_h, cur_w = H // lod, W // lod
    img = F.interpolate(F.avg_pool2d(image, 2)[None], (cur_h, cur_w), mode="bilinear", align_corners=True)[0]
    init_proba = get_lapla_norm(img, disc)
    penalty = 0
    if render is not None:
        r = F.interpolate(exposed(render, exposure)[None], (cur_h, cur_w), mode="bilinear", align_corners=True)[0]
        penalty = get_lapla_norm(r, disc)
    init_proba *= init_proba_scaler
    penalty *= init_proba_scaler
    sample_mask = uniforms < (init_proba - penalty) * gs_add_ratio
    sampled = sample_mask.clone()
    uv = uvs(W, H, lod, dev)[sample_mask]
    depths = sample(point_map[:, 2:], uv[None, None], W // lod, H // lod)[0, 0, 0]
    confs = sample(conf, uv[None, None], W // lod, H // lod)[0, 0, 0]
    valid_mask = (confs >= 0) * (depths > qmin)
    sample_mask[sample_mask.clone()] = valid_mask
    valid = torch.zeros_like(sampled)
    valid[sampled] = valid_mask
    uv, depths, confs = uv[valid_mask], depths[valid_mask], confs[valid_mask]
    centre = torch.tensor([(W - 1) / 2, (H - 1) / 2], device=dev) / lod
    pts = depth2points(uv, depths.unsqueeze(-1), f / lod, centre)
    pts = (pts - t) @ R
    f_dc = (img[:, sample_mask].permute(1, 0).unsqueeze(1) - 0.5) / C0
    scales = 1 / torch.sqrt(init_proba[sample_mask])
    scales.clamp_(1, W / 10)
    scales.mul_(1 / f)
    scales *= torch.linalg.vector_norm(pts - approx_centre[None], dim=-1)
    scales = torch.log(lod * scales.clamp(1e-6, 1e6)).unsqueeze(-1).repeat(1, 3)
    opacities = torch.ones(f_dc.shape[0], 1, device=dev)
    opacities[: uv.shape[0]] *= 0.2 * confs[..., None]
    penalty_map = penalty if torch.is_tensor(penalty) else torch.zeros_like(init_proba)
    return dict(init_proba=init_proba, penalty=penalty_map, sampled=sampled, valid=valid, xyz=pts, f_dc=f_dc, scaling=scales,
                opacity=inverse_sigmoid(opacities), d_max=depths.unsqueeze(-1) * lod, n=int(pts.shape[0]))


def add_and_prune(params, ext, mask):
    for k, v in ext.items():
        if k not in params:
            continue
        if k == "global_feat":
            params[k] = torch.cat([params[k], v], 0)
        else:
            params[k] = torch.cat([params[k][mask], v], 0)


def _cpu_voxel(new_xyz, xyz, cls_id, voxel_size, lod=None):
    dev = new_xyz.device
    out = voxel_ref.update_voxel(new_xyz.cpu(), xyz.cpu(), cls_id.cpu(), voxel_size)
    return tuple(o.to(dev) if torch.is_tensor(o) else o for o in out)


def add_new_gaussians(params, frame, render, *, keyframe_id, cam_centres, width, height, f, init_proba_scaler, gs_add_ratio,
                      voxel_size, visible_threshold, sh_degree=3, local_feat_dim, global_feat_dim, uniforms=None,
                      update_voxel=_cpu_voxel):
    """The whole method on ``params`` (modified in place).  ``render(cls_id)`` returns the raw render of the current scene.
    ``update_voxel(new_xyz, xyz, cls_id, voxel_size, lod)`` may be replaced.  Returns dict(uniforms, rows, renders, and the
    ``ext`` / ``valid_gs_mask`` handed to add_and_prune)."""
    out = dict(uniforms=[], rows=[], renders=0)
    if frame["is_test"]:
        return out
    dev = frame["image"].device
    disc = disc_kernel(dev)
    qmin = depth_threshold(frame["point_map"])
    ext = {}
    valid_gs_mask = None
    for i, lod in enumerate(LODS):
        raw = None
        if params["xyz"].shape[0] > 0:
            raw = render(params["cls_id"])
            out["renders"] += 1
        u = uniforms[i] if uniforms is not None else torch.rand(height // lod, width // lod, device=dev)
        out["uniforms"].append(u)
        rows = sample_lod(frame["image"], raw, frame["point_map"], frame["conf"], frame["R"], frame["t"],
                          frame["approx_centre"], frame["exposure"], lod=lod, f=f, init_proba_scaler=init_proba_scaler,
                          gs_add_ratio=gs_add_ratio, uniforms=u, qmin=qmin, disc=disc)
        L = rows["n"]
        out["rows"].append(rows)
        if params["xyz"].shape[0] > 0:
            upd, new_cls, nv = update_voxel(rows["xyz"], params["xyz"], params["cls_id"], voxel_size, lod)
            params["cls_id"] = upd
        else:
            new_cls, nv = update_voxel(rows["xyz"], params["xyz"], params["cls_id"], voxel_size, lod)
        rotation = torch.zeros((L, 4), device=dev)
        rotation[:, 0] = 1
        valid_gs_mask = prune_mask(params, frame["approx_centre"], f, width)
        ext[lod] = dict(id=torch.full((L, 1), keyframe_id, device=dev, dtype=torch.long), cls_id=new_cls, d_max=rows["d_max"],
                        xyz=rows["xyz"], f_dc=rows["f_dc"], f_rest=torch.zeros(L, (sh_degree + 1) ** 2 - 1, 3, device=dev),
                        opacity=rows["opacity"], scaling=rows["scaling"], rotation=rotation,
                        local_feat=torch.zeros((L, local_feat_dim), device=dev),
                        global_feat=torch.zeros((nv, global_feat_dim), device=dev))
    out["ext"] = {k: torch.cat([ext[lod][k] for lod in LODS], 0) for k in ext[1]}
    out["valid_gs_mask"] = valid_gs_mask
    add_and_prune(params, out["ext"], valid_gs_mask)
    weed_out(params, cam_centres, visible_threshold)
    return out


def weed_out(params, cam_centres, visible_threshold):
    xyz = params["xyz"]
    count = torch.zeros(xyz.shape[0], dtype=torch.int, device=xyz.device)
    for c in cam_centres:
        dist = (xyz - c).norm(dim=1, keepdim=True)
        count += (dist < 2 * params["d_max"]).squeeze(-1).int()
    # the reference's count / len(keyframes) on a CUDA tensor is count * fl32(1 / K) (PyTorch's CPU-scalar fast path);
    # written out so that the oracle gives that answer on the CPU as well
    inv = torch.tensor(np.float32(1.0) / np.float32(len(cam_centres)), device=count.device)
    mask = (count.float() * inv) > visible_threshold
    add_and_prune(params, {k: v[:0] for k, v in params.items()}, mask)
