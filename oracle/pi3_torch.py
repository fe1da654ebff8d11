"""TEST INFRASTRUCTURE ONLY.  Plain-PyTorch restatement of the reference's Pi3 inference path and of the Backend's
accurate loop-closure scoring, written functionally over a state dict that uses the REFERENCE'S parameter names.

Restates (all under the ARTDECO tree's VSLAM/):
  forward                thirdparty/Pi3/pi3/models/pi3.py:132-216
  DINOv2 encoder         thirdparty/Pi3/pi3/models/dinov2/models/vision_transformer.py:181-234,262-275,
                         dinov2/layers/block.py:88-113, attention.py:56-69, patch_embed.py:68-78
  BlockRope / qk-norm    thirdparty/Pi3/pi3/models/layers/block.py:259-335, attention.py:238-347
  RoPE2D                 thirdparty/Pi3/pi3/models/layers/pos_embed.py:111-158
  TransformerDecoder     thirdparty/Pi3/pi3/models/layers/transformer_head.py:9-80
  CameraHead             thirdparty/Pi3/pi3/models/layers/camera_head.py:7-93
  accurate_loop_closure  mast3r_slam/retrieval_database.py:21-41,263-326 (without the similarity graph)
PINNED BY RUNNING THE REFERENCE: tests/golden/make_pi3_golden.py runs the real module on CPU with the same deterministic
weights, checks this file against it and writes the golden outputs the GPU tests use.

Attention runs through ``F.scaled_dot_product_attention`` so the same code serves as the fp32 oracle and, under bf16
autocast on a GPU, as the way the reference itself runs (tests/perf/time_pi3.py)."""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

IMAGE_MEAN = (0.485, 0.456, 0.406)
IMAGE_STD = (0.229, 0.224, 0.225)
PATCH = 14
N_SPECIAL = 5          # encoder: cls + 4 registers; decoder: 5 register tokens


def _ln(x, sd, pre, eps=1e-6):
    return F.layer_norm(x, (x.shape[-1],), sd[pre + ".weight"], sd[pre + ".bias"], eps)


def _lin(x, sd, pre):
    return F.linear(x, sd[pre + ".weight"], sd.get(pre + ".bias"))


def interpolate_pos_embed(pos_embed, gh, gw):
    """The [1, 1 + gh*gw, C] table of vision_transformer.py:181-213 (bicubic, antialias, no offset)."""
    N = pos_embed.shape[1] - 1
    M = int(math.sqrt(N))
    if gh == M and gw == M:
        return pos_embed
    pe = pos_embed.float()
    patch = pe[:, 1:].reshape(1, M, M, -1).permute(0, 3, 1, 2)
    patch = F.interpolate(patch, mode="bicubic", antialias=True, size=(gh, gw))
    patch = patch.permute(0, 2, 3, 1).reshape(1, gh * gw, -1)
    return torch.cat((pe[:, 0].unsqueeze(0), patch), dim=1).to(pos_embed.dtype)


def rope2d(t, pos, base=100.0):
    """t [B,h,N,64], pos [B,N,2] (y, x) int64: rotate_half RoPE on each 32-wide half."""
    D = t.shape[-1] // 2
    inv = 1.0 / (base ** (torch.arange(0, D, 2, device=t.device).float() / D))

    def one(u, p):
        fr = p[..., None].to(inv.dtype) * inv
        fr = torch.cat([fr, fr], -1)[:, None].to(u.dtype)
        rot = torch.cat([-u[..., D // 2:], u[..., :D // 2]], -1)
        return u * fr.cos() + rot * fr.sin()

    y, x = t.chunk(2, dim=-1)
    return torch.cat([one(y, pos[..., 0]), one(x, pos[..., 1])], -1)


def _attention(x, sd, pre, heads, pos=None, qk_norm=False):
    B, N, C = x.shape
    qkv = _lin(x, sd, pre + ".qkv").reshape(B, N, 3, heads, C // heads).permute(2, 0, 3, 1, 4)
    q, k, v = qkv[0], qkv[1], qkv[2]
    if qk_norm:   # nn.LayerNorm(head_dim) with its default eps (attention.py:248,261)
        q = F.layer_norm(q, (q.shape[-1],), sd[pre + ".q_norm.weight"], sd[pre + ".q_norm.bias"], 1e-5).to(v.dtype)
        k = F.layer_norm(k, (k.shape[-1],), sd[pre + ".k_norm.weight"], sd[pre + ".k_norm.bias"], 1e-5).to(v.dtype)
    if pos is not None:
        q, k = rope2d(q, pos), rope2d(k, pos)
    o = F.scaled_dot_product_attention(q, k, v)
    return _lin(o.transpose(1, 2).reshape(B, N, C), sd, pre + ".proj")


def _block(x, sd, pre, heads, pos=None, qk_norm=False):
    ls1, ls2 = sd.get(pre + ".ls1.gamma"), sd.get(pre + ".ls2.gamma")
    a = _attention(_ln(x, sd, pre + ".norm1"), sd, pre + ".attn", heads, pos, qk_norm)
    x = x + (a * ls1 if ls1 is not None else a)
    m = _lin(F.gelu(_lin(_ln(x, sd, pre + ".norm2"), sd, pre + ".mlp.fc1")), sd, pre + ".mlp.fc2")
    return x + (m * ls2 if ls2 is not None else m)


def encode(sd, imgs):
    """imgs [BN,3,H,W] in [0,1] -> x_norm_patchtokens [BN, gh*gw, 1024]."""
    mean = torch.tensor(IMAGE_MEAN, device=imgs.device).view(1, 3, 1, 1)
    std = torch.tensor(IMAGE_STD, device=imgs.device).view(1, 3, 1, 1)
    x = (imgs - mean) / std
    BN, _, H, W = x.shape
    gh, gw = H // PATCH, W // PATCH
    x = F.conv2d(x, sd["encoder.patch_embed.proj.weight"], sd["encoder.patch_embed.proj.bias"], stride=PATCH)
    x = x.flatten(2).transpose(1, 2)
    x = torch.cat((sd["encoder.cls_token"].expand(BN, -1, -1), x), dim=1)
    x = x + interpolate_pos_embed(sd["encoder.pos_embed"], gh, gw)
    x = torch.cat((x[:, :1], sd["encoder.register_tokens"].expand(BN, -1, -1), x[:, 1:]), dim=1)
    i = 0
    while f"encoder.blocks.{i}.norm1.weight" in sd:
        x = _block(x, sd, f"encoder.blocks.{i}", 16)
        i += 1
    return _ln(x, sd, "encoder.norm")[:, N_SPECIAL:]


def positions(BN, gh, gw, device):
    """pi3.py:147-154: (y, x) + 1 for patches, 0 for the 5 register tokens."""
    yy, xx = torch.meshgrid(torch.arange(gh, device=device), torch.arange(gw, device=device), indexing="ij")
    p = torch.stack([yy.reshape(-1), xx.reshape(-1)], -1) + 1
    p = torch.cat([torch.zeros(N_SPECIAL, 2, dtype=p.dtype, device=device), p], 0)
    return p[None].expand(BN, -1, -1).contiguous()


def decoder(sd, hidden, N, gh, gw):
    """pi3.py:132-171 -> ([BN, hw, 2048] concat of the last two blocks, pos [BN, hw, 2])."""
    BN, n, C = hidden.shape
    B = BN // N
    hidden = torch.cat([sd["register_token"].reshape(1, N_SPECIAL, C).expand(BN, -1, -1), hidden], 1)
    hw = hidden.shape[1]
    pos = positions(BN, gh, gw, hidden.device)
    depth = 0
    while f"decoder.{depth}.norm1.weight" in sd:
        depth += 1
    out = []
    for i in range(depth):
        if i % 2 == 0:
            hidden = _block(hidden.reshape(BN, hw, C), sd, f"decoder.{i}", 16, pos.reshape(BN, hw, 2), qk_norm=True)
        else:
            hidden = _block(hidden.reshape(B, N * hw, C), sd, f"decoder.{i}", 16, pos.reshape(B, N * hw, 2), qk_norm=True)
        if i + 1 in (depth - 1, depth):
            out.append(hidden.reshape(BN, hw, C))
    return torch.cat(out, -1), pos


def head_decoder(sd, pre, hidden, pos):
    """TransformerDecoder.forward (transformer_head.py:48-56)."""
    h = _lin(hidden, sd, pre + ".projects")
    i = 0
    while f"{pre}.blocks.{i}.norm1.weight" in sd:
        h = _block(h, sd, f"{pre}.blocks.{i}", 16, pos)
        i += 1
    return _lin(h, sd, pre + ".linear_out")


def linear_pts(sd, pre, tokens, H, W):
    """LinearPts3d.forward (transformer_head.py:70-80) -> [BN, H, W, c]."""
    BN, S, _ = tokens.shape
    feat = _lin(tokens, sd, pre + ".proj").transpose(-1, -2).reshape(BN, -1, H // PATCH, W // PATCH)
    return F.pixel_shuffle(feat, PATCH).permute(0, 2, 3, 1)


def svd_orthogonalize(m):
    """camera_head.py:74-93: m [BN, 9] -> R [BN, 3, 3]."""
    m = m.reshape(-1, 3, 3)
    mt = F.normalize(m, p=2, dim=-1).transpose(-1, -2)
    u, s, v = torch.svd(mt)
    det = torch.det(v @ u.transpose(-2, -1))
    return torch.cat([v[:, :, :-1], v[:, :, -1:] * det.view(-1, 1, 1)], dim=2) @ u.transpose(-2, -1)


def camera_head(sd, feat):
    """CameraHead.forward (camera_head.py:48-72) on the patch tokens [BN, hw', 512] -> (pose, fc_rot, fc_t)."""
    p = "camera_head"
    for i in range(2):
        x = F.relu(_lin(feat, sd, f"{p}.res_conv.{i}.res_conv1"))
        x = F.relu(_lin(x, sd, f"{p}.res_conv.{i}.res_conv2"))
        x = F.relu(_lin(x, sd, f"{p}.res_conv.{i}.res_conv3"))
        feat = feat + x
    f = feat.mean(1)
    f = F.relu(_lin(F.relu(_lin(f, sd, f"{p}.more_mlps.0")), sd, f"{p}.more_mlps.2"))
    t = _lin(f.float(), sd, f"{p}.fc_t")
    r = _lin(f.float(), sd, f"{p}.fc_rot")
    BN = f.shape[0]
    pose = torch.zeros(BN, 4, 4, device=f.device, dtype=torch.float32)
    pose[:, :3, :3] = svd_orthogonalize(r.float())
    pose[:, :3, 3] = t.float()
    pose[:, 3, 3] = 1.0
    return pose, r, t


def forward(sd, imgs, stages: dict | None = None):
    """Pi3.forward (pi3.py:173-216): imgs [B,N,3,H,W] in [0,1] -> dict(points, local_points, conf, camera_poses).
    ``stages``, when given, receives the intermediate tensors the golden files record."""
    B, N, _, H, W = imgs.shape
    gh, gw = H // PATCH, W // PATCH
    enc = encode(sd, imgs.reshape(B * N, 3, H, W))
    hidden, pos = decoder(sd, enc, N, gh, gw)
    ph = head_decoder(sd, "point_decoder", hidden, pos)
    ch = head_decoder(sd, "conf_decoder", hidden, pos)
    cam = head_decoder(sd, "camera_decoder", hidden, pos)
    with torch.autocast(device_type=imgs.device.type, enabled=False):     # pi3.py:192: the heads run in fp32
        return _heads(sd, ph, ch, cam, B, N, H, W, hidden, enc, stages)


def _heads(sd, ph, ch, cam, B, N, H, W, hidden, enc, stages):
    ret = linear_pts(sd, "point_head", ph[:, N_SPECIAL:].float(), H, W).reshape(B, N, H, W, -1)
    xy, z = ret.split([2, 1], dim=-1)
    z = torch.exp(z)
    local_points = torch.cat([xy * z, z], dim=-1)
    conf = linear_pts(sd, "conf_head", ch[:, N_SPECIAL:].float(), H, W).reshape(B, N, H, W, -1)
    pose, r, t = camera_head(sd, cam[:, N_SPECIAL:].float())
    pose = pose.reshape(B, N, 4, 4)
    homog = torch.cat([local_points, torch.ones_like(local_points[..., :1])], -1)
    points = torch.einsum("bnij, bnhwj -> bnhwi", pose, homog)[..., :3]
    if stages is not None:
        stages.update(encoder=enc, decoder=hidden, point_hidden=ph, conf_hidden=ch, camera_hidden=cam, fc_rot=r, fc_t=t)
    return dict(points=points, local_points=local_points, conf=conf, camera_poses=pose)


# ---- accurate loop closure (retrieval_database.py:21-41,263-326) -------------------------------------------------
def prepare_window(images, H=392, W=518):
    """inverse_normalize then bilinear resize: [N,3,h,w] in [-1,1] -> [1,N,3,H,W] in [0,1]."""
    x = (images * 0.5 + 0.5).clamp(0, 1)
    return F.interpolate(x, size=(H, W), mode="bilinear", align_corners=False)[None].contiguous()


def score_window(points, idxs_all, config, match_fn, chunk=32):
    """points [N,H,W,3] with the query last -> (selected ids, per-pair valid counts [N-1]).  ``match_fn`` is
    ``match_pi3(config, X11, X21)`` returning (idx, valid [b, H*W])."""
    ii = list(idxs_all[:-1])
    n = len(ii)
    valid = []
    for i in range(0, n, chunk):
        e = min(i + chunk, n)
        _, v = match_fn(config, points[i:e], points[-1:].expand(e - i, -1, -1, -1).contiguous())
        valid.append(v)
    valid = torch.cat(valid, 0)
    pct = valid.sum(-1) / valid[0].numel()
    order = torch.argsort(pct, descending=True)
    keep = order[pct[order] > config["retrieval"]["accurate_min"]]
    ids = [ii[i] for i in keep.tolist()]
    return ids[:config["retrieval"]["k"]], valid.sum(-1)
