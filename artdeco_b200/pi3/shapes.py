"""The parameter table of the reference's ``Pi3`` (VSLAM/thirdparty/Pi3/pi3/models/pi3.py:17-130): every key
inference reads, with its shape.  ``synthetic.det_weights(param_shapes())`` builds deterministic weights that load into
both the reference module and ``artdeco_b200.pi3.Pi3``."""
from __future__ import annotations

PATCH = 14
N_SPECIAL = 5          # encoder: cls + 4 registers; decoder: 5 register tokens


def param_shapes(depth_enc=24, depth_dec=36, depth_head=5):
    """{reference key: shape} of every parameter inference reads (no ``mask_token``; DINOv2's head is an Identity)."""
    s = {}
    E = 1024

    def lin(pre, o, i):
        s[pre + ".weight"] = (o, i)
        s[pre + ".bias"] = (o,)

    def ln(pre, c=E):
        s[pre + ".weight"] = (c,)
        s[pre + ".bias"] = (c,)

    def block(pre, ls, qk):
        ln(pre + ".norm1")
        lin(pre + ".attn.qkv", 3 * E, E)
        if qk:
            ln(pre + ".attn.q_norm", 64)
            ln(pre + ".attn.k_norm", 64)
        lin(pre + ".attn.proj", E, E)
        if ls:
            s[pre + ".ls1.gamma"] = (E,)
        ln(pre + ".norm2")
        lin(pre + ".mlp.fc1", 4 * E, E)
        lin(pre + ".mlp.fc2", E, 4 * E)
        if ls:
            s[pre + ".ls2.gamma"] = (E,)

    s["encoder.cls_token"] = (1, 1, E)
    s["encoder.pos_embed"] = (1, 37 * 37 + 1, E)
    s["encoder.register_tokens"] = (1, 4, E)
    s["encoder.patch_embed.proj.weight"] = (E, 3, PATCH, PATCH)
    s["encoder.patch_embed.proj.bias"] = (E,)
    for i in range(depth_enc):
        block(f"encoder.blocks.{i}", True, False)
    ln("encoder.norm")
    for i in range(depth_dec):
        block(f"decoder.{i}", True, True)
    s["register_token"] = (1, 1, N_SPECIAL, E)
    for name, out in (("point_decoder", E), ("conf_decoder", E), ("camera_decoder", 512)):
        lin(name + ".projects", E, 2 * E)
        for i in range(depth_head):
            block(f"{name}.blocks.{i}", False, False)
        lin(name + ".linear_out", out, E)
    lin("point_head.proj", 3 * PATCH * PATCH, E)
    lin("conf_head.proj", PATCH * PATCH, E)
    for i in range(2):
        for j in (1, 2, 3):
            lin(f"camera_head.res_conv.{i}.res_conv{j}", 512, 512)
    lin("camera_head.more_mlps.0", 512, 512)
    lin("camera_head.more_mlps.2", 512, 512)
    lin("camera_head.fc_t", 3, 512)
    lin("camera_head.fc_rot", 9, 512)
    return s
