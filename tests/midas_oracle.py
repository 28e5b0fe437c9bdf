"""Plain-PyTorch fp32 restatement of the conditioner's depth tower, the yardstick of the native one (hi3d_official_b200/midas.py):
MiDaS `DPTDepthModel(backbone="vitb_rn50_384", readout="project", non_negative=True, features=256)` (annotator/midas/dpt_depth.py,
vit.py, blocks.py) over timm's `vit_base_resnet50_384`:

  bit_forward   ResNetV2(layers=(3, 4, 9), preact=False, stem_type='same', conv_layer=StdConv2dSame(eps=1e-8)): weight-standardised
                convs with TF "same" padding, GroupNorm(32) (+ ReLU), non-pre-activation bottlenecks; returns the three stage outputs
  vit_forward   the hybrid patch embedding (1x1 conv of the /16 map, class token, positional embedding resized bilinearly as
                vit.py:104-121 does), then pre-LN blocks; returns the outputs of blocks 8 and 11 (the final norm is dead)
  dpt_forward   reassemble (ProjectReadout + 1x1 conv, + a 3x3 stride-2 conv for layer 4), layerN_rn, the four fusion blocks and
                the head -> (n, H, W) inverse depth

Nothing here imports the package under test or the reference.  `random_dpt_hybrid_sd` makes seeded weights with the reference's
state-dict keys, at full size or with reduced widths.
"""
import math

import torch
import torch.nn.functional as F

BB = "pretrained.model.patch_embed.backbone."
VIT = "pretrained.model."
HOOKS = (8, 11)


def _count(sd, prefix):
    return len({int(k[len(prefix):].split(".")[0]) for k in sd if k.startswith(prefix)})


def std_weight(w, eps=1e-8):
    m = w.mean(dim=(1, 2, 3), keepdim=True)
    v = w.var(dim=(1, 2, 3), unbiased=False, keepdim=True)
    return (w - m) / torch.sqrt(v + eps)


def pad_same(x, k, s, value=0.0):
    ih, iw = x.shape[-2:]
    ph = max((math.ceil(ih / s) - 1) * s + k - ih, 0)
    pw = max((math.ceil(iw / s) - 1) * s + k - iw, 0)
    return F.pad(x, (pw // 2, pw - pw // 2, ph // 2, ph - ph // 2), value=value)


def std_conv_same(x, w, stride):
    return F.conv2d(pad_same(x, w.shape[-1], stride), std_weight(w), stride=stride)


def gn(x, sd, p, act):
    y = F.group_norm(x, 32, sd[p + "weight"], sd[p + "bias"], eps=1e-5)
    return F.relu(y) if act else y


def bit_forward(sd, x):
    x = gn(std_conv_same(x, sd[BB + "stem.conv.weight"], 2), sd, BB + "stem.norm.", True)
    x = F.max_pool2d(pad_same(x, 3, 2, value=float("-inf")), 3, 2)
    feats = []
    for si in range(_count(sd, BB + "stages.")):
        for bi in range(_count(sd, BB + f"stages.{si}.blocks.")):
            p = BB + f"stages.{si}.blocks.{bi}."
            stride = 2 if (bi == 0 and si > 0) else 1
            sc = x
            if p + "downsample.conv.weight" in sd:
                sc = gn(std_conv_same(x, sd[p + "downsample.conv.weight"], stride), sd, p + "downsample.norm.", False)
            y = gn(std_conv_same(x, sd[p + "conv1.weight"], 1), sd, p + "norm1.", True)
            y = gn(std_conv_same(y, sd[p + "conv2.weight"], stride), sd, p + "norm2.", True)
            y = gn(std_conv_same(y, sd[p + "conv3.weight"], 1), sd, p + "norm3.", False)
            x = F.relu(y + sc)
        feats.append(x)
    return feats


def resize_pos_embed(pos, gh, gw):
    """vit.py:104-121: the grid part of (1, 1 + g*g, C) resized bilinearly (align_corners=False) to gh x gw."""
    tok, grid = pos[:, :1], pos[0, 1:]
    g = int(math.sqrt(len(grid)))
    grid = grid.reshape(1, g, g, -1).permute(0, 3, 1, 2)
    grid = F.interpolate(grid, size=(gh, gw), mode="bilinear")
    return torch.cat([tok, grid.permute(0, 2, 3, 1).reshape(1, gh * gw, -1)], 1)


def vit_block(sd, p, x):
    n, L, C = x.shape
    heads = C // 64
    h = F.layer_norm(x, (C,), sd[p + "norm1.weight"], sd[p + "norm1.bias"], eps=1e-6)
    q, k, v = F.linear(h, sd[p + "attn.qkv.weight"], sd[p + "attn.qkv.bias"]).reshape(n, L, 3, heads, 64).permute(2, 0, 3, 1, 4)
    a = torch.softmax((q @ k.transpose(-1, -2)) * 64 ** -0.5, -1) @ v
    x = x + F.linear(a.transpose(1, 2).reshape(n, L, C), sd[p + "attn.proj.weight"], sd[p + "attn.proj.bias"])
    h = F.layer_norm(x, (C,), sd[p + "norm2.weight"], sd[p + "norm2.bias"], eps=1e-6)
    h = F.gelu(F.linear(h, sd[p + "mlp.fc1.weight"], sd[p + "mlp.fc1.bias"]))
    return x + F.linear(h, sd[p + "mlp.fc2.weight"], sd[p + "mlp.fc2.bias"])


def vit_forward(sd, trunk):
    t = F.conv2d(trunk, sd[VIT + "patch_embed.proj.weight"], sd[VIT + "patch_embed.proj.bias"])
    n, C, gh, gw = t.shape
    t = t.flatten(2).transpose(1, 2)
    x = torch.cat([sd[VIT + "cls_token"].expand(n, -1, -1), t], 1) + resize_pos_embed(sd[VIT + "pos_embed"], gh, gw)
    outs = []
    for i in range(_count(sd, VIT + "blocks.")):
        x = vit_block(sd, VIT + f"blocks.{i}.", x)
        if i in HOOKS:
            outs.append(x)
    return outs, (gh, gw)


def reassemble(sd, x, idx, grid):
    """act_postprocess{3,4} (vit.py:446-477): ProjectReadout, unflatten, 1x1 conv [, 3x3 stride-2 conv]."""
    p = f"pretrained.act_postprocess{idx}."
    tok = x[:, 1:]
    r = F.gelu(F.linear(torch.cat([tok, x[:, :1].expand_as(tok)], -1), sd[p + "0.project.0.weight"], sd[p + "0.project.0.bias"]))
    r = r.transpose(1, 2).reshape(x.shape[0], -1, *grid)
    r = F.conv2d(r, sd[p + "3.weight"], sd[p + "3.bias"])
    if idx == 4:
        r = F.conv2d(r, sd[p + "4.weight"], sd[p + "4.bias"], stride=2, padding=1)
    return r


def rcu(sd, p, x):
    y = F.conv2d(F.relu(x), sd[p + "conv1.weight"], sd[p + "conv1.bias"], padding=1)
    return F.conv2d(F.relu(y), sd[p + "conv2.weight"], sd[p + "conv2.bias"], padding=1) + x


def fusion(sd, i, x0, x1=None):
    p = f"scratch.refinenet{i}."
    out = x0 if x1 is None else x0 + rcu(sd, p + "resConfUnit1.", x1)
    out = rcu(sd, p + "resConfUnit2.", out)
    out = F.interpolate(out, scale_factor=2, mode="bilinear", align_corners=True)
    return F.conv2d(out, sd[p + "out_conv.weight"], sd[p + "out_conv.bias"])


def dpt_forward(sd, x):
    """x: (n, 3, H, W) with H, W multiples of 32.  Returns (n, H, W)."""
    sd = {k: v.to(x.dtype) if v.is_floating_point() else v for k, v in sd.items()}
    l1, l2, trunk = bit_forward(sd, x)
    (h8, h11), grid = vit_forward(sd, trunk)
    layers = [l1, l2, reassemble(sd, h8, 3, grid), reassemble(sd, h11, 4, grid)]
    rn = [F.conv2d(t, sd[f"scratch.layer{i + 1}_rn.weight"], padding=1) for i, t in enumerate(layers)]
    path = fusion(sd, 4, rn[3])
    path = fusion(sd, 3, path, rn[2])
    path = fusion(sd, 2, path, rn[1])
    path = fusion(sd, 1, path, rn[0])
    h = F.conv2d(path, sd["scratch.output_conv.0.weight"], sd["scratch.output_conv.0.bias"], padding=1)
    h = F.interpolate(h, scale_factor=2, mode="bilinear", align_corners=True)
    h = F.relu(F.conv2d(h, sd["scratch.output_conv.2.weight"], sd["scratch.output_conv.2.bias"], padding=1))
    h = F.relu(F.conv2d(h, sd["scratch.output_conv.4.weight"], sd["scratch.output_conv.4.bias"]))
    return h[:, 0]


FULL = dict(stem=64, stage_out=(256, 512, 1024), stage_mid=(64, 128, 256), depths=(3, 4, 9), width=768, layers=12, features=256,
            grid=24)
# reduced widths: every channel count a multiple of 64 (the GEMM engine's K granule), 12 ViT blocks (the hooks are 8 and 11)
SMALL = dict(stem=64, stage_out=(128, 128, 256), stage_mid=(64, 64, 64), depths=(1, 1, 1), width=128, layers=12, features=128,
             grid=24)


def random_dpt_hybrid_sd(seed=0, stem=64, stage_out=(256, 512, 1024), stage_mid=(64, 128, 256), depths=(3, 4, 9), width=768,
                         layers=12, features=256, grid=24, mlp_ratio=4, device="cpu"):
    """Seeded weights under the reference's keys, dead `pretrained.model.norm.*` / `head.*` and the unused
    `refinenet4.resConfUnit1.*` included.  The BiT convs are standardised, so their scale does not matter; the fusion path is not
    normalised, so its convs are scaled to keep it O(1), and the last bias is positive so that the final ReLU keeps a varied map."""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s, std=1.0: (torch.randn(*s, generator=g) * std).to(device)   # noqa: E731
    sd = {}

    def norm(p, c, beta=0.1):
        sd[p + "weight"], sd[p + "bias"] = 1 + r(c, std=0.1), r(c, std=beta)

    def conv(p, co, ci, k, bias=True, gain=1.0):
        sd[p + "weight"] = r(co, ci, k, k, std=gain * (ci * k * k) ** -0.5)
        if bias:
            sd[p + "bias"] = r(co, std=0.05)

    sd[BB + "stem.conv.weight"] = r(stem, 3, 7, 7) + 0.1
    norm(BB + "stem.norm.", stem)
    cin = stem
    for si, (co, mid, d) in enumerate(zip(stage_out, stage_mid, depths)):
        for bi in range(d):
            p = BB + f"stages.{si}.blocks.{bi}."
            if bi == 0:
                sd[p + "downsample.conv.weight"] = r(co, cin, 1, 1)
                norm(p + "downsample.norm.", co)
            sd[p + "conv1.weight"] = r(mid, cin if bi == 0 else co, 1, 1)
            norm(p + "norm1.", mid)
            sd[p + "conv2.weight"] = r(mid, mid, 3, 3)
            norm(p + "norm2.", mid)
            sd[p + "conv3.weight"] = r(co, mid, 1, 1)
            norm(p + "norm3.", co)
        cin = co
    conv(VIT + "patch_embed.proj.", width, cin, 1)
    sd[VIT + "cls_token"] = r(1, 1, width, std=0.5)
    sd[VIT + "pos_embed"] = r(1, 1 + grid * grid, width, std=0.5)
    sc = width ** -0.5
    for i in range(layers):
        p = VIT + f"blocks.{i}."
        sd.update({p + "norm1.weight": 1 + r(width, std=0.1), p + "norm1.bias": r(width, std=0.05),
                   p + "attn.qkv.weight": r(3 * width, width, std=sc), p + "attn.qkv.bias": r(3 * width, std=0.02),
                   p + "attn.proj.weight": r(width, width, std=sc * 0.5), p + "attn.proj.bias": r(width, std=0.02),
                   p + "norm2.weight": 1 + r(width, std=0.1), p + "norm2.bias": r(width, std=0.05),
                   p + "mlp.fc1.weight": r(mlp_ratio * width, width, std=sc), p + "mlp.fc1.bias": r(mlp_ratio * width, std=0.02),
                   p + "mlp.fc2.weight": r(width, mlp_ratio * width, std=(mlp_ratio * width) ** -0.5 * 0.5),
                   p + "mlp.fc2.bias": r(width, std=0.02)})
    sd[VIT + "norm.weight"], sd[VIT + "norm.bias"] = 1 + r(width, std=0.1), r(width, std=0.05)
    sd[VIT + "head.weight"], sd[VIT + "head.bias"] = r(1000, width, std=sc), r(1000, std=0.02)
    for idx in (3, 4):
        p = f"pretrained.act_postprocess{idx}."
        sd[p + "0.project.0.weight"] = r(width, 2 * width, std=(2 * width) ** -0.5)
        sd[p + "0.project.0.bias"] = r(width, std=0.05)
        conv(p + "3.", width, width, 1)
        if idx == 4:
            conv(p + "4.", width, width, 3)
    for i, ci in enumerate((stage_out[0], stage_out[1], width, width)):
        conv(f"scratch.layer{i + 1}_rn.", features, ci, 3, bias=False)
    for i in (1, 2, 3, 4):
        p = f"scratch.refinenet{i}."
        for u in ("resConfUnit1.", "resConfUnit2."):
            conv(p + u + "conv1.", features, features, 3, gain=2 ** 0.5)
            conv(p + u + "conv2.", features, features, 3, gain=0.5)
        conv(p + "out_conv.", features, features, 1)
    conv("scratch.output_conv.0.", features // 2, features, 3)
    conv("scratch.output_conv.2.", 32, features // 2, 3, gain=2 ** 0.5)
    conv("scratch.output_conv.4.", 1, 32, 1)
    sd["scratch.output_conv.4.bias"] = torch.full((1,), 2.0, device=device)
    return sd


def relerr(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm())
