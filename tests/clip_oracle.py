"""Plain-PyTorch fp32 restatement of the conditioner's CLIP image towers, the yardstick of the native ones
(hi3d_official_b200/clip_vision.py):

  vision_forward     open_clip 2.24 VisionTransformer.forward (class token, no patch dropout, 'tok' pooling, ln_post, proj) /
                     OpenAI clip/model.py VisionTransformer.forward -- the same network, with nn.GELU or QuickGELU
  kornia_resize      kornia 0.6.9 geometry.resize(bicubic, align_corners=True, antialias=True), written out independently
  aesthetic_mlp      tools/aes_score.py MLP (five Linear layers, dropout = identity), unfolded

Nothing here imports the package under test or the reference.  `random_visual_sd` makes seeded `visual.*` weights with
open_clip's initialisation scales, for tests of any width.
"""
import torch
import torch.nn.functional as F

CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)


def _mha(x, w_in, b_in, w_out, b_out, heads):
    n, L, C = x.shape
    d = C // heads
    q, k, v = (x @ w_in.t() + b_in).split(C, -1)
    q, k, v = (t.reshape(n, L, heads, d).transpose(1, 2) for t in (q, k, v))
    a = torch.softmax((q * d ** -0.5) @ k.transpose(-1, -2), -1) @ v
    return a.transpose(1, 2).reshape(n, L, C) @ w_out.t() + b_out


def vision_forward(sd, x, head_width, quick_gelu):
    """sd: `visual.*` tensors without the prefix; x: (n, 3, H, W) normalised images.  Returns (n, out_dim)."""
    sd = {k: v.to(x.dtype) if v.is_floating_point() else v for k, v in sd.items()}
    width = sd["conv1.weight"].shape[0]
    heads = width // head_width
    layers = len({k.split(".")[2] for k in sd if k.startswith("transformer.resblocks.")})
    y = F.conv2d(x, sd["conv1.weight"], stride=sd["conv1.weight"].shape[-1])
    y = y.reshape(y.shape[0], width, -1).permute(0, 2, 1)
    cls = sd["class_embedding"].reshape(1, 1, width).expand(y.shape[0], 1, width)
    y = torch.cat([cls.to(y.dtype), y], 1) + sd["positional_embedding"].to(y.dtype)
    y = F.layer_norm(y, (width,), sd["ln_pre.weight"], sd["ln_pre.bias"])
    for i in range(layers):
        p = f"transformer.resblocks.{i}."
        h = F.layer_norm(y, (width,), sd[p + "ln_1.weight"], sd[p + "ln_1.bias"])
        y = y + _mha(h, sd[p + "attn.in_proj_weight"], sd[p + "attn.in_proj_bias"], sd[p + "attn.out_proj.weight"],
                     sd[p + "attn.out_proj.bias"], heads)
        h = F.layer_norm(y, (width,), sd[p + "ln_2.weight"], sd[p + "ln_2.bias"])
        h = F.linear(h, sd[p + "mlp.c_fc.weight"], sd[p + "mlp.c_fc.bias"])
        h = h * torch.sigmoid(1.702 * h) if quick_gelu else F.gelu(h)
        y = y + F.linear(h, sd[p + "mlp.c_proj.weight"], sd[p + "mlp.c_proj.bias"])
    pooled = F.layer_norm(y[:, 0], (width,), sd["ln_post.weight"], sd["ln_post.bias"])
    return pooled @ sd["proj"]


def normalize(x):
    m = torch.tensor(CLIP_MEAN, device=x.device, dtype=x.dtype).view(1, 3, 1, 1)
    s = torch.tensor(CLIP_STD, device=x.device, dtype=x.dtype).view(1, 3, 1, 1)
    return (x - m) / s


def gaussian_kernel1d(ks, sigma):
    x = torch.arange(ks, dtype=torch.float64) - ks // 2
    if ks % 2 == 0:
        x = x + 0.5
    g = torch.exp(-x ** 2 / (2 * sigma ** 2))
    return (g / g.sum()).float()


def kornia_resize(x, size=(224, 224)):
    h, w = x.shape[-2:]
    if (h, w) == tuple(size):
        return x
    factors = (h / size[0], w / size[1])
    if max(factors) > 1:                          # kornia blurs only when downscaling
        sig = [max((f - 1.0) / 2.0, 0.001) for f in factors]
        ks = [int(max(4.0 * s, 3)) for s in sig]
        ks = [k + (k % 2 == 0) for k in ks]
        k2 = gaussian_kernel1d(ks[0], sig[0])[:, None] * gaussian_kernel1d(ks[1], sig[1])[None, :]
        c = x.shape[1]
        xp = F.pad(x, (ks[1] // 2, ks[1] // 2, ks[0] // 2, ks[0] // 2), mode="reflect")
        x = F.conv2d(xp, k2.to(x).expand(c, 1, *k2.shape), groups=c)
    return F.interpolate(x, size=size, mode="bicubic", align_corners=True)


def openclip_embed(sd, images):
    """FrozenOpenCLIPImageEmbedder.forward without the autocast: [-1, 1] images -> resize -> [0, 1] -> CLIP normalisation -> ViT-H."""
    return vision_forward(sd, normalize((kornia_resize(images.float()) + 1) / 2), 80, False)


def aesthetic_mlp(mlp_sd, x):
    for i in (0, 2, 4, 6, 7):
        x = F.linear(x, mlp_sd[f"layers.{i}.weight"].to(x), mlp_sd[f"layers.{i}.bias"].to(x))
    return x


def aesthetic_score(visual_sd, mlp_sd, x_normalised):
    f = vision_forward(visual_sd, x_normalised, 64, True)
    return aesthetic_mlp(mlp_sd, f / f.norm(dim=-1, keepdim=True))


def random_visual_sd(width, layers, head_width, out_dim, patch=14, grid=16, mlp_ratio=4, seed=0, device="cpu"):
    """Seeded `visual.*` tensors (no prefix) with the initialisation scales of open_clip's VisionTransformer /
    Transformer.init_parameters; LayerNorm affine and biases are perturbed so that every term matters."""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s, std=1.0: (torch.randn(*s, generator=g) * std).to(device)   # noqa: E731
    mlp = width * mlp_ratio
    sc = width ** -0.5
    sd = {"conv1.weight": r(width, 3, patch, patch, std=(3 * patch * patch) ** -0.5),
          "class_embedding": r(width, std=sc), "positional_embedding": r(grid * grid + 1, width, std=sc),
          "ln_pre.weight": 1 + r(width, std=0.1), "ln_pre.bias": r(width, std=0.05),
          "ln_post.weight": 1 + r(width, std=0.1), "ln_post.bias": r(width, std=0.05), "proj": r(width, out_dim, std=sc)}
    proj_std = sc * (2 * layers) ** -0.5
    for i in range(layers):
        p = f"transformer.resblocks.{i}."
        sd.update({p + "ln_1.weight": 1 + r(width, std=0.1), p + "ln_1.bias": r(width, std=0.05),
                   p + "attn.in_proj_weight": r(3 * width, width, std=sc), p + "attn.in_proj_bias": r(3 * width, std=0.02),
                   p + "attn.out_proj.weight": r(width, width, std=proj_std), p + "attn.out_proj.bias": r(width, std=0.02),
                   p + "ln_2.weight": 1 + r(width, std=0.1), p + "ln_2.bias": r(width, std=0.05),
                   p + "mlp.c_fc.weight": r(mlp, width, std=(2 * width) ** -0.5), p + "mlp.c_fc.bias": r(mlp, std=0.02),
                   p + "mlp.c_proj.weight": r(width, mlp, std=proj_std), p + "mlp.c_proj.bias": r(width, std=0.02)})
    return sd


def random_aesthetic_mlp(dim=768, seed=0):
    g = torch.Generator().manual_seed(seed)
    sd, prev = {}, dim
    for i, n in zip((0, 2, 4, 6, 7), (1024, 128, 64, 16, 1)):
        sd[f"layers.{i}.weight"] = torch.randn(n, prev, generator=g) * prev ** -0.5
        sd[f"layers.{i}.bias"] = torch.randn(n, generator=g) * 0.1
        prev = n
    return sd


def relerr(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm())

