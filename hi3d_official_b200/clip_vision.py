"""CLIP image towers of the conditioner on this package's kernels (SURVEY §8f N2):

  OpenCLIP ViT-H/14   FrozenOpenCLIPImageEmbedder (sgm/modules/encoders/modules.py:570-728) -> crossattn (B, 1, 1024)
  OpenAI CLIP ViT-L/14 + the aesthetic MLP   AesEmbedder (vtdm/encoders.py:56-90, tools/aes_score.py) -> vector[:, :256]

Both are pre-LN CLIP vision transformers (open_clip 2.24 `VisionTransformer`, OpenAI `clip/model.py`), so one engine serves
both; per image of 224^2 (P = 256 patches of 14^2, 257 tokens with the class token):

  hi3d_clip_patchify (CLIP mean / std, a zero class-token row) -> patch GEMM (conv1, no bias)
  -> hi3d_layernorm with addvec = positional_embedding (+ class_embedding in row 0), i.e. x + pos fused with ln_pre
  -> per residual block: ln_1 -> in_proj GEMM (bias) -> hi3d_attention_d80_tc5 / _d64_tc5 -> out_proj GEMM (bias) -> + x
                         ln_2 -> c_fc GEMM (GELU | QuickGELU epilogue) -> c_proj GEMM (bias) -> + x
  -> ln_post on the class rows -> proj GEMM.

The residual stream x is kept in fp32, as the reference's autocast forward keeps it; its two adds per block and the fp16 copy
that feeds the next LayerNorm are element-wise torch ops on a [257 n, width] tensor.  With the stream in fp16 (the GEMMs'
residual epilogue) the 64 rounded adds of ViT-H/14 gave 3.0x the error of the fp32 oracle run under autocast, against 2x
allowed (SURVEY §8c); the tower runs once per video, so the extra traffic does not matter.

Weights are the `visual.*` tensors of an open_clip / OpenAI checkpoint; width, layers, patch size, grid and output width are
read from their shapes, the head width comes from the architecture (80 for ViT-H-14, 64 for OpenAI CLIP: clip.build_model's
vision_width // 64).  Activations are fp16 with fp32 accumulation; LayerNorm statistics are fp32.
"""
from __future__ import annotations

import os
import re
from typing import Dict, Optional, Tuple

import torch
import torch.nn.functional as F

CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)

# head width and MLP activation per architecture (open_clip model configs; OpenAI CLIP: 64, QuickGELU)
ARCH_HEAD_WIDTH = {"ViT-H-14": 80, "ViT-g-14": 88, "ViT-bigG-14": 104}
OPENAI_HEAD_WIDTH = 64


def head_width_of(arch: str) -> int:
    return ARCH_HEAD_WIDTH.get(arch, 64)


# ---- checkpoint readers -------------------------------------------------------------------------------------------------
def _visual(sd: Dict[str, torch.Tensor], prefix: str = "visual.") -> Dict[str, torch.Tensor]:
    out = {k[len(prefix):]: v for k, v in sd.items() if k.startswith(prefix)}
    if not out:
        raise KeyError(f"no '{prefix}*' tensors in the checkpoint ({len(sd)} keys)")
    return out


def load_open_clip(path: str) -> Dict[str, torch.Tensor]:
    """open_clip .bin / .pt: a plain state dict, possibly wrapped in 'state_dict' and prefixed 'module.'.  Returns the image
    tower's tensors without the 'visual.' prefix; text-tower keys are ignored."""
    sd = torch.load(path, map_location="cpu", weights_only=True)
    if isinstance(sd, dict) and "state_dict" in sd and isinstance(sd["state_dict"], dict):
        sd = sd["state_dict"]
    sd = {(k[len("module."):] if k.startswith("module.") else k): v for k, v in sd.items()}
    return _visual(sd)


def load_openai_clip(path: str) -> Dict[str, torch.Tensor]:
    """OpenAI CLIP checkpoint (ckpts/ViT-L-14.pt): a TorchScript archive, read with torch.jit.load(...).state_dict(); a plain
    saved state dict is read with torch.load."""
    try:
        sd = torch.jit.load(path, map_location="cpu").state_dict()
    except RuntimeError:
        sd = torch.load(path, map_location="cpu", weights_only=True)
    return _visual(dict(sd))


def load_aesthetic_mlp(path: str) -> Tuple[torch.Tensor, torch.Tensor]:
    """tools/aes_score.py MLP state dict (layers.{0,2,4,6,7} Linear; the Dropouts are identities at inference and there is no
    nonlinearity): folded, in fp32, into one affine map score = w . x + b.  Returns (w (in,), b ())."""
    sd = torch.load(path, map_location="cpu", weights_only=True)
    if isinstance(sd, dict) and "state_dict" in sd:
        sd = sd["state_dict"]
    return fold_linear_chain(sd)


def fold_linear_chain(sd: Dict[str, torch.Tensor]) -> Tuple[torch.Tensor, torch.Tensor]:
    idx = sorted({int(m.group(1)) for k in sd for m in [re.match(r"layers\.(\d+)\.weight$", k)] if m})
    if not idx:
        raise KeyError("aesthetic MLP: no layers.N.weight tensors")
    W = sd[f"layers.{idx[0]}.weight"].double()
    b = sd[f"layers.{idx[0]}.bias"].double()
    for i in idx[1:]:
        Wi, bi = sd[f"layers.{i}.weight"].double(), sd[f"layers.{i}.bias"].double()
        W, b = Wi @ W, Wi @ b + bi
    if W.shape[0] != 1:
        raise ValueError(f"aesthetic MLP: expected one output, got {W.shape[0]}")
    return W[0].float(), b[0].float()


# ---- preprocessing (host glue, once per video) -------------------------------------------------------------------------
def _gaussian_taps(ks: int, sigma: float, device) -> torch.Tensor:
    x = torch.arange(ks, dtype=torch.float32, device=device) - ks // 2
    if ks % 2 == 0:
        x = x + 0.5
    g = torch.exp(-x.pow(2.0) / (2.0 * sigma ** 2))
    return g / g.sum()


def kornia_resize(x: torch.Tensor, size: Tuple[int, int] = (224, 224)) -> torch.Tensor:
    """kornia.geometry.resize(x, size, interpolation='bicubic', align_corners=True, antialias=True) of kornia 0.6.9: when
    downscaling, a separable Gaussian blur (sigma = max((factor - 1) / 2, 0.001) per axis, odd kernel size int(max(4 sigma,
    3)), reflect padding) and then bicubic interpolation with aligned corners."""
    h, w = x.shape[-2:]
    if (h, w) == tuple(size):
        return x
    fh, fw = h / size[0], w / size[1]
    if max(fh, fw) > 1:
        sig = (max((fh - 1.0) / 2.0, 0.001), max((fw - 1.0) / 2.0, 0.001))
        ks = [int(max(2.0 * 2 * s, 3)) for s in sig]
        ks = [k + 1 if k % 2 == 0 else k for k in ks]
        n, c = x.shape[:2]
        ky, kx = _gaussian_taps(ks[0], sig[0], x.device), _gaussian_taps(ks[1], sig[1], x.device)
        y = F.pad(x.reshape(n * c, 1, h, w), (ks[1] // 2, ks[1] // 2, ks[0] // 2, ks[0] // 2), mode="reflect")
        y = F.conv2d(y, kx.view(1, 1, 1, -1).to(y.dtype))
        y = F.conv2d(y, ky.view(1, 1, -1, 1).to(y.dtype))
        x = y.reshape(n, c, h, w)
    return F.interpolate(x, size=size, mode="bicubic", align_corners=True)


def openclip_preprocess(x: torch.Tensor) -> torch.Tensor:
    """FrozenOpenCLIPImageEmbedder.preprocess (modules.py:632-644) up to the CLIP normalisation, which hi3d_clip_patchify applies:
    images in [-1, 1] -> 224^2 -> [0, 1], fp32."""
    return (kornia_resize(x.float(), (224, 224)) + 1.0) / 2.0


# ---- the tower ----------------------------------------------------------------------------------------------------------
class ClipVisionTower:
    """A CLIP vision transformer on the hi3d kernels.  `sd`: the `visual.*` tensors without the prefix (CPU or CUDA, any float
    dtype); `head_width`: 80 for OpenCLIP ViT-H-14, 64 for OpenAI CLIP; `quick_gelu`: OpenAI CLIP's MLP activation.  The
    packed weights live on `device` (fp16 matrices, fp32 biases and LayerNorm parameters)."""

    def __init__(self, sd: Dict[str, torch.Tensor], head_width: int, quick_gelu: bool, device="cuda"):
        from . import ops
        if head_width not in (64, 80):
            raise ValueError(f"head width {head_width}: the attention kernels cover 64 and 80")
        dev = torch.device(device)
        f16 = lambda t: t.detach().to(dev, torch.float16).contiguous()   # noqa: E731
        f32 = lambda t: t.detach().to(dev, torch.float32).contiguous()   # noqa: E731
        w1 = sd["conv1.weight"]
        self.width, _, self.patch, _ = w1.shape
        self.tokens = sd["positional_embedding"].shape[0]
        self.grid = int(round((self.tokens - 1) ** 0.5))
        if self.grid * self.grid + 1 != self.tokens:
            raise ValueError(f"positional_embedding of {self.tokens} rows is not a square grid plus a class token")
        self.layers = len({int(m.group(1)) for k in sd for m in [re.match(r"transformer\.resblocks\.(\d+)\.", k)] if m})
        self.out_dim = sd["proj"].shape[1]
        self.mlp = sd["transformer.resblocks.0.mlp.c_fc.weight"].shape[0]
        self.head_width = head_width
        self.heads = self.width // head_width
        if self.heads * head_width != self.width or self.width % 64 or self.mlp % 64:
            raise ValueError(f"width {self.width} / MLP {self.mlp} / head width {head_width}: need width = heads x head width "
                             f"and multiples of 64")
        self.act = ops.ACT_QUICKGELU if quick_gelu else ops.ACT_GELU
        self.device = dev
        k = 3 * self.patch * self.patch
        self.kpad = (k + 63) // 64 * 64
        wp = torch.zeros(self.width, self.kpad, dtype=torch.float32)
        wp[:, :k] = w1.detach().float().reshape(self.width, k).cpu()
        self.w_patch = f16(wp)
        pos = sd["positional_embedding"].detach().float().clone().cpu()
        pos[0] += sd["class_embedding"].detach().float().cpu()     # the class token enters through row 0 of the addvec
        self.addvec = f16(pos)
        self.ln_pre = (f32(sd["ln_pre.weight"]), f32(sd["ln_pre.bias"]))
        self.blocks = []
        for i in range(self.layers):
            p = f"transformer.resblocks.{i}."
            self.blocks.append(dict(
                ln_1=(f32(sd[p + "ln_1.weight"]), f32(sd[p + "ln_1.bias"])),
                in_w=f16(sd[p + "attn.in_proj_weight"]), in_b=f32(sd[p + "attn.in_proj_bias"]),
                out_w=f16(sd[p + "attn.out_proj.weight"]), out_b=f32(sd[p + "attn.out_proj.bias"]),
                ln_2=(f32(sd[p + "ln_2.weight"]), f32(sd[p + "ln_2.bias"])),
                fc_w=f16(sd[p + "mlp.c_fc.weight"]), fc_b=f32(sd[p + "mlp.c_fc.bias"]),
                pr_w=f16(sd[p + "mlp.c_proj.weight"]), pr_b=f32(sd[p + "mlp.c_proj.bias"])))
        self.ln_post = (f32(sd["ln_post.weight"]), f32(sd["ln_post.bias"]))
        self.w_proj = f16(sd["proj"].t())                          # x @ proj == x @ (proj^T)^T
        self.flops_per_image = 2.0 * self.tokens * (self.kpad * self.width + self.layers * (
            4 * self.width * self.width + 2 * self.width * self.mlp + 2 * self.tokens * self.width)) + 2.0 * self.width * self.out_dim

    @torch.no_grad()
    def __call__(self, img: torch.Tensor, normalize: bool = True) -> torch.Tensor:
        """img: (n, 3, 224, 224) fp32 / fp16 in [0, 1] (normalize=True: the CLIP mean / std is applied by the patch kernel) or
        already normalised (normalize=False).  Returns the image embedding (n, out_dim) fp32."""
        from . import ops
        if img.dim() != 4 or img.shape[1] != 3 or img.shape[-1] != self.grid * self.patch or img.shape[-2] != self.grid * self.patch:
            raise ValueError(f"expected (n, 3, {self.grid * self.patch}, {self.grid * self.patch}) images, got {tuple(img.shape)}")
        img = img.to(self.device)
        if img.dtype not in (torch.float32, torch.float16):
            img = img.float()
        img = img.contiguous()
        n, L, Wd = img.shape[0], self.tokens, self.width
        M = n * L
        e = lambda *s: torch.empty(*s, dtype=torch.float16, device=self.device)   # noqa: E731
        rows = e(M, self.kpad)
        ops.clip_patchify(img, self.patch, rows, normalize=normalize)
        tok = e(M, Wd)
        ops.Gemm([ops.SegSpec(rows)], self.w_patch, tok, M, engine="tc5")()
        x, br, h, a = e(M, Wd), e(M, Wd), e(M, Wd), e(M, Wd)
        ops.layernorm(tok, *self.ln_pre, x, M, addvec=self.addvec, add_div=1, add_mod=L)
        x32 = x.float()                    # the residual stream, fp32; x = its fp16 copy that feeds the LayerNorms
        qkv, mid = e(M, 3 * Wd), e(M, self.mlp)
        scale = self.head_width ** -0.5
        for b in self.blocks:
            ops.layernorm(x, *b["ln_1"], h, M)
            ops.Gemm([ops.SegSpec(h)], b["in_w"], qkv, M, bias=b["in_b"], engine="tc5")()
            if self.head_width == 80:
                ops.attention_d80(qkv, n, L, self.heads, a, scale)
            else:
                ops.attention_d64(qkv, n, L, self.heads, a, scale, engine="tc5")
            ops.Gemm([ops.SegSpec(a)], b["out_w"], br, M, bias=b["out_b"], engine="tc5")()
            x32 += br
            x.copy_(x32)
            ops.layernorm(x, *b["ln_2"], h, M)
            ops.Gemm([ops.SegSpec(h)], b["fc_w"], mid, M, bias=b["fc_b"], act=self.act, engine="tc5")()
            ops.Gemm([ops.SegSpec(mid)], b["pr_w"], br, M, bias=b["pr_b"], engine="tc5")()
            x32 += br
            x.copy_(x32)
        cls = x.view(n, L, Wd)[:, 0].contiguous()
        cls_n = e(n, Wd)
        ops.layernorm(cls, *self.ln_post, cls_n, n)
        out = e(n, self.out_dim)
        ops.Gemm([ops.SegSpec(cls_n)], self.w_proj, out, n, engine="tc5")()
        return out.float()


class AestheticScorer:
    """AesEmbedder's scorer (vtdm/encoders.py:80-86): OpenAI CLIP ViT-L/14 image features -> L2 normalisation -> the aesthetic
    MLP, folded at load time into one affine map.  Input: images already normalised by AesEmbedder.preprocess."""

    def __init__(self, visual_sd: Dict[str, torch.Tensor], mlp_w: torch.Tensor, mlp_b: torch.Tensor, device="cuda"):
        self.tower = ClipVisionTower(visual_sd, OPENAI_HEAD_WIDTH, quick_gelu=True, device=device)
        self.w = mlp_w.to(self.tower.device, torch.float32)
        self.b = mlp_b.to(self.tower.device, torch.float32)

    @torch.no_grad()
    def __call__(self, x: torch.Tensor) -> torch.Tensor:
        f = self.tower(x, normalize=False)
        f = f / f.norm(dim=-1, keepdim=True).clamp_min(1e-30)         # aes_score.normalized (a zero norm stays zero)
        return (f @ self.w + self.b)[:, None]


def open_clip_file(version: Optional[str]) -> Optional[str]:
    return version if isinstance(version, str) and os.path.isfile(version) else None
