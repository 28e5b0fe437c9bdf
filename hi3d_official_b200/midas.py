"""MiDaS DPT-Hybrid depth tower of the stage-2 conditioner on this package's kernels (SURVEY §8f N2): the reference's
`MiDaSInference(model_type="dpt_hybrid")` (annotator/midas/api.py:146-165), i.e. `DPTDepthModel(backbone="vitb_rn50_384",
readout="project", non_negative=True, features=256)` over timm's `vit_base_resnet50_384`.  DepthEmbedder (vtdm/encoders.py:15-53)
feeds it (16, 3, sH, sW) frames in [-1, 1] and turns the (16, sH, sW) inverse depth into the 9 depth channels of `concat`.

Per call, everything channels-last fp16 with fp32 accumulation, every conv / linear one hi3d_gemm_tc5:

  BiT ResNet-50 trunk   hi3d_dpt_stem_rows -> stem GEMM -> its GroupNorm statistics -> hi3d_groupnorm_apply_add
                        (GN + ReLU) -> hi3d_maxpool3x3s2_same; per bottleneck conv1 / conv2 / conv3 GEMMs (the weights are
                        standardised once at load) with GN + ReLU applies in between, and one hi3d_groupnorm_apply_add for
                        relu(GN3(conv3) + shortcut), the shortcut being x or GN(downsample conv) of the same pass
  ViT-B/16              patch-embedding GEMM over the trunk's /16 map written with one zero row per image, so the class token and
                        the positional embedding enter through the epilogue's `rowbias`; then pre-LN blocks: hi3d_layernorm,
                        qkv GEMM, hi3d_attention_d64_tc5, proj GEMM + residual, fc1 GEMM (GELU), fc2 GEMM + residual
  reassemble 3 / 4      ProjectReadout as W[:, :C] token + (W[:, C:] cls + b): the cls term is a per-image `rowbias`, and the
                        token GEMM reads rows 1..P of each image as frames 1..P of a (1 + P)-frame clip (temporal row mode with a
                        frame offset), which also drops the class rows from the output; 1x1 conv GEMM [+ 3x3 stride-2 GEMM]
  neck / head           layerN_rn GEMMs; per fusion block hi3d_relu_copy + two conv GEMMs (ReLU epilogue, residual epilogue) per
                        residual conv unit, out_conv at the LOW resolution (a 1x1 conv commutes with the bilinear x2, whose
                        weights sum to one), then hi3d_upsample2x_bilinear_ac, which also adds the next block's resConfUnit1
                        output; head convs with the ReLU epilogue, the 32 channels stored into a 64-wide zero-padded buffer.

The ViT's residual stream is the fp16 residual epilogue of the proj / fc2 GEMMs.  Widths and depths are read from the tensor
shapes (reduced widths work when every channel count is a multiple of 64); the ViT must have at least 12 blocks, since DPT taps
blocks 8 and 11.
"""
from __future__ import annotations

import math
import re
from typing import Dict, List, Optional, Set

import torch
import torch.nn.functional as F

BB = "pretrained.model.patch_embed.backbone."
VIT = "pretrained.model."
HOOKS = (8, 11)
# in the reference's state dict but unused by its forward: ViT's final norm and classifier, and refinenet4's first unit
DEAD_PREFIXES = (VIT + "norm.", VIT + "head.", "scratch.refinenet4.resConfUnit1.")


def _indices(keys, prefix: str) -> List[int]:
    return sorted({int(m.group(1)) for k in keys for m in [re.match(re.escape(prefix) + r"(\d+)\.", k)] if m})


def dead_keys(sd) -> Set[str]:
    return {k for k in sd if k.startswith(DEAD_PREFIXES)}


def expected_keys(sd) -> Set[str]:
    """Every tensor the forward uses, for the stage / block / ViT-block counts found in `sd`."""
    wb = lambda p: {p + "weight", p + "bias"}   # noqa: E731
    keys = {BB + "stem.conv.weight"} | wb(BB + "stem.norm.")
    stages = _indices(sd, BB + "stages.")
    if stages != [0, 1, 2]:
        raise KeyError(f"DPT-Hybrid: expected BiT stages 0..2, found {stages}")
    for s in stages:
        blocks = _indices(sd, BB + f"stages.{s}.blocks.")
        if not blocks or blocks != list(range(len(blocks))):
            raise KeyError(f"DPT-Hybrid: BiT stage {s} blocks {blocks}")
        for b in blocks:
            p = BB + f"stages.{s}.blocks.{b}."
            keys |= {p + f"conv{i}.weight" for i in (1, 2, 3)} | wb(p + "norm1.") | wb(p + "norm2.") | wb(p + "norm3.")
            if b == 0:
                keys |= {p + "downsample.conv.weight"} | wb(p + "downsample.norm.")
    blocks = _indices(sd, VIT + "blocks.")
    if len(blocks) <= max(HOOKS) or blocks != list(range(len(blocks))):
        raise KeyError(f"DPT-Hybrid: ViT blocks {blocks}; blocks 0..{max(HOOKS)} are needed")
    keys |= wb(VIT + "patch_embed.proj.") | {VIT + "cls_token", VIT + "pos_embed"}
    for i in blocks:
        p = VIT + f"blocks.{i}."
        for m in ("norm1.", "attn.qkv.", "attn.proj.", "norm2.", "mlp.fc1.", "mlp.fc2."):
            keys |= wb(p + m)
    for idx in (3, 4):
        p = f"pretrained.act_postprocess{idx}."
        keys |= wb(p + "0.project.0.") | wb(p + "3.") | (wb(p + "4.") if idx == 4 else set())
    keys |= {f"scratch.layer{i}_rn.weight" for i in (1, 2, 3, 4)}
    for i in (1, 2, 3, 4):
        p = f"scratch.refinenet{i}."
        units = ("resConfUnit2.",) if i == 4 else ("resConfUnit1.", "resConfUnit2.")
        for u in units:
            keys |= wb(p + u + "conv1.") | wb(p + u + "conv2.")
        keys |= wb(p + "out_conv.")
    for i in (0, 2, 4):
        keys |= wb(f"scratch.output_conv.{i}.")
    return keys


def live_state_dict(sd: Dict[str, torch.Tensor], strict: bool = True) -> Dict[str, torch.Tensor]:
    """The tensors the forward uses.  Raises KeyError on a missing one and, with `strict`, on a key that is neither used nor one
    of the dead ones (a file of another model or with another prefix)."""
    want = expected_keys(sd)
    missing = sorted(want - set(sd))
    if missing:
        raise KeyError(f"DPT-Hybrid state dict: {len(missing)} missing tensors, e.g. {missing[:4]}")
    if strict:
        unexpected = sorted(set(sd) - want - dead_keys(sd))
        if unexpected:
            raise KeyError(f"DPT-Hybrid state dict: {len(unexpected)} unexpected tensors, e.g. {unexpected[:4]}")
    return {k: sd[k] for k in want}


def load_dpt_hybrid(path: str) -> Dict[str, torch.Tensor]:
    """The reference's ckpts/dpt_hybrid_384.pt (annotator/midas/base_model.py:6-17): a state dict, or a training checkpoint
    {'model': state dict, 'optimizer': ...}.  Returns the live tensors (CPU)."""
    sd = torch.load(path, map_location="cpu", weights_only=True)
    if isinstance(sd, dict) and "optimizer" in sd:
        sd = sd["model"]
    return live_state_dict(sd)


def resize_pos_embed(pos: torch.Tensor, gh: int, gw: int) -> torch.Tensor:
    """vit.py:104-121 on a (1 + g*g, C) positional embedding: the grid rows resized bilinearly (align_corners=False) to gh x gw,
    the class row kept."""
    g = int(math.sqrt(pos.shape[0] - 1))
    if (gh, gw) == (g, g):
        return pos
    grid = pos[1:].reshape(1, g, g, -1).permute(0, 3, 1, 2)
    grid = F.interpolate(grid, size=(gh, gw), mode="bilinear")
    return torch.cat([pos[:1], grid.permute(0, 2, 3, 1).reshape(gh * gw, -1)], 0)


def _std_weight(w: torch.Tensor, eps: float = 1e-8) -> torch.Tensor:
    """timm StdConv2dSame: per output channel (w - mean) / sqrt(biased var + eps), folded once since the weights are frozen."""
    w = w.double()
    m = w.mean(dim=(1, 2, 3), keepdim=True)
    v = w.var(dim=(1, 2, 3), unbiased=False, keepdim=True)
    return ((w - m) / torch.sqrt(v + eps)).float()


def _gemm_weight(w: torch.Tensor) -> torch.Tensor:
    """Conv OIHW -> [Co, kh * kw * Ci], K ordered (tap, ci) like ops.conv_taps; a Linear [Co, Ci] is kept."""
    return w.permute(0, 2, 3, 1).reshape(w.shape[0], -1) if w.dim() == 4 else w


class DPTHybridTower:
    """DPT-Hybrid on the hi3d kernels.  `sd`: the reference's state dict (CPU or CUDA, any float dtype); the packed weights live
    on `device` (fp16 matrices, fp32 biases and normalisation parameters).  Raises KeyError when a tensor is missing."""

    def __init__(self, sd: Dict[str, torch.Tensor], device="cuda"):
        sd = live_state_dict(sd, strict=False)
        dev = torch.device(device)
        self.device = dev
        f16 = lambda t: t.detach().to(dev, torch.float16).contiguous()   # noqa: E731
        f32 = lambda t: t.detach().to(dev, torch.float32).contiguous()   # noqa: E731
        W = lambda k: f16(_gemm_weight(sd[k].detach().float().cpu()))    # noqa: E731
        Wstd = lambda k: f16(_gemm_weight(_std_weight(sd[k].detach().cpu())))   # noqa: E731
        norm = lambda p: (f32(sd[p + "weight"]), f32(sd[p + "bias"]))    # noqa: E731
        wb = lambda p: (W(p + "weight"), f32(sd[p + "bias"]))             # noqa: E731

        stem = _std_weight(sd[BB + "stem.conv.weight"].detach().cpu())
        self.stem_width = stem.shape[0]
        self.kpad = 192                                                  # 3 * 7 * 7 = 147 -> a multiple of 64
        ws = torch.zeros(self.stem_width, self.kpad)
        ws[:, :147] = stem.reshape(self.stem_width, 147)
        self.w_stem, self.stem_norm = f16(ws), norm(BB + "stem.norm.")
        self.stages = []
        for s in range(3):
            blocks = []
            for b in _indices(sd, BB + f"stages.{s}.blocks."):
                p = BB + f"stages.{s}.blocks.{b}."
                blk = dict(w1=Wstd(p + "conv1.weight"), n1=norm(p + "norm1."), w2=Wstd(p + "conv2.weight"), n2=norm(p + "norm2."),
                           w3=Wstd(p + "conv3.weight"), n3=norm(p + "norm3."), stride=2 if (b == 0 and s > 0) else 1)
                if b == 0:
                    blk.update(wd=Wstd(p + "downsample.conv.weight"), nd=norm(p + "downsample.norm."))
                blocks.append(blk)
            self.stages.append(blocks)
        self.w_pe, self.b_pe = wb(VIT + "patch_embed.proj.")
        self.width = self.w_pe.shape[0]
        self.heads = self.width // 64
        self.trunk_width = self.w_pe.shape[1]
        self.cls = sd[VIT + "cls_token"].detach().float().cpu().reshape(-1)
        self.pos = sd[VIT + "pos_embed"].detach().float().cpu().reshape(-1, self.width)
        self._posadj = {}
        self.blocks = []
        for i in _indices(sd, VIT + "blocks."):
            p = VIT + f"blocks.{i}."
            self.blocks.append(dict(ln1=norm(p + "norm1."), qkv=wb(p + "attn.qkv."), proj=wb(p + "attn.proj."), ln2=norm(p + "norm2."),
                                    fc1=wb(p + "mlp.fc1."), fc2=wb(p + "mlp.fc2.")))
        self.reassemble = {}
        for idx in (3, 4):
            p = f"pretrained.act_postprocess{idx}."
            w = sd[p + "0.project.0.weight"].detach().float()
            r = dict(w_tok=f16(w[:, :self.width]), w_cls=f16(w[:, self.width:]), b_ro=f32(sd[p + "0.project.0.bias"]), post=wb(p + "3."))
            if idx == 4:
                r["resize"] = wb(p + "4.")
            self.reassemble[idx] = r
        self.rn = [W(f"scratch.layer{i}_rn.weight") for i in (1, 2, 3, 4)]
        self.features = self.rn[0].shape[0]
        self.fusion = {}
        for i in (1, 2, 3, 4):
            p = f"scratch.refinenet{i}."
            units = {u: (wb(p + u + "conv1."), wb(p + u + "conv2.")) for u in ("resConfUnit1.", "resConfUnit2.") if i < 4 or u[-2] == "2"}
            self.fusion[i] = dict(units=units, out=wb(p + "out_conv."))
        self.oc0, self.oc2 = wb("scratch.output_conv.0."), wb("scratch.output_conv.2.")
        self.head_mid = self.oc2[0].shape[0]                             # 32: stored into a zero-padded buffer of 64 columns
        w4 = torch.zeros(8, 64)
        w4[0, :self.head_mid] = sd["scratch.output_conv.4.weight"].detach().float().cpu().reshape(-1)
        b4 = torch.zeros(8)
        b4[0] = float(sd["scratch.output_conv.4.bias"].reshape(-1)[0])
        self.oc4 = (f16(w4), f32(b4))
        for name, c in (("stem", self.stem_width), ("trunk", self.trunk_width), ("width", self.width), ("features", self.features),
                        ("head", self.oc0[0].shape[0])):
            if c % 64:
                raise ValueError(f"DPT-Hybrid: {name} width {c} is not a multiple of 64")
        if self.head_mid > 64:
            raise ValueError(f"DPT-Hybrid: head width {self.head_mid} > 64")

    def posadj(self, gh: int, gw: int) -> torch.Tensor:
        """rowbias of the patch-embedding GEMM for a gh x gw grid, cached: row 0 = cls_token + pos[0] - bias (the zero class row
        of the A operand plus the bias gives cls_token + pos[0]), rows 1.. = the resized positional embedding."""
        if (gh, gw) not in self._posadj:
            pos = resize_pos_embed(self.pos, gh, gw).clone()
            pos[0] += self.cls - self.b_pe.float().cpu()
            self._posadj[(gh, gw)] = pos.to(self.device, torch.float16).contiguous()
        return self._posadj[(gh, gw)]

    @torch.no_grad()
    def __call__(self, img: torch.Tensor) -> torch.Tensor:
        """img: (n, 3, H, W) fp32 / fp16 with H, W multiples of 32 (no normalisation is applied).  Returns (n, H, W) fp32."""
        from . import ops
        if img.dim() != 4 or img.shape[1] != 3 or img.shape[2] % 32 or img.shape[3] % 32 or img.shape[2] == 0 or img.shape[3] == 0:
            raise ValueError(f"expected (n, 3, 32a, 32b) images, got {tuple(img.shape)}")
        img = img.to(self.device)
        if img.dtype not in (torch.float32, torch.float16):
            img = img.float()
        img = img.contiguous()
        n, _, H, W = img.shape
        dev = self.device
        e = lambda *s: torch.empty(*s, dtype=torch.float16, device=dev)   # noqa: E731
        n_stats = 1 + sum(3 * len(s) + 1 for s in self.stages)
        stats_all = torch.zeros(n_stats, n * 64, dtype=torch.float32, device=dev)
        stats_iter = iter(stats_all)

        def gemm(segs, w, out, M, mode=ops.ROWS_PLAIN, geom=None, gn_rows=0, **kw):
            """gn_rows > 0: also the GroupNorm unit table of `out` (images of gn_rows rows), which is returned."""
            ops.Gemm(segs, w, out, M, mode=mode, geom=geom, engine="tc5", **kw)()
            if not gn_rows:
                return None
            st = next(stats_iter)
            ops.groupnorm_unit_stats(out, M // gn_rows, gn_rows, w.shape[0] // 32, st)
            return st

        def conv3(x, w, h, wd, out, stride=1, pad_lo=1, **kw):
            ho, wo = h // stride, wd // stride
            return gemm(ops.conv_taps([x], pad_lo=pad_lo), w, out, n * ho * wo, mode=ops.ROWS_CONV2D,
                        geom=dict(Ho=ho, Wo=wo, Hs=h, Ws=wd, stride=stride), **kw)

        def gn_apply(x, st, nrm, y, **kw):
            ops.groupnorm_apply_add(x, st, nrm[0], nrm[1], x.shape[-1] // 32, n, y, **kw)
            return y

        # ---- BiT trunk ----
        h, w = (H + 1) // 2, (W + 1) // 2
        rows = e(n * h * w, self.kpad)
        ops.dpt_stem_rows(img, rows)
        s0 = e(n * h * w, self.stem_width)
        st = gemm([ops.SegSpec(rows)], self.w_stem, s0, n * h * w, gn_rows=h * w)
        a0 = gn_apply(s0, st, self.stem_norm, e(n * h * w, self.stem_width), relu=True)
        x = e(n * ((h + 1) // 2) * ((w + 1) // 2), self.stem_width)
        ops.maxpool3x3s2_same(a0, n, h, w, x)
        h, w = (h + 1) // 2, (w + 1) // 2
        feats = []
        gh, gw = H // 16, W // 16
        P = gh * gw
        L = 1 + P
        tokens_in = torch.zeros(n * L, self.trunk_width, dtype=torch.float16, device=dev)   # one zero class row per image
        for si, blocks in enumerate(self.stages):
            for bi, b in enumerate(blocks):
                s = b["stride"]
                ho, wo = h // s, w // s
                mid, cout = b["w1"].shape[0], b["w3"].shape[0]
                c1 = e(n * h * w, mid)
                st1 = gemm([ops.SegSpec(x)], b["w1"], c1, n * h * w, gn_rows=h * w)
                a1 = gn_apply(c1, st1, b["n1"], e(n * h * w, mid), relu=True)
                c2 = e(n * ho * wo, mid)
                st2 = conv3(a1, b["w2"], h, w, c2, stride=s, pad_lo=1 if s == 1 else 0, gn_rows=ho * wo)   # "same": pad (0, 1) at s = 2
                a2 = gn_apply(c2, st2, b["n2"], e(n * ho * wo, mid), relu=True)
                c3 = e(n * ho * wo, cout)
                st3 = gemm([ops.SegSpec(a2)], b["w3"], c3, n * ho * wo, gn_rows=ho * wo)
                add = dict(add=x)
                if "wd" in b:
                    d = e(n * ho * wo, cout)
                    if s == 1:
                        std_ = gemm([ops.SegSpec(x)], b["wd"], d, n * ho * wo, gn_rows=ho * wo)
                    else:
                        std_ = gemm([ops.SegSpec(x)], b["wd"], d, n * ho * wo, mode=ops.ROWS_CONV2D,
                                    geom=dict(Ho=ho, Wo=wo, Hs=h, Ws=w, stride=s), gn_rows=ho * wo)
                    add = dict(add=d, add_stats=std_, add_gamma=b["nd"][0], add_beta=b["nd"][1])
                last = si == len(self.stages) - 1 and bi == len(blocks) - 1
                if last:
                    if (ho, wo) != (gh, gw):
                        raise ValueError(f"BiT output grid {ho} x {wo} != {gh} x {gw}")
                    x = gn_apply(c3, st3, b["n3"], tokens_in, relu=True, y_sample_rows=L, y_row_off=1, **add)
                else:
                    x = gn_apply(c3, st3, b["n3"], e(n * ho * wo, cout), relu=True, **add)
                h, w = ho, wo
            feats.append(x)

        # ---- ViT-B/16 ----
        C_ = self.width
        M = n * L
        x = e(M, C_)
        gemm([ops.SegSpec(tokens_in)], self.w_pe, x, M, bias=self.b_pe, rowbias=self.posadj(gh, gw), rb_div=1, rb_mod=L)
        hbuf, qkv, att = e(M, C_), e(M, 3 * C_), e(M, C_)
        mlp = e(M, self.blocks[0]["fc1"][0].shape[0])
        taps = {}
        for i, b in enumerate(self.blocks[:max(HOOKS) + 1]):
            ops.layernorm(x, *b["ln1"], hbuf, M, eps=1e-6)
            gemm([ops.SegSpec(hbuf)], b["qkv"][0], qkv, M, bias=b["qkv"][1])
            ops.attention_d64(qkv, n, L, self.heads, att, scale=0.125, engine="tc5")
            x1 = e(M, C_)
            gemm([ops.SegSpec(att)], b["proj"][0], x1, M, bias=b["proj"][1], residual=x)
            ops.layernorm(x1, *b["ln2"], hbuf, M, eps=1e-6)
            gemm([ops.SegSpec(hbuf)], b["fc1"][0], mlp, M, bias=b["fc1"][1], act=ops.ACT_GELU)
            x = e(M, C_)
            gemm([ops.SegSpec(mlp)], b["fc2"][0], x, M, bias=b["fc2"][1], residual=x1)
            if i in HOOKS:
                taps[i] = x

        # ---- reassemble: layer_3 (/16) and layer_4 (/32) ----
        for idx, blk in zip((3, 4), HOOKS):
            r = self.reassemble[idx]
            X = taps[blk]
            rb = e(n, C_)
            gemm([ops.SegSpec(X, C_=C_, ld=L * C_)], r["w_cls"], rb, n, bias=r["b_ro"])          # row b = class row of image b
            ro = e(n * P, C_)
            gemm([ops.SegSpec(X)], r["w_tok"], ro, n * P, mode=ops.ROWS_TEMPORAL,
                 geom=dict(Ho=1, Wo=1, T=P, Tin=L, t_off=1), rowbias=rb, rb_div=P, rb_mod=n, act=ops.ACT_GELU)
            pc = e(n * P, C_)
            gemm([ops.SegSpec(ro)], r["post"][0], pc, n * P, bias=r["post"][1])
            if idx == 4:
                p4 = e(n * (gh // 2) * (gw // 2), C_)
                conv3(pc, r["resize"][0], gh, gw, p4, stride=2, pad_lo=1, bias=r["resize"][1])
                pc = p4
            feats.append(pc)
        layers = [feats[0], feats[1], feats[3], feats[4]]
        grids = [(H // 4, W // 4), (H // 8, W // 8), (gh, gw), (gh // 2, gw // 2)]

        # ---- neck ----
        Fc = self.features
        rn = []
        for i in range(4):
            gy, gx = grids[i]
            t = e(n * gy * gx, Fc)
            conv3(layers[i], self.rn[i], gy, gx, t)
            rn.append(t)

        def rcu(xx, unit, gy, gx):
            (w1, b1), (w2, b2) = unit
            r_ = e(*xx.shape)
            ops.relu_copy(xx, r_)
            c = e(*xx.shape)
            conv3(r_, w1, gy, gx, c, bias=b1, act=ops.ACT_RELU)
            o = e(*xx.shape)
            conv3(c, w2, gy, gx, o, bias=b2, residual=xx)
            return o

        o = None
        for i in (4, 3, 2, 1):
            gy, gx = grids[i - 1]
            fb = self.fusion[i]
            if o is None:
                s_ = rn[3]
            else:
                t = rcu(rn[i - 1], fb["units"]["resConfUnit1."], gy, gx)
                s_ = e(n * gy * gx, Fc)
                ops.upsample2x_bilinear_ac(o, n, gy // 2, gx // 2, s_, add=t)
            u = rcu(s_, fb["units"]["resConfUnit2."], gy, gx)
            o = e(n * gy * gx, Fc)
            gemm([ops.SegSpec(u)], fb["out"][0], o, n * gy * gx, bias=fb["out"][1])
        gy, gx = grids[0]
        path = e(n * 4 * gy * gx, Fc)
        ops.upsample2x_bilinear_ac(o, n, gy, gx, path)
        gy, gx = 2 * gy, 2 * gx

        # ---- head ----
        h0 = e(n * gy * gx, self.oc0[0].shape[0])
        conv3(path, self.oc0[0], gy, gx, h0, bias=self.oc0[1])
        h1 = e(n * 4 * gy * gx, h0.shape[1])
        ops.upsample2x_bilinear_ac(h0, n, gy, gx, h1)
        gy, gx = 2 * gy, 2 * gx
        h2 = torch.zeros(n * gy * gx, 64, dtype=torch.float16, device=dev)
        conv3(h1, self.oc2[0], gy, gx, h2, bias=self.oc2[1], act=ops.ACT_RELU)
        d = e(n * gy * gx, 8)
        gemm([ops.SegSpec(h2)], self.oc4[0], d, n * gy * gx, bias=self.oc4[1], act=ops.ACT_RELU)
        out = torch.empty(n, 1, gy, gx, dtype=torch.float32, device=dev)
        ops.nhwc_to_nchw(d, out)
        return out.view(n, gy, gx)
