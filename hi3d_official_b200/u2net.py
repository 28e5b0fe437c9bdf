"""U^2-Net (Qin et al. 2020, U-2-Net `model/u2net.py`) on this package's kernels: the salient-object network behind rembg's default
`remove`, which the reference's stage 1 uses to cut the input image out of its background (pipeline_i2v_eval_v01.py:153-168).

Graph.  REBNCONV(in, out, d) = relu(BN(conv3x3(x, padding=d, dilation=d))).  RSU-L (L = 7, 6, 5, 4) is a small U-Net of
REBNCONVs: rebnconvin (in -> out), rebnconv1 (out -> mid), then rebnconv2 .. rebnconv(L-1) each after a ceil-mode 2x2 max-pool,
the bottom rebnconvL with dilation 2 and no pool, and the decoder rebnconv{k}d on cat(up(hx(k+1)d), hxk) for k = L-1 .. 1 (the
first on cat(hxL, hx(L-1))); it returns hx1d + hxin.  RSU4F has no pools: dilations 1, 2, 4, 8 down and 4, 2, 1 up.  U2NET
chains six encoder stages and five decoder stages the same way; side heads (3x3 conv to one channel) on hx1d .. hx5d and hx6
are upsampled to the input size and mixed by `outconv` (1x1, 6 -> 1); output 0 = sigmoid(d0) is what rembg uses.

Per call, everything channels-last fp16 with fp32 accumulation:
  every REBNCONV        one hi3d_gemm_tc5 (BatchNorm folded into the conv at load, ReLU epilogue; rebnconv1d adds hxin through
                        the residual epilogue, which comes after the activation), dilated taps as segment offsets
  every `cat`           free: a level's decoder concat buffer is allocated once; the encoder conv stores hxk into its upper
                        channel slice and hi3d_resize_bilinear stores the upsampled decoder output into the lower one
  pools                 hi3d_maxpool2x2_ceil, reading the channel slice
  side heads + outconv  outconv's weights are folded into the side heads (bilinear weights sum to one), so the five resizes,
                        the concat and the 1x1 conv are one hi3d_u2net_fuse_sides pass that also applies the sigmoid

The buffers and the launches of a call (118 GEMMs: 112 REBNCONVs and 6 side heads; outconv has none) are built once per input
shape, with every GEMM parameter block pre-baked, and reused while the shape stays the same (rembg always runs 1 x 320^2), so a
call costs the launches, the input conversion and a copy of the output on the host side.

A GEMM segment spans a multiple of 64 channels.  A tensor of fewer live channels (the mid widths 32 and 16, the 3-channel image)
is read as a 64-channel window whose other channels are zero, with zero weight columns there; such buffers are zero-filled when
allocated, and their padding channels are never written.  Widths are read from the tensor shapes, so U2NET and U2NETP (every
mid 16, every out 64) both load.
"""
from __future__ import annotations

import functools
from typing import Dict, List, Sequence, Tuple

import torch

BN_EPS = 1e-5
# stage -> RSU depth L (4 with `pooled` False is RSU4F)
STAGES = (("stage1", 7, True), ("stage2", 6, True), ("stage3", 5, True), ("stage4", 4, True), ("stage5", 4, False),
          ("stage6", 4, False), ("stage5d", 4, False), ("stage4d", 4, True), ("stage3d", 5, True), ("stage2d", 6, True),
          ("stage1d", 7, True))
STAGE_KIND = {s: (L, pooled) for s, L, pooled in STAGES}
BN_PARAMS = ("weight", "bias", "running_mean", "running_var")


def rsu_convs(L: int, pooled: bool) -> List[Tuple[str, int]]:
    """(name, dilation) of the REBNCONVs of an RSU-L (pooled) or RSU4F, in forward order."""
    if pooled:
        enc = [("rebnconvin", 1)] + [(f"rebnconv{k}", 1) for k in range(1, L)] + [(f"rebnconv{L}", 2)]
        return enc + [(f"rebnconv{k}d", 1) for k in range(L - 1, 0, -1)]
    return [("rebnconvin", 1), ("rebnconv1", 1), ("rebnconv2", 2), ("rebnconv3", 4), ("rebnconv4", 8), ("rebnconv3d", 4),
            ("rebnconv2d", 2), ("rebnconv1d", 1)]


def expected_keys() -> set:
    keys = set()
    for stage, L, pooled in STAGES:
        for name, _ in rsu_convs(L, pooled):
            p = f"{stage}.{name}."
            keys |= {p + "conv_s1.weight", p + "conv_s1.bias"} | {p + "bn_s1." + b for b in BN_PARAMS}
    for k in range(1, 7):
        keys |= {f"side{k}.weight", f"side{k}.bias"}
    return keys | {"outconv.weight", "outconv.bias"}


def live_state_dict(sd: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """The tensors the forward uses, from a U-2-Net state dict: a `module.` prefix (DataParallel) is stripped and BatchNorm's
    `num_batches_tracked` ignored.  Raises KeyError on a missing tensor or an unexpected one."""
    sd = {(k[len("module."):] if k.startswith("module.") else k): v for k, v in sd.items()}
    sd = {k: v for k, v in sd.items() if not k.endswith(".num_batches_tracked")}
    want = expected_keys()
    missing = sorted(want - set(sd))
    if missing:
        raise KeyError(f"U^2-Net state dict: {len(missing)} missing tensors, e.g. {missing[:4]}")
    unexpected = sorted(set(sd) - want)
    if unexpected:
        raise KeyError(f"U^2-Net state dict: {len(unexpected)} unexpected tensors, e.g. {unexpected[:4]}")
    return sd


def load_u2net(path: str) -> Dict[str, torch.Tensor]:
    """U-2-Net's released `u2net.pth` / `u2netp.pth` (a state dict).  Returns the live tensors (CPU)."""
    return live_state_dict(torch.load(path, map_location="cpu", weights_only=True))


def fold(sd: Dict[str, torch.Tensor]) -> dict:
    """Load-time algebra in fp64 (CPU): every REBNCONV with its eval BatchNorm folded in, w * g / sqrt(var + eps) and
    (b - mean) * g / sqrt(var + eps) + beta, keyed 'stage.name' -> (w, b, dilation); the side heads scaled by their outconv
    weight, 'sides' -> [(w_k, b_k)] for k = 1..6; and outconv's bias 'b0'.  Then d0 = b0 + sum_k up(side_k'(h_k))."""
    d = lambda k: sd[k].detach().to("cpu", torch.float64)   # noqa: E731
    out = {}
    for stage, L, pooled in STAGES:
        for name, dil in rsu_convs(L, pooled):
            p = f"{stage}.{name}."
            s = d(p + "bn_s1.weight") / torch.sqrt(d(p + "bn_s1.running_var") + BN_EPS)
            w = d(p + "conv_s1.weight") * s[:, None, None, None]
            b = (d(p + "conv_s1.bias") - d(p + "bn_s1.running_mean")) * s + d(p + "bn_s1.bias")
            out[f"{stage}.{name}"] = (w, b, dil)
    wo = d("outconv.weight").reshape(-1)
    if wo.numel() != 6:
        raise KeyError(f"U^2-Net outconv: expected 6 inputs, got {wo.numel()}")
    out["sides"] = [(d(f"side{k}.weight") * wo[k - 1], d(f"side{k}.bias") * wo[k - 1]) for k in range(1, 7)]
    out["b0"] = float(d("outconv.bias").reshape(-1)[0])
    return out


def _pad64(c: int) -> int:
    return (c + 63) // 64 * 64


class U2NetTower:
    """U^2-Net on the hi3d kernels.  `sd`: a U-2-Net state dict (CPU or CUDA, any float dtype; U2NET or U2NETP widths).
    Raises KeyError when a tensor is missing or unexpected.  Call: fp32 (n, 3, H, W), already normalised, any H, W ->
    fp32 (n, H, W) = sigmoid(d0)."""

    def __init__(self, sd: Dict[str, torch.Tensor], device="cuda"):
        self.device = torch.device(device)
        f = fold(live_state_dict(sd))
        self.convs = {k: v for k, v in f.items() if k not in ("sides", "b0")}
        self.sides, self.b0 = f["sides"], f["b0"]
        self._packed = {}
        self._plan = None                 # (input shape, x0, launches, out) of the last input shape
        self._steps = None

    # ---- weights, packed for the channel layout of the inputs on first use -----------------------------------------------------
    def _packed_conv(self, key, w64: torch.Tensor, b64: torch.Tensor, layout):
        """fp16 [Co_pad, 9 * Ktap] with K ordered (tap, window channel) and fp32 bias [Co_pad]; layout = [(window, offset,
        channels)] of the GEMM segments over the conv's input channels in order."""
        if key not in self._packed:
            co, ci = w64.shape[:2]
            co_pad = (co + 7) // 8 * 8
            kt = sum(win for win, _, _ in layout)
            wp = torch.zeros(co_pad, 3, 3, kt, dtype=torch.float64)
            c0 = k0 = 0
            for win, off, c in layout:
                wp[:co, :, :, k0 + off:k0 + off + c] = w64[:, c0:c0 + c].permute(0, 2, 3, 1)
                c0 += c
                k0 += win
            if c0 != ci:
                raise ValueError(f"U^2-Net {key[0]}: inputs carry {c0} channels, the weight takes {ci}")
            bp = torch.zeros(co_pad, dtype=torch.float64)
            bp[:co] = b64
            self._packed[key] = (wp.reshape(co_pad, -1).to(self.device, torch.float16).contiguous(),
                                 bp.to(self.device, torch.float32).contiguous())
        return self._packed[key]

    def _conv(self, name, w64, b64, dil, inputs: Sequence, n, h, w, out: torch.Tensor, residual=None, relu=True):
        """Records out[:, :Co] = [relu](conv(cat(inputs))) [+ residual]; inputs: SegSpecs (channel ranges of NHWC buffers)."""
        from . import ops
        pieces = []
        for s in inputs:                  # merge adjacent channel ranges of one buffer (a concat buffer's two halves)
            q = pieces[-1] if pieces else None
            if q is not None and q.src.data_ptr() == s.src.data_ptr() and q.ld == s.ld and q.c_off + q.C == s.c_off:
                pieces[-1] = ops.SegSpec(q.src, C_=q.C + s.C, c_off=q.c_off, ld=q.ld)
            else:
                pieces.append(s)
        segs, layout = [], []
        for s in pieces:
            if s.C % 64 == 0:
                segs.append(s)
                layout.append((s.C, 0, s.C))
            else:                         # a 64-channel window whose other channels are zero
                lo = s.c_off // 64 * 64
                if s.c_off + s.C > lo + 64 or lo + 64 > s.ld:
                    raise ValueError(f"U^2-Net {name}: channels {s.c_off}..{s.c_off + s.C} of a {s.ld}-wide buffer")
                segs.append(ops.SegSpec(s.src, C_=64, c_off=lo, ld=s.ld))
                layout.append((64, s.c_off - lo, s.C))
        wt, bias = self._packed_conv((name, tuple(layout)), w64, b64, layout)
        if out.shape[1] != w64.shape[0] and not (out.shape[1] == wt.shape[0] and out.is_contiguous()):
            raise ValueError(f"U^2-Net {name}: output of {out.shape[1]} channels for {w64.shape[0]}")
        self._steps.append(ops.Gemm(ops.conv_taps(segs, dilation=dil), wt, out, n * h * w, mode=ops.ROWS_CONV2D,
                                    geom=dict(Ho=h, Wo=w, Hs=h, Ws=w, stride=1), bias=bias,
                                    act=ops.ACT_RELU if relu else ops.ACT_NONE, residual=residual, engine="tc5"))

    def _buf(self, rows, live, zero=False):
        """NHWC buffer of `live` channels padded to 64; zero-filled when padded (the pad channels are read with zero weights)."""
        width = _pad64(live)
        if width == live and not zero:
            return torch.empty(rows, width, dtype=torch.float16, device=self.device)
        return torch.zeros(rows, width, dtype=torch.float16, device=self.device)

    def _rsu(self, stage: str, inputs, n: int, H: int, W: int, out: torch.Tensor):
        """Records one RSU-L / RSU4F on `inputs` (SegSpecs at H x W), storing hx1d + hxin into `out` (a [n*H*W, out] view)."""
        from . import ops
        L, pooled = STAGE_KIND[stage]
        cv = lambda name, *a, **k: self._conv(f"{stage}.{name}", *self.convs[f"{stage}.{name}"], *a, **k)   # noqa: E731
        mid = self.convs[f"{stage}.rebnconv1"][0].shape[0]
        cout = self.convs[f"{stage}.rebnconvin"][0].shape[0]
        sizes = [(H, W)]
        for _ in range(1, L - 1):
            h, w = sizes[-1]
            sizes.append(((h + 1) // 2, (w + 1) // 2) if pooled else (h, w))
        rows = [n * h * w for h, w in sizes]
        hxin = self._buf(rows[0], cout)
        cv("rebnconvin", inputs, n, H, W, hxin[:, :cout])
        # level k (1-based) = sizes[k - 1]; D[k]: decoder concat [up(hx(k+1)d) | hxk] of levels 1 .. L-2
        # (zero-filled whenever a half is not 64-aligned: a conv may read a half as a window that spans the other one)
        D = [None] + [self._buf(rows[k - 1], 2 * mid, zero=mid % 64 != 0) for k in range(1, L - 1)]
        if not pooled and mid % 64:
            # RSU4F's encoder reads an upper half through a window that spans the lower half, which this call's decoder writes
            # only later: zero it first, so that no value of the previous call meets the zero weight columns there
            self._steps += [functools.partial(torch.Tensor.zero_, D[k][:, :mid]) for k in range(1, L - 1)]
        E, B = self._buf(rows[-1], mid), self._buf(rows[-1], mid)         # hx(L-1) and hxL at the deepest level
        upper = lambda k: ops.SegSpec(D[k], C_=mid, c_off=mid)            # noqa: E731
        lower = lambda k: ops.SegSpec(D[k], C_=mid, c_off=0)              # noqa: E731
        src = ops.SegSpec(hxin, C_=cout)
        for k in range(1, L):
            h, w = sizes[k - 1]
            if k > 1 and pooled:
                ph, pw = sizes[k - 2]
                P = self._buf(rows[k - 1], mid)
                self._steps.append(functools.partial(ops.maxpool2x2_ceil, D[k - 1][:, mid:2 * mid], n, ph, pw, P[:, :mid]))
                src = ops.SegSpec(P, C_=mid)
            dst = D[k][:, mid:2 * mid] if k < L - 1 else E[:, :mid]
            cv(f"rebnconv{k}", [src], n, h, w, dst)
            src = upper(k) if k < L - 1 else ops.SegSpec(E, C_=mid)
        h, w = sizes[-1]
        cv(f"rebnconv{L}", [ops.SegSpec(E, C_=mid)], n, h, w, B[:, :mid])
        cur = [ops.SegSpec(B, C_=mid), ops.SegSpec(E, C_=mid)]
        for k in range(L - 1, 0, -1):
            h, w = sizes[k - 1]
            if k == 1:
                cv("rebnconv1d", cur, n, h, w, out, residual=hxin)
                break
            if pooled:
                U = torch.empty(rows[k - 1], mid, dtype=torch.float16, device=self.device)
                cv(f"rebnconv{k}d", cur, n, h, w, U)
                th, tw = sizes[k - 2]
                self._steps.append(functools.partial(ops.resize_bilinear, U, n, h, w, D[k - 1][:, :mid], th, tw))
            else:                     # RSU4F: one size throughout, so the conv stores into the next concat's lower half
                cv(f"rebnconv{k}d", cur, n, h, w, D[k - 1][:, :mid])
            cur = [lower(k - 1), upper(k - 1)]

    @torch.no_grad()
    def __call__(self, img: torch.Tensor) -> torch.Tensor:
        from . import ops
        if img.dim() != 4 or img.shape[1] != 3 or img.shape[2] == 0 or img.shape[3] == 0:
            raise ValueError(f"expected (n, 3, H, W) images, got {tuple(img.shape)}")
        img = img.to(self.device)
        if img.dtype not in (torch.float32, torch.float16):
            img = img.float()
        img = img.contiguous()
        n, _, H, W = img.shape
        if self._plan is None or self._plan[0] != (n, H, W):
            self._plan = None                                            # release the previous shape's buffers first
            self._plan = ((n, H, W),) + self._build(n, H, W)
        _, x0, steps, out = self._plan
        ops.nchw_to_nhwc(img, x0)                                        # channels 3..63 zero
        for step in steps:
            step()
        return out.clone()

    def _build(self, n: int, H: int, W: int):
        """The launch plan for (n, 3, H, W) inputs: every buffer, allocated once (padding channels zero-filled once, never
        written), and the list of launches with their GEMM parameter blocks pre-baked.  Returns (x0, steps, out)."""
        from . import ops
        self._steps = []
        e = lambda r, c: torch.empty(r, c, dtype=torch.float16, device=self.device)   # noqa: E731
        x0 = e(n * H * W, 64)
        sizes = [(H, W)]
        for _ in range(5):
            h, w = sizes[-1]
            sizes.append(((h + 1) // 2, (w + 1) // 2))
        rows = [n * h * w for h, w in sizes]
        width = lambda s: self.convs[f"{s}.rebnconvin"][0].shape[0]      # noqa: E731
        enc_out = [width(f"stage{k}") for k in range(1, 7)]
        dec_out = [width(f"stage{k}d") for k in range(1, 6)] + [enc_out[5]]
        # T[k]: input concat of stage{k}d, [up(hx(k+1)d or hx6) | hxk]
        T = [e(rows[k], dec_out[k + 1] + enc_out[k]) for k in range(5)]
        hx6 = e(rows[5], enc_out[5])
        src = [ops.SegSpec(x0, C_=3)]
        for k in range(6):
            h, w = sizes[k]
            if k > 0:
                ph, pw = sizes[k - 1]
                P = e(rows[k], enc_out[k - 1])
                self._steps.append(functools.partial(ops.maxpool2x2_ceil, T[k - 1][:, dec_out[k]:], n, ph, pw, P))
                src = [ops.SegSpec(P)]
            dst = T[k][:, dec_out[k + 1]:] if k < 5 else hx6
            self._rsu(f"stage{k + 1}", src, n, h, w, dst)
        prev, side_in = hx6, [None] * 6
        side_in[5] = hx6
        for k in range(4, -1, -1):
            h, w = sizes[k]
            ph, pw = sizes[k + 1]
            self._steps.append(functools.partial(ops.resize_bilinear, prev, n, ph, pw, T[k][:, :dec_out[k + 1]], h, w))
            hd = e(rows[k], dec_out[k])
            self._rsu(f"stage{k + 1}d", [ops.SegSpec(T[k])], n, h, w, hd)
            side_in[k] = prev = hd
        sides = []
        for k in range(6):
            h, w = sizes[k]
            sw, sb = self.sides[k]
            s = e(rows[k], 8)
            self._conv(f"side{k + 1}", sw, sb, 1, [ops.SegSpec(side_in[k])], n, h, w, s, relu=False)
            sides.append((s, h, w))
        out = torch.empty(n, H, W, dtype=torch.float32, device=self.device)
        self._steps.append(functools.partial(ops.u2net_fuse_sides, sides, self.b0, n, H, W, out))
        steps, self._steps = self._steps, None
        return x0, steps, out


def param_count(sd: Dict[str, torch.Tensor]) -> int:
    """Learnable parameters (conv weights and biases, BatchNorm affine), as nn.Module.parameters() counts them."""
    return sum(v.numel() for k, v in sd.items() if not k.endswith(("running_mean", "running_var", "num_batches_tracked")))


__all__ = ["U2NetTower", "load_u2net", "live_state_dict", "fold", "expected_keys", "param_count", "rsu_convs", "STAGES"]
