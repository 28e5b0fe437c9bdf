"""Weight re-packing from the reference state_dict layout (OIHW convs, [out, in] linears) into the fp16
K-major [N, K] matrices the implicit-GEMM engine consumes.  Done once at load time."""
from __future__ import annotations

from typing import Optional, Tuple

import torch

F16 = torch.float16
E4M3 = torch.float8_e4m3fn
E4M3_MAX = 448.0


def _pad_to(x: int, m: int) -> int:
    return (x + m - 1) // m * m


def pack_conv2d(w: torch.Tensor, cin_pad: Optional[int] = None, cout_pad: Optional[int] = None) -> torch.Tensor:
    """(Co, Ci, kh, kw) -> fp16 [Co_p, kh*kw*Ci_p], K ordered (ky, kx, ci) == ops.conv_taps order."""
    co, ci, kh, kw = w.shape
    cip = cin_pad or ci
    cop = cout_pad or co
    out = torch.zeros(cop, kh, kw, cip, dtype=torch.float32, device=w.device)
    out[:co, :, :, :ci] = w.float().permute(0, 2, 3, 1)
    return out.reshape(cop, kh * kw * cip).to(F16).contiguous()


def pack_conv3d_t(w: torch.Tensor, cin_pad: Optional[int] = None, cout_pad: Optional[int] = None) -> torch.Tensor:
    """(Co, Ci, 3, 1, 1) temporal conv -> fp16 [Co_p, 3*Ci_p], K ordered (kt, ci) == ops.temporal_taps order."""
    co, ci = w.shape[:2]
    if tuple(w.shape[2:]) != (3, 1, 1):
        raise NotImplementedError(f"temporal conv kernel {tuple(w.shape[2:])}: only (3, 1, 1) (the SVD / Hi3D video_kernel_size) "
                                  f"maps onto the frame-tap GEMM mode")
    cip, cop = cin_pad or ci, cout_pad or co
    out = torch.zeros(cop, 3, cip, dtype=torch.float32, device=w.device)
    out[:co, :, :ci] = w.float()[:, :, :, 0, 0].permute(0, 2, 1)
    return out.reshape(cop, 3 * cip).to(F16).contiguous()


def pack_linear(w: torch.Tensor, cout_pad: Optional[int] = None) -> torch.Tensor:
    w = w.float().reshape(w.shape[0], -1)
    if cout_pad and cout_pad > w.shape[0]:
        w = torch.cat([w, w.new_zeros(cout_pad - w.shape[0], w.shape[1])], 0)
    return w.to(F16).contiguous()


def pack_bias(b: Optional[torch.Tensor], n: int, cout_pad: Optional[int] = None, device=None) -> torch.Tensor:
    out = torch.zeros(cout_pad or n, dtype=torch.float32, device=device if b is None else b.device)
    if b is not None:
        out[:n] = b.float()
    return out.contiguous()


def pack_geglu(w: torch.Tensor, b: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """GEGLU projection (attention.py:87-94): rows [value(4C) ; gate(4C)] -> interleaved (value_j, gate_j) so
    the pair lands in one accumulator fragment and x*gelu(gate) is thread-local in the epilogue."""
    inner = w.shape[0] // 2
    wi = torch.stack([w[:inner].float(), w[inner:].float()], dim=1).reshape(2 * inner, -1)
    bi = torch.stack([b[:inner].float(), b[inner:].float()], dim=1).reshape(2 * inner)
    return wi.to(F16).contiguous(), bi.contiguous()


# nearest-x2 upsample followed by a 3x3 conv (openaimodel.py:154-156, model.py:67-71) == four parity-specific 2x2 convs on
# the SOURCE grid: output pixel (2y+py, 2x+px) with tap dy reads source row y + floor((py+dy)/2), so the three taps of
# one axis collapse onto two source shifts and their weights can be summed up front (4/9 of the FLOPs, no upsampled tensor).
UP_SHIFTS = {0: ((-1, (0,)), (0, (1, 2))), 1: ((0, (0, 1)), (1, (2,)))}     # parity -> ((shift, kernel indices), ...)


def pack_upconv_parity(w: torch.Tensor):
    """(Co, Ci, 3, 3) -> {(py, px): (fp16 [Co, 4*Ci], [(sy, sx), ...])}: K ordered like ops.conv_taps over the listed
    (dy, dx) source shifts."""
    co, ci = w.shape[:2]
    wf = w.float()
    out = {}
    for py in (0, 1):
        for px in (0, 1):
            mats, shifts = [], []
            for sy, kys in UP_SHIFTS[py]:
                for sx, kxs in UP_SHIFTS[px]:
                    acc = torch.zeros(co, ci, dtype=torch.float32, device=w.device)
                    for ky in kys:
                        for kx in kxs:
                            acc += wf[:, :, ky, kx]
                    mats.append(acc)
                    shifts.append((sy, sx))
            out[(py, px)] = (torch.cat(mats, dim=1).to(F16).contiguous(), shifts)
    return out


def cat_k(*mats: torch.Tensor) -> torch.Tensor:
    """Concatenate packed matrices along K (e.g. [3x3 conv | 1x1 skip] fused into one GEMM)."""
    return torch.cat(mats, dim=1).contiguous()


def pack_e4m3(w: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """Packed fp16 [N, K] weight matrix -> (e4m3 [N, K], fp32 [N] scale) for hi3d_gemm_tc5_fp8: row n is stored as
    w[n] / scale[n] rounded to nearest even and saturated to +-448, with scale[n] = amax(|w[n]|) / 448 (1 for an all-zero row),
    so that w[n] ~ e4m3[n] * scale[n].  Zero padding along K stays zero."""
    if w.dtype != F16 or w.dim() != 2:
        raise ValueError(f"pack_e4m3: expected a packed fp16 [N, K] matrix, got {w.dtype} {tuple(w.shape)}")
    wf = w.float()
    amax = wf.abs().amax(dim=1)
    scale = torch.where(amax > 0, amax / E4M3_MAX, torch.ones_like(amax))
    q = (wf / scale[:, None]).clamp(-E4M3_MAX, E4M3_MAX).to(E4M3)
    return q.contiguous(), scale.contiguous()
