"""ORACLE -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

A from-scratch, functional, plain-PyTorch fp32 restatement of the Hi3D denoising hot path
(EDM sampler x VideoUNet + AutoencoderKL).  Only `tests/`, `__graft_entry__.smoke()` and the
`cpu_baseline` / `--impl reference` legs of `bench.py` may import this file; the product package
`hi3d_official_b200` never does (it fails loudly when its CUDA library is missing instead).

Every function cites the reference file:line (relative to /root/reference) that it restates.  The
functions take the reference's own `state_dict` (same key names / shapes, SURVEY.md App. B) so the
very same weights can be loaded into the real reference (build container only, `oracle/ref_import.py`),
into this oracle (anywhere, CPU or GPU fp32) and into the CUDA product.

Parity pinning: the reference ships NO tests / golden vectors for this path (SURVEY.md F10, §8c), so
the oracle is pinned against *outputs of the reference itself run in the build container*:
`tests/test_oracle_vs_reference.py` (against stored outputs of the reference) and the committed fixtures
`tests/golden/*.pt` produced by `tools/make_golden.py` from the real reference modules.

Numerics: everything is computed in the dtype of the inputs/weights (fp32 on the oracle path); the
reference's fp16-autocast rounding points (SURVEY.md App. E) are deliberately NOT reproduced -- the
fp32 result is the ground truth both the reference-fp16 path and the CUDA path are compared against.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence

import torch
import torch.nn.functional as F

P = Dict[str, torch.Tensor]

# ----------------------------------------------------------------------------------------------
# small helpers
# ----------------------------------------------------------------------------------------------


def timestep_embedding(t: torch.Tensor, dim: int, max_period: float = 10000.0) -> torch.Tensor:
    """[cos | sin] sinusoidal embedding, fp32.  sgm/modules/diffusionmodules/util.py:207-231."""
    half = dim // 2
    freqs = torch.exp(-math.log(max_period) * torch.arange(half, dtype=torch.float32, device=t.device) / half)
    args = t.float()[:, None] * freqs[None]
    emb = torch.cat([torch.cos(args), torch.sin(args)], dim=-1)
    if dim % 2:
        emb = torch.cat([emb, torch.zeros_like(emb[:, :1])], dim=-1)
    return emb


def _lin(p: P, name: str, x: torch.Tensor) -> torch.Tensor:
    return F.linear(x, p[name + ".weight"], p.get(name + ".bias"))


def _gn(p: P, name: str, x: torch.Tensor, eps: float) -> torch.Tensor:
    """32-group GroupNorm over (C/32, *spatial).  util.py:259-276 (eps 1e-5, UNet ResBlocks / out) and
    attention.py:125-128 / model.py:52-55 (eps 1e-6, transformers and VAE)."""
    return F.group_norm(x, 32, p[name + ".weight"], p[name + ".bias"], eps)


def _ln(p: P, name: str, x: torch.Tensor) -> torch.Tensor:
    return F.layer_norm(x, (x.shape[-1],), p[name + ".weight"], p[name + ".bias"], 1e-5)


def _has(p: P, prefix: str) -> bool:
    return any(k.startswith(prefix) for k in p)


# ----------------------------------------------------------------------------------------------
# UNet blocks
# ----------------------------------------------------------------------------------------------


def resblock(p: P, pre: str, x: torch.Tensor, emb: torch.Tensor, temporal: bool = False) -> torch.Tensor:
    """ResBlock._forward, openaimodel.py:328-354 (no up/down, no scale-shift-norm).
    temporal=True is the `time_stack` instance: x is (b, c, t, h, w), Conv3d kernel (3,1,1) padding (1,0,0),
    emb is (b, t, E) and is applied as (b, c, t, 1, 1) (`exchange_temb_dims`, openaimodel.py:350-352)."""
    conv = F.conv3d if temporal else F.conv2d
    pad = (1, 0, 0) if temporal else 1
    h = F.silu(_gn(p, pre + "in_layers.0", x, 1e-5))
    h = conv(h, p[pre + "in_layers.2.weight"], p[pre + "in_layers.2.bias"], padding=pad)
    e = _lin(p, pre + "emb_layers.1", F.silu(emb))
    if temporal:
        e = e.permute(0, 2, 1)[..., None, None]          # (b, t, c) -> (b, c, t, 1, 1)
    else:
        e = e[..., None, None]
    h = h + e
    h = F.silu(_gn(p, pre + "out_layers.0", h, 1e-5))
    h = conv(h, p[pre + "out_layers.3.weight"], p[pre + "out_layers.3.bias"], padding=pad)
    if pre + "skip_connection.weight" in p:
        x = conv(x, p[pre + "skip_connection.weight"], p[pre + "skip_connection.bias"])
    return x + h


def video_resblock(p: P, pre: str, x: torch.Tensor, emb: torch.Tensor, T: int) -> torch.Tensor:
    """VideoResBlock.forward, video_model.py:62-81, with AlphaBlender 'learned_with_images' and
    image_only_indicator == 0 (util.py:341-369): alpha = sigmoid(mix_factor)."""
    x = resblock(p, pre, x, emb)
    n, c, hh, ww = x.shape
    b = n // T
    x5 = x.view(b, T, c, hh, ww).permute(0, 2, 1, 3, 4)
    xt = resblock(p, pre + "time_stack.", x5, emb.view(b, T, -1), temporal=True)
    a = torch.sigmoid(p[pre + "time_mixer.mix_factor"]).to(x.dtype)
    out = a * x5 + (1.0 - a) * xt
    return out.permute(0, 2, 1, 3, 4).reshape(n, c, hh, ww)


def attention_core(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, heads: int) -> torch.Tensor:
    """softmax(q k^T / sqrt(d)) v with (b, n, h*d) tensors.  attention.py:309-340 (SDPA, default scale)."""
    b, n, hd = q.shape
    d = hd // heads
    q = q.view(b, n, heads, d).transpose(1, 2)
    k = k.view(b, k.shape[1], heads, d).transpose(1, 2)
    v = v.view(b, v.shape[1], heads, d).transpose(1, 2)
    # same arithmetic for every batch element; batch chunks only bound the size of the materialised score matrix
    # (32 x 5 x 16384^2 fp32 scores of the stage-2 top level would be 172 GB)
    per = heads * n * k.shape[2] * 4
    step = max(1, min(b, (2 << 30) // max(per, 1)))
    outs = []
    for i in range(0, b, step):
        s = torch.matmul(q[i:i + step], k[i:i + step].transpose(-1, -2)) * (d ** -0.5)
        outs.append(torch.matmul(torch.softmax(s.float(), dim=-1).to(q.dtype), v[i:i + step]))
    o = outs[0] if len(outs) == 1 else torch.cat(outs, 0)
    return o.transpose(1, 2).reshape(b, n, hd)


def cross_attention(p: P, pre: str, x: torch.Tensor, ctx: Optional[torch.Tensor], heads: int) -> torch.Tensor:
    """CrossAttention.forward, attention.py:281-344 (to_q/to_k/to_v have no bias; to_out.0 has)."""
    ctx = x if ctx is None else ctx
    q = F.linear(x, p[pre + "to_q.weight"])
    k = F.linear(ctx, p[pre + "to_k.weight"])
    v = F.linear(ctx, p[pre + "to_v.weight"])
    return _lin(p, pre + "to_out.0", attention_core(q, k, v, heads))


def feed_forward(p: P, pre: str, x: torch.Tensor) -> torch.Tensor:
    """FeedForward with GEGLU (exact-erf GELU), attention.py:87-113."""
    a, g = _lin(p, pre + "net.0.proj", x).chunk(2, dim=-1)
    return _lin(p, pre + "net.2", a * F.gelu(g))


def basic_transformer_block(p: P, pre: str, x: torch.Tensor, ctx: torch.Tensor, heads: int) -> torch.Tensor:
    """BasicTransformerBlock._forward, attention.py:551-572."""
    x = cross_attention(p, pre + "attn1.", _ln(p, pre + "norm1", x), None, heads) + x
    x = cross_attention(p, pre + "attn2.", _ln(p, pre + "norm2", x), ctx, heads) + x
    x = feed_forward(p, pre + "ff.", _ln(p, pre + "norm3", x)) + x
    return x


def video_transformer_block(p: P, pre: str, x: torch.Tensor, ctx: torch.Tensor, heads: int, T: int) -> torch.Tensor:
    """VideoTransformerBlock._forward, video_attention.py:109-140 (ff_in present, is_res, attn2 = cross-attn)."""
    B, S, C = x.shape
    b = B // T
    x = x.view(b, T, S, C).permute(0, 2, 1, 3).reshape(b * S, T, C)       # (b t) s c -> (b s) t c
    x = feed_forward(p, pre + "ff_in.", _ln(p, pre + "norm_in", x)) + x
    x = cross_attention(p, pre + "attn1.", _ln(p, pre + "norm1", x), None, heads) + x
    x = cross_attention(p, pre + "attn2.", _ln(p, pre + "norm2", x), ctx, heads) + x
    x = feed_forward(p, pre + "ff.", _ln(p, pre + "norm3", x)) + x
    return x.view(b, S, T, C).permute(0, 2, 1, 3).reshape(B, S, C)


def spatial_video_transformer(p: P, pre: str, x: torch.Tensor, context: torch.Tensor, T: int, heads: int,
                              max_period: float = 10000.0) -> torch.Tensor:
    """SpatialVideoTransformer.forward, video_attention.py:230-301 (use_linear, use_spatial_context, depth 1..n)."""
    n, c, hh, ww = x.shape
    x_in = x
    # time context = context of the first frame of every clip, repeated over pixels  (:249-253)
    tctx = context[::T]
    tctx = tctx[:, None].expand(-1, hh * ww, *tctx.shape[1:]).reshape(-1, *tctx.shape[1:])
    x = _gn(p, pre + "norm", x, 1e-6)
    x = x.permute(0, 2, 3, 1).reshape(n, hh * ww, c)
    x = _lin(p, pre + "proj_in", x)
    frames = torch.arange(T, device=x.device).repeat(n // T)
    emb = timestep_embedding(frames, c, max_period).to(x.dtype)
    emb = _lin(p, pre + "time_pos_embed.2", F.silu(_lin(p, pre + "time_pos_embed.0", emb)))[:, None, :]
    a = torch.sigmoid(p[pre + "time_mixer.mix_factor"]).to(x.dtype)
    d = 0
    while pre + f"transformer_blocks.{d}.norm1.weight" in p:
        x = basic_transformer_block(p, pre + f"transformer_blocks.{d}.", x, context, heads)
        x_mix = video_transformer_block(p, pre + f"time_stack.{d}.", x + emb, tctx, heads, T)
        x = a * x + (1.0 - a) * x_mix
        d += 1
    x = _lin(p, pre + "proj_out", x)
    x = x.view(n, hh, ww, c).permute(0, 3, 1, 2)
    return x + x_in


def _run_block(p: P, pre: str, h: torch.Tensor, emb: torch.Tensor, context: torch.Tensor, T: int,
               head_ch: int) -> torch.Tensor:
    """TimestepEmbedSequential.forward dispatch, openaimodel.py:72-104, driven by which keys exist."""
    i = 0
    while _has(p, f"{pre}{i}."):
        q = f"{pre}{i}."
        if q + "in_layers.0.weight" in p:
            h = video_resblock(p, q, h, emb, T)
        elif q + "transformer_blocks.0.norm1.weight" in p:
            h = spatial_video_transformer(p, q, h, context, T, h.shape[1] // head_ch)
        elif q + "op.weight" in p:        # Downsample: conv3x3 stride 2 pad 1, openaimodel.py:192-199
            h = F.conv2d(h, p[q + "op.weight"], p[q + "op.bias"], stride=2, padding=1)
        elif q + "conv.weight" in p:      # Upsample: nearest x2 then conv3x3, openaimodel.py:154-156
            h = F.interpolate(h, scale_factor=2, mode="nearest")
            h = F.conv2d(h, p[q + "conv.weight"], p[q + "conv.bias"], padding=1)
        elif q + "weight" in p:           # input_blocks.0.0 plain conv
            h = F.conv2d(h, p[q + "weight"], p[q + "bias"], padding=1)
        else:
            raise KeyError(q)
        i += 1
    return h


def unet_forward(p: P, x: torch.Tensor, timesteps: torch.Tensor, context: torch.Tensor, y: torch.Tensor,
                 num_video_frames: int = 16, num_head_channels: int = 64) -> torch.Tensor:
    """VideoUNet.forward, video_model.py:442-501 (image_only_indicator == 0)."""
    T = num_video_frames
    mc = p["time_embed.0.weight"].shape[1]
    emb = _lin(p, "time_embed.2", F.silu(_lin(p, "time_embed.0", timestep_embedding(timesteps, mc).to(x.dtype))))
    if y.shape[0] != x.shape[0]:          # Hi3D "fast implementation" broadcast, :459-465
        y = y.repeat_interleave(T, dim=0)
    if context.shape[0] != x.shape[0]:
        context = context.repeat_interleave(T, dim=0)
    emb = emb + _lin(p, "label_emb.0.2", F.silu(_lin(p, "label_emb.0.0", y.to(x.dtype))))
    hs: List[torch.Tensor] = []
    h = x
    i = 0
    while _has(p, f"input_blocks.{i}."):
        h = _run_block(p, f"input_blocks.{i}.", h, emb, context, T, num_head_channels)
        hs.append(h)
        i += 1
    h = _run_block(p, "middle_block.", h, emb, context, T, num_head_channels)
    i = 0
    while _has(p, f"output_blocks.{i}."):
        h = torch.cat([h, hs.pop()], dim=1)
        h = _run_block(p, f"output_blocks.{i}.", h, emb, context, T, num_head_channels)
        i += 1
    h = F.silu(_gn(p, "out.0", h, 1e-5))
    return F.conv2d(h, p["out.2.weight"], p["out.2.bias"], padding=1)


def wrapper_forward(p: P, x: torch.Tensor, t: torch.Tensor, c: Dict[str, torch.Tensor], **kw) -> torch.Tensor:
    """OpenAIWrapper.forward, wrappers.py:23-34."""
    if "concat" in c:
        x = torch.cat((x, c["concat"].to(x.dtype)), dim=1)
    return unet_forward(p, x, t, c["crossattn"].to(x.dtype), c["vector"], **kw)


# ----------------------------------------------------------------------------------------------
# EDM sampler
# ----------------------------------------------------------------------------------------------


def edm_sigmas(n: int, sigma_min: float = 0.002, sigma_max: float = 700.0, rho: float = 7.0,
               device="cpu") -> torch.Tensor:
    """EDMDiscretization.get_sigmas + append_zero, discretizer.py:17-39."""
    ramp = torch.linspace(0, 1, n, device=device)
    mi, ma = sigma_min ** (1 / rho), sigma_max ** (1 / rho)
    s = (ma + ramp * (mi - ma)) ** rho
    return torch.cat([s, s.new_zeros(1)])


def vscaling_edm_cnoise(sigma: torch.Tensor):
    """VScalingWithEDMcNoise, denoiser_scaling.py:51-59 -> (c_skip, c_out, c_in, c_noise)."""
    return (1.0 / (sigma ** 2 + 1.0), -sigma / (sigma ** 2 + 1.0) ** 0.5, 1.0 / (sigma ** 2 + 1.0) ** 0.5,
            0.25 * sigma.log())


def denoise(p: P, x: torch.Tensor, sigma: torch.Tensor, cond: Dict[str, torch.Tensor], **kw) -> torch.Tensor:
    """Denoiser.forward, denoiser.py:23-39."""
    s = sigma.view(-1, *([1] * (x.ndim - 1)))
    c_skip, c_out, c_in, c_noise = vscaling_edm_cnoise(s)
    return wrapper_forward(p, x * c_in, c_noise.reshape(sigma.shape), cond, **kw) * c_out + x * c_skip


def guider_scale(num_frames: int, max_scale: float, min_scale: float = 1.0) -> torch.Tensor:
    """LinearPredictionGuider.scale, guiders.py:71."""
    return torch.linspace(min_scale, max_scale, num_frames)


def cfg_denoise(p: P, x: torch.Tensor, sigma: torch.Tensor, c: dict, uc: dict, scale: torch.Tensor,
                **kw) -> torch.Tensor:
    """BaseDiffusionSampler.denoise with LinearPredictionGuider: prepare_inputs (guiders.py:88-99),
    denoiser, combine x_u + s_t (x_c - x_u) per frame (guiders.py:78-86)."""
    T = scale.numel()
    cc = {k: torch.cat((uc[k], c[k]), 0) for k in c if k in ("vector", "crossattn", "concat")}
    d = denoise(p, torch.cat([x] * 2), torch.cat([sigma] * 2), cc, **kw)
    x_u, x_c = d.chunk(2)
    sc = scale.to(x.device, x.dtype).repeat(x_u.shape[0] // T).view(-1, 1, 1, 1)
    return x_u + sc * (x_c - x_u)


def euler_step(p: P, x: torch.Tensor, sigma: float, next_sigma: float, c: dict, uc: dict, scale: torch.Tensor,
               **kw) -> torch.Tensor:
    """EDMSampler.sampler_step with gamma = 0 (s_churn = 0), sampling.py:93-107; to_d sampling_utils.py:34."""
    s = x.new_full((x.shape[0],), float(sigma))
    den = cfg_denoise(p, x, s, c, uc, scale, **kw)
    d = (x - den) / sigma
    return x + d * (next_sigma - sigma)


def sample(p: P, x: torch.Tensor, c: dict, uc: dict, num_steps: int = 25, max_scale: float = 2.5,
           num_frames: int = 16, sigma_max: float = 700.0, **kw) -> torch.Tensor:
    """EDMSampler.__call__, sampling.py:126-147 (prepare_sampling_loop :41-52)."""
    sig = edm_sigmas(num_steps, sigma_max=sigma_max, device=x.device)
    x = x * torch.sqrt(1.0 + sig[0] ** 2.0)
    scale = guider_scale(num_frames, max_scale)
    for i in range(num_steps):
        x = euler_step(p, x, float(sig[i]), float(sig[i + 1]), c, uc, scale, num_video_frames=num_frames, **kw)
    return x


def v02_alpha(i: int, num_steps: int = 25, alpha_pow: float = 40.0) -> float:
    """pipeline_i2v_eval_v02.py:128-129."""
    return math.pow(0.5 * (1 + math.cos(i * 1.0 / num_steps)), alpha_pow)


def sample_v02(p: P, init_latents: torch.Tensor, z: torch.Tensor, c: dict, uc: dict, num_steps: int = 25,
               max_scale: float = 2.0, num_frames: int = 16, sigma_max: float = 700.0, **kw) -> torch.Tensor:
    """Stage-2 re-noise/blend loop, pipeline_i2v_eval_v02.py:86-135."""
    sig = edm_sigmas(num_steps, sigma_max=sigma_max, device=init_latents.device)
    lat = init_latents.clone() * torch.sqrt(1.0 + sig[0] ** 2.0)
    scale = guider_scale(num_frames, max_scale)
    for i in range(num_steps):
        a = v02_alpha(i, num_steps)
        lat = lat * (1 - a) + (init_latents * sig[i] + z) * a
        lat = euler_step(p, lat, float(sig[i]), float(sig[i + 1]), c, uc, scale, num_video_frames=num_frames, **kw)
    return lat


# ----------------------------------------------------------------------------------------------
# AutoencoderKL (2-D, per frame)
# ----------------------------------------------------------------------------------------------


def _swish(x):
    return x * torch.sigmoid(x)


def vae_resnet_block(p: P, pre: str, x: torch.Tensor) -> torch.Tensor:
    """ResnetBlock.forward (temb None), model.py:131-151."""
    h = F.conv2d(_swish(_gn(p, pre + "norm1", x, 1e-6)), p[pre + "conv1.weight"], p[pre + "conv1.bias"], padding=1)
    h = F.conv2d(_swish(_gn(p, pre + "norm2", h, 1e-6)), p[pre + "conv2.weight"], p[pre + "conv2.bias"], padding=1)
    if pre + "nin_shortcut.weight" in p:
        x = F.conv2d(x, p[pre + "nin_shortcut.weight"], p[pre + "nin_shortcut.bias"])
    return x + h


def vae_attn_block(p: P, pre: str, x: torch.Tensor) -> torch.Tensor:
    """AttnBlock.forward, model.py:180-201: single head, d = C, scale C^-0.5, 1x1 convs."""
    b, c, hh, ww = x.shape
    h = _gn(p, pre + "norm", x, 1e-6)
    q, k, v = (F.conv2d(h, p[pre + n + ".weight"], p[pre + n + ".bias"]).flatten(2).transpose(1, 2)
               for n in ("q", "k", "v"))
    o = attention_core(q, k, v, 1).transpose(1, 2).reshape(b, c, hh, ww)
    return x + F.conv2d(o, p[pre + "proj_out.weight"], p[pre + "proj_out.bias"])


def vae_encoder(p: P, x: torch.Tensor, pre: str = "encoder.") -> torch.Tensor:
    """Encoder.forward, model.py:576-601; Downsample = pad (0,1,0,1) + conv3x3 s2 p0, model.py:84-88."""
    h = F.conv2d(x, p[pre + "conv_in.weight"], p[pre + "conv_in.bias"], padding=1)
    lvl = 0
    while _has(p, f"{pre}down.{lvl}."):
        blk = 0
        while _has(p, f"{pre}down.{lvl}.block.{blk}."):
            h = vae_resnet_block(p, f"{pre}down.{lvl}.block.{blk}.", h)
            blk += 1
        if f"{pre}down.{lvl}.downsample.conv.weight" in p:
            h = F.pad(h, (0, 1, 0, 1))
            h = F.conv2d(h, p[f"{pre}down.{lvl}.downsample.conv.weight"], p[f"{pre}down.{lvl}.downsample.conv.bias"],
                         stride=2)
        lvl += 1
    h = vae_resnet_block(p, pre + "mid.block_1.", h)
    h = vae_attn_block(p, pre + "mid.attn_1.", h)
    h = vae_resnet_block(p, pre + "mid.block_2.", h)
    h = _swish(_gn(p, pre + "norm_out", h, 1e-6))
    return F.conv2d(h, p[pre + "conv_out.weight"], p[pre + "conv_out.bias"], padding=1)


def vae_decoder(p: P, z: torch.Tensor, pre: str = "decoder.") -> torch.Tensor:
    """Decoder.forward, model.py:715-748; Upsample = nearest x2 + conv3x3, model.py:67-71."""
    h = F.conv2d(z, p[pre + "conv_in.weight"], p[pre + "conv_in.bias"], padding=1)
    h = vae_resnet_block(p, pre + "mid.block_1.", h)
    h = vae_attn_block(p, pre + "mid.attn_1.", h)
    h = vae_resnet_block(p, pre + "mid.block_2.", h)
    nlev = 0
    while _has(p, f"{pre}up.{nlev}."):
        nlev += 1
    for lvl in reversed(range(nlev)):
        blk = 0
        while _has(p, f"{pre}up.{lvl}.block.{blk}."):
            h = vae_resnet_block(p, f"{pre}up.{lvl}.block.{blk}.", h)
            blk += 1
        if f"{pre}up.{lvl}.upsample.conv.weight" in p:
            h = F.interpolate(h, scale_factor=2.0, mode="nearest")
            h = F.conv2d(h, p[f"{pre}up.{lvl}.upsample.conv.weight"], p[f"{pre}up.{lvl}.upsample.conv.bias"],
                         padding=1)
    h = _swish(_gn(p, pre + "norm_out", h, 1e-6))
    return F.conv2d(h, p[pre + "conv_out.weight"], p[pre + "conv_out.bias"], padding=1)


def vae_encode_moments(p: P, x: torch.Tensor) -> torch.Tensor:
    """AutoencodingEngineLegacy.encode up to the regulariser, autoencoder.py:468-482."""
    return F.conv2d(vae_encoder(p, x), p["quant_conv.weight"], p["quant_conv.bias"])


def vae_encode(p: P, x: torch.Tensor, noise: Optional[torch.Tensor] = None, scale_factor: float = 0.18215):
    """encode_first_stage, diffusion.py:137-150 + DiagonalGaussianDistribution.sample/mode,
    distributions.py:24-41,71 (noise=None -> mode; else mean + std * noise, noise drawn by the caller)."""
    mean, logvar = vae_encode_moments(p, x).chunk(2, dim=1)
    if noise is not None:
        logvar = logvar.clamp(-30.0, 20.0)
        mean = mean + torch.exp(0.5 * logvar) * noise
    return scale_factor * mean


def vae_decode(p: P, z: torch.Tensor, scale_factor: float = 0.18215) -> torch.Tensor:
    """decode_first_stage, diffusion.py:117-135 + AutoencodingEngineLegacy.decode, autoencoder.py:490-505."""
    z = z / scale_factor
    return vae_decoder(p, F.conv2d(z, p["post_quant_conv.weight"], p["post_quant_conv.bias"]))


# ----------------------------------------------------------------------------------------------
# SURVEY §8(f) N1: temporal VAE decoder `VideoDecoder` (time_mode "conv-only", the SVD setting) -- oracle only so far;
# the CUDA path is the next row to build.  Pinned against the reference class in tests/test_oracle_vs_reference.py.
# ----------------------------------------------------------------------------------------------


def _tpad(w: torch.Tensor):
    """padding of a Conv3d whose kernel is (kt, kh, kw): k // 2 per axis (temporal_ae.py:88-92, openaimodel.py:263-270)."""
    return tuple(int(k) // 2 for k in w.shape[2:])


def vae_time_stack(p: P, pre: str, x5: torch.Tensor) -> torch.Tensor:
    """The `time_stack` of temporal_ae.VideoResBlock: openaimodel.ResBlock(dims=3, skip_t_emb=True, no up/down, same
    channels -> identity skip), openaimodel.py:328-354 with emb_out = 0.  x5: (b, c, t, h, w)."""
    w1, w2 = p[pre + "in_layers.2.weight"], p[pre + "out_layers.3.weight"]
    h = F.conv3d(F.silu(_gn(p, pre + "in_layers.0", x5, 1e-5)), w1, p[pre + "in_layers.2.bias"], padding=_tpad(w1))
    h = F.conv3d(F.silu(_gn(p, pre + "out_layers.0", h, 1e-5)), w2, p[pre + "out_layers.3.bias"], padding=_tpad(w2))
    return x5 + h


def vae_video_resblock(p: P, pre: str, x: torch.Tensor, T: int) -> torch.Tensor:
    """temporal_ae.VideoResBlock.forward, temporal_ae.py:62-81.  NOTE the blend direction: alpha = sigmoid(mix_factor)
    weighs the TEMPORAL branch here (x = alpha * time_stack(x) + (1 - alpha) * x), the opposite of the UNet's
    AlphaBlender."""
    x = vae_resnet_block(p, pre, x)
    n, c, hh, ww = x.shape
    x5 = x.view(n // T, T, c, hh, ww).permute(0, 2, 1, 3, 4)
    a = torch.sigmoid(p[pre + "mix_factor"]).to(x.dtype)
    out = a * vae_time_stack(p, pre + "time_stack.", x5) + (1.0 - a) * x5
    return out.permute(0, 2, 1, 3, 4).reshape(n, c, hh, ww)


def vae_video_decoder(p: P, z: torch.Tensor, T: int, pre: str = "decoder.") -> torch.Tensor:
    """temporal_ae.VideoDecoder (time_mode 'conv-only': VideoResBlocks, plain AttnBlock, AE3DConv only as conv_out)
    run through Decoder.forward(z, timesteps=T), model.py:715-748 / temporal_ae.py:293-349."""
    h = F.conv2d(z, p[pre + "conv_in.weight"], p[pre + "conv_in.bias"], padding=1)
    h = vae_video_resblock(p, pre + "mid.block_1.", h, T)
    h = vae_attn_block(p, pre + "mid.attn_1.", h)
    h = vae_video_resblock(p, pre + "mid.block_2.", h, T)
    nlev = 0
    while _has(p, f"{pre}up.{nlev}."):
        nlev += 1
    for lvl in reversed(range(nlev)):
        blk = 0
        while _has(p, f"{pre}up.{lvl}.block.{blk}."):
            h = vae_video_resblock(p, f"{pre}up.{lvl}.block.{blk}.", h, T)
            blk += 1
        if f"{pre}up.{lvl}.upsample.conv.weight" in p:
            h = F.interpolate(h, scale_factor=2.0, mode="nearest")
            h = F.conv2d(h, p[f"{pre}up.{lvl}.upsample.conv.weight"], p[f"{pre}up.{lvl}.upsample.conv.bias"], padding=1)
    h = _swish(_gn(p, pre + "norm_out", h, 1e-6))
    # AE3DConv (temporal_ae.py:84-108): the 2-D conv, then a Conv3d over (t, h, w) of the (b, c, t, h, w) view
    h = F.conv2d(h, p[pre + "conv_out.weight"], p[pre + "conv_out.bias"], padding=1)
    n, c, hh, ww = h.shape
    wt = p[pre + "conv_out.time_mix_conv.weight"]
    h5 = F.conv3d(h.view(n // T, T, c, hh, ww).permute(0, 2, 1, 3, 4), wt, p[pre + "conv_out.time_mix_conv.bias"],
                  padding=_tpad(wt))
    return h5.permute(0, 2, 1, 3, 4).reshape(n, c, hh, ww)
