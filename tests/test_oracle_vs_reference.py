"""Pins the oracle restatement (oracle/hi3d_oracle.py) and the param specs (hi3d_official_b200/spec.py)
against the UNMODIFIED reference modules, through what those modules computed on the same seeded cases: parameter
shapes and outputs stored under tests/golden/oracle_ref_*.pt by tools/make_golden.py --only-oracle."""
import os

import pytest
import torch

from oracle import hi3d_oracle as O
from oracle import ref_import as R
from hi3d_official_b200 import spec

G = os.path.join(os.path.dirname(__file__), "golden")
SMALL = dict(model_channels=64, channel_mult=[1, 2, 4, 4], adm_in_channels=768)
_FIX = {}


def _fix(name):
    if name not in _FIX:
        _FIX[name] = torch.load(os.path.join(G, f"oracle_ref_{name}.pt"), weights_only=False)
    return _FIX[name]


def _inputs(cin_cat=4, adm=768, hw=16, T=4, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(T, 4, hw, hw, generator=g)
    c = dict(crossattn=torch.randn(1, 1, 1024, generator=g), vector=torch.randn(1, adm, generator=g),
             concat=torch.randn(T, cin_cat, hw, hw, generator=g) * 0.18)
    uc = dict(crossattn=torch.zeros(1, 1, 1024), vector=c["vector"].clone(), concat=torch.zeros(T, cin_cat, hw, hw))
    return x, c, uc


@pytest.fixture(scope="module")
def small_unet():
    cfg = spec.UNetConfig.from_kwargs(**dict(R.UNET_S1, **SMALL))
    shapes = spec.unet_param_shapes(cfg)
    assert dict(shapes) == _fix("unet")["shapes"]["unet_small"]
    sd = spec.synth_state_dict(shapes, seed=1)
    return sd


def test_unet_param_spec_full_size_matches_reference_on_meta():
    for tag, kw in (("unet_s1", R.UNET_S1), ("unet_s2", R.UNET_S2)):
        ref_shapes = _fix("unet")["shapes"][tag]
        mine = spec.unet_param_shapes(spec.UNetConfig.from_kwargs(**kw))
        assert dict(mine) == ref_shapes
        assert sum(torch.Size(s).numel() for s in mine.values()) in (1524623082, 1524321322)


def test_unet_forward_matches_reference(small_unet):
    sd = small_unet
    T = 4
    x, c, uc = _inputs(T=T)
    xin = torch.cat([torch.cat([x, x]), torch.cat([uc["concat"], c["concat"]])], 1)
    t = torch.full((2 * T,), 0.7)
    ctx = torch.cat([uc["crossattn"], c["crossattn"]])
    y = torch.cat([uc["vector"], c["vector"]])
    a = _fix("unet")["unet_forward"]
    with torch.no_grad():
        b = O.unet_forward(sd, xin, t, ctx, y, num_video_frames=T)
    assert a.abs().mean() > 1e-2
    torch.testing.assert_close(b, a, rtol=1e-4, atol=2e-4)


def test_sampler_matches_reference(small_unet):
    sd = small_unet
    T, steps = 4, 3
    x, c, uc = _inputs(T=T, seed=3)
    a = _fix("unet")["sampled3"]
    with torch.no_grad():
        b = O.sample(sd, x.clone(), c, uc, num_steps=steps, max_scale=2.5, num_frames=T)
    torch.testing.assert_close(b, a, rtol=1e-4, atol=1e-3)


def test_sampler_constants():
    s = O.edm_sigmas(25)
    ref = _fix("unet")["sigmas25"]
    torch.testing.assert_close(s, ref, rtol=0, atol=0)
    assert abs(float(s[0]) - 700.0001) < 1e-3 and float(s[-1]) == 0.0 and abs(float(s[-2]) - 0.002) < 1e-6
    cs = O.vscaling_edm_cnoise(torch.tensor(700.0))
    assert abs(float(cs[3]) - 1.6377701) < 1e-6 and abs(float(cs[2]) - 1.4285699e-03) < 1e-9
    assert abs(O.v02_alpha(1) - 0.984126) < 1e-6 and O.v02_alpha(0) == 1.0


def test_single_key_cross_attention_is_constant(small_unet):
    """SURVEY F7: attn2 with one context token == to_out(to_v(ctx)) for every query."""
    sd = small_unet
    pre = "input_blocks.1.1.transformer_blocks.0.attn2."
    x = torch.randn(3, 10, 64)
    ctx = torch.randn(3, 1, 1024)
    full = O.cross_attention(sd, pre, x, ctx, 1)
    const = torch.nn.functional.linear(torch.nn.functional.linear(ctx, sd[pre + "to_v.weight"]),
                                       sd[pre + "to_out.0.weight"], sd[pre + "to_out.0.bias"])
    torch.testing.assert_close(full, const.expand_as(full), rtol=1e-5, atol=1e-6)


def test_vae_matches_reference():
    fix = _fix("vae")
    cfg = spec.VAEConfig.from_ddconfig(dict(R.VAE_DD, ch=32), 4)
    shapes = spec.vae_param_shapes(cfg)
    assert dict(shapes) == fix["shapes"]
    sd = spec.synth_state_dict(shapes, seed=2)
    img = fix["img"]
    with torch.no_grad():
        zb = O.vae_encode(sd, img, scale_factor=1.0)
        torch.testing.assert_close(zb, fix["z_mode"], rtol=1e-4, atol=1e-4)
        z = fix["z"]
        torch.testing.assert_close(O.vae_decode(sd, z, scale_factor=1.0), fix["dec"], rtol=1e-4, atol=2e-4)
        # sampled posterior: the reference draws CPU randn (distributions.py:37-41)
        zs = fix["z_sampled"]
        torch.manual_seed(7)
        noise = torch.randn(2, 4, 8, 8)
        torch.testing.assert_close(O.vae_encode(sd, img, noise=noise, scale_factor=1.0), zs, rtol=1e-4, atol=1e-4)


def test_vae_full_size_spec_on_meta():
    ref = _fix("unet")["shapes"]["vae_full"]
    mine = {k: v for k, v in spec.vae_param_shapes(spec.VAEConfig.from_ddconfig(R.VAE_DD, 4)).items()
            if not k.startswith(("quant_conv", "post_quant_conv"))}
    assert mine == ref


@pytest.mark.parametrize("vks", [[3, 1, 1], 3])
def test_video_decoder_oracle_matches_reference(vks):
    """SURVEY §8(f) N1: the oracle restatement of temporal_ae.VideoDecoder (time_mode 'conv-only'; kernel (3,1,1) as in
    SVD and the full 3x3x3 default) against the unmodified reference class, seeded synthetic weights."""
    fix = _fix("video_decoder")[str(vks)]
    g = torch.Generator().manual_seed(11)
    sd = {}
    for k, shape in fix["shapes"].items():      # the reference's state_dict order: the draws of g depend on it
        v = torch.empty(shape)
        if k.endswith("mix_factor"):
            sd[k] = torch.full_like(v, 0.3)
        elif v.ndim == 1 and ("norm" in k or "in_layers.0" in k or "out_layers.0" in k) and k.endswith("weight"):
            sd[k] = 1.0 + 0.1 * torch.randn(v.shape, generator=g)
        elif v.ndim == 1:
            sd[k] = 0.05 * torch.randn(v.shape, generator=g)
        else:                       # incl. the zero_module'd out_layers conv of every time_stack (F8)
            fan_in = v[0].numel()
            sd[k] = torch.randn(v.shape, generator=g) * fan_in ** -0.5
    T = 3
    z = torch.randn(2 * T, 4, 8, 8, generator=g)
    a = fix["dec"]
    with torch.no_grad():
        b = O.vae_video_decoder({"decoder." + k: v for k, v in sd.items()}, z, T)
    assert a.shape == (2 * T, 3, 64, 64)
    torch.testing.assert_close(b, a, rtol=1e-4, atol=2e-4)
    # the temporal branch matters: shuffling the frames changes more than a permutation of the output
    assert fix["flip_max_diff"] > 1e-3


@pytest.mark.parametrize("vks", [[3, 1, 1], 3])
def test_video_decoder_param_spec_matches_reference_on_meta(vks):
    ref_shapes = _fix("unet")["shapes"][f"video_decoder_{vks}"]
    mine = spec.video_decoder_param_shapes(spec.VAEConfig.from_ddconfig(R.VAE_DD, 4), vks)
    assert dict(mine) == ref_shapes
