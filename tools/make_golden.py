#!/usr/bin/env python
"""Generates tests/golden/*.pt by running the UNMODIFIED reference modules (imported read-only through
oracle/ref_import.py; HI3D_REFERENCE_ROOT names the reference checkout) on seeded synthetic weights + inputs, CPU fp32.
The test suite never imports the reference: these small fixtures are what pins parity.  Re-run only where the
reference checkout exists:

    python tools/make_golden.py                  # everything
    python tools/make_golden.py --only-video     # the temporal VideoDecoder fixture
    python tools/make_golden.py --only-oracle    # the fixtures of tests/test_oracle_vs_reference.py
    python tools/make_golden.py --only-cpu-surface   # samplers, conditioner pieces, inference configs
    python tools/make_golden.py --only-cpu-samplers  # ancestral, LMS and churned EDM samplers (test_samplers_more_cpu.py)
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_import as R  # noqa: E402
from hi3d_official_b200 import spec  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
UNET_KW = dict(R.UNET_S1, model_channels=64)
UNET2_KW = dict(R.UNET_S2, model_channels=64)
VAE_DD = dict(R.VAE_DD, ch=64)


def cond(T, cc, adm, hw, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(T, 4, hw, hw, generator=g)
    c = dict(crossattn=torch.randn(1, 1, 1024, generator=g), vector=torch.randn(1, adm, generator=g),
             concat=torch.randn(T, cc, hw, hw, generator=g) * 0.18)
    uc = dict(crossattn=torch.zeros(1, 1, 1024), vector=c["vector"].clone(), concat=torch.zeros(T, cc, hw, hw))
    return x, c, uc


@torch.no_grad()
def video_decoder_fixture():
    """SURVEY 8f N1: the unmodified temporal_ae.VideoDecoder (time_mode 'conv-only', video_kernel_size [3, 1, 1]) run as
    Decoder.forward(z, timesteps=T) on seeded synthetic weights, 2 clips x 4 frames, 8x8 latents."""
    R.setup()
    from sgm.modules.autoencoding.temporal_ae import VideoDecoder
    dd = dict(VAE_DD, attn_type="vanilla")
    cfg = spec.VAEConfig.from_ddconfig(VAE_DD, 4)
    sd = spec.synth_state_dict(spec.video_decoder_param_shapes(cfg, (3, 1, 1)), seed=2)
    ref = VideoDecoder(**dd, video_kernel_size=[3, 1, 1], time_mode="conv-only").eval()
    ref.load_state_dict({k[len("decoder."):]: v for k, v in sd.items()}, strict=True)
    T = 4
    g = torch.Generator().manual_seed(8)
    z = torch.randn(2 * T, 4, 8, 8, generator=g)
    out = ref(z, timesteps=T)
    fix = dict(ddconfig=VAE_DD, seed=2, T=T, z=z, dec=out, video_kernel_size=[3, 1, 1])
    torch.save(fix, os.path.join(OUT, "vae_video_ch64.pt"))
    print("video decoder", tuple(out.shape), float(out.abs().mean()))


def _shapes(module, prefix=""):
    return {prefix + k: tuple(v.shape) for k, v in module.state_dict().items()}


def _oracle_inputs(cin_cat=4, adm=768, hw=16, T=4, seed=0):
    """tests/test_oracle_vs_reference.py::_inputs"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(T, 4, hw, hw, generator=g)
    c = dict(crossattn=torch.randn(1, 1, 1024, generator=g), vector=torch.randn(1, adm, generator=g),
             concat=torch.randn(T, cin_cat, hw, hw, generator=g) * 0.18)
    uc = dict(crossattn=torch.zeros(1, 1, 1024), vector=c["vector"].clone(), concat=torch.zeros(T, cin_cat, hw, hw))
    return x, c, uc


@torch.no_grad()
def oracle_fixtures():
    """What tests/test_oracle_vs_reference.py compares the oracle restatement against, from the unmodified reference: the
    parameter shapes of the full-size modules (meta device) and the outputs of the small seeded cases of each test."""
    R.setup()
    from sgm.models.autoencoder import AutoencoderKL  # noqa: F401
    from sgm.modules.autoencoding.temporal_ae import VideoDecoder
    from sgm.modules.diffusionmodules.model import Decoder, Encoder
    from sgm.modules.diffusionmodules.video_model import VideoUNet
    small = dict(model_channels=64, channel_mult=[1, 2, 4, 4], adm_in_channels=768)
    shapes = {}
    with torch.device("meta"):
        shapes["unet_s1"] = _shapes(VideoUNet(**R.UNET_S1))
        shapes["unet_s2"] = _shapes(VideoUNet(**R.UNET_S2))
        shapes["vae_full"] = dict(_shapes(Encoder(**R.VAE_DD), "encoder."), **_shapes(Decoder(**R.VAE_DD), "decoder."))
        for vks in ([3, 1, 1], 3):
            shapes[f"video_decoder_{vks}"] = _shapes(
                VideoDecoder(**dict(R.VAE_DD, attn_type="vanilla"), video_kernel_size=vks, time_mode="conv-only"), "decoder.")
    # small UNet: forward and 3-step sampler
    torch.manual_seed(0)
    ref = R.build_unet(**small)
    shapes["unet_small"] = _shapes(ref)
    sd = spec.synth_state_dict(spec.unet_param_shapes(spec.UNetConfig.from_kwargs(**dict(R.UNET_S1, **small))), seed=1)
    ref.load_state_dict(sd, strict=True)
    T = 4
    x, c, uc = _oracle_inputs(T=T)
    xin = torch.cat([torch.cat([x, x]), torch.cat([uc["concat"], c["concat"]])], 1)
    fwd = ref(xin, timesteps=torch.full((2 * T,), 0.7), context=torch.cat([uc["crossattn"], c["crossattn"]]),
              y=torch.cat([uc["vector"], c["vector"]]), num_video_frames=T, image_only_indicator=torch.zeros(2, T))
    x, c, uc = _oracle_inputs(T=T, seed=3)
    smp = R.build_sampler(num_steps=3, max_scale=2.5, num_frames=T)
    den, net = R.build_denoiser(), R.wrap(ref)
    kw = dict(image_only_indicator=torch.zeros(2, T), num_video_frames=T)
    sampled = smp(lambda inp, s, cc: den(net, inp, s, cc, **kw), x.clone(), cond=c, uc=uc)
    sigmas25 = R.build_sampler().discretization(25, device="cpu")
    torch.save(dict(shapes=shapes, unet_forward=fwd, sampled3=sampled, sigmas25=sigmas25),
               os.path.join(OUT, "oracle_ref_unet.pt"))
    # small VAE: encode (mode / sampled) and decode; the reference draws its own weights' init and the image from the global RNG
    torch.manual_seed(0)
    ae = R.build_vae(sample=False, ch=32, ch_mult=[1, 2, 4, 4])
    vae_shapes = _shapes(ae)
    sdv = spec.synth_state_dict(spec.vae_param_shapes(spec.VAEConfig.from_ddconfig(dict(R.VAE_DD, ch=32), 4)), seed=2)
    ae.load_state_dict(sdv, strict=True)
    img = torch.rand(2, 3, 64, 64) * 2 - 1
    z_mode = ae.encode(img)
    z = torch.randn(2, 4, 8, 8)
    dec = ae.decode(z)
    ae.regularization.sample = True
    torch.manual_seed(7)
    z_sampled = ae.encode(img)
    # temporal VideoDecoder: the test's own seeded weights (drawn in the reference's state_dict order), 2 clips x 3 frames
    video = {}
    for vks in ([3, 1, 1], 3):
        torch.manual_seed(0)
        dd = dict(R.VAE_DD, ch=32, ch_mult=[1, 2, 4, 4], attn_type="vanilla")
        vd = VideoDecoder(**dd, video_kernel_size=vks, time_mode="conv-only").eval()
        g = torch.Generator().manual_seed(11)
        sdd = {}
        for k, v in vd.state_dict().items():
            if k.endswith("mix_factor"):
                sdd[k] = torch.full_like(v, 0.3)
            elif v.ndim == 1 and ("norm" in k or "in_layers.0" in k or "out_layers.0" in k) and k.endswith("weight"):
                sdd[k] = 1.0 + 0.1 * torch.randn(v.shape, generator=g)
            elif v.ndim == 1:
                sdd[k] = 0.05 * torch.randn(v.shape, generator=g)
            else:
                sdd[k] = torch.randn(v.shape, generator=g) * v[0].numel() ** -0.5
        vd.load_state_dict(sdd, strict=True)
        zt = torch.randn(6, 4, 8, 8, generator=g)
        a = vd(zt, timesteps=3)
        a2 = vd(zt.flip(0), timesteps=3).flip(0)
        video[str(vks)] = dict(shapes=_shapes(vd), dec=a, flip_max_diff=float((a2 - a).abs().max()))
    torch.save(dict(shapes=vae_shapes, img=img, z=z, z_mode=z_mode, dec=dec, z_sampled=z_sampled),
               os.path.join(OUT, "oracle_ref_vae.pt"))
    torch.save(video, os.path.join(OUT, "oracle_ref_video_decoder.pt"))
    print("oracle fixtures", float(fwd.abs().mean()), float(sampled.abs().mean()), float(dec.abs().mean()))


@torch.no_grad()
def cpu_surface_fixtures():
    """What tests/test_samplers_cpu.py and tests/test_conditioner_cpu.py compare against: the reference samplers on the
    analytic toy denoiser, the reference conditioner pieces, and the two inference configs (data) of the reference."""
    import shutil
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import test_samplers_cpu as TS
    R.setup()
    import sgm.modules.diffusionmodules.sampling as RS
    from sgm.modules.encoders.modules import ConcatTimestepEmbedderND, VideoPredictionEmbedderWithEncoder
    samplers = {}
    for name in ("EulerEDMSampler", "HeunEDMSampler", "DPMPP2MSampler"):
        for guider in TS.GUIDERS:
            kw = dict(num_steps=7, device="cpu", verbose=False, discretization_config=TS.DISC, guider_config=TS.GUIDERS[guider])
            c, uc = TS._cond()
            x0 = torch.randn(4, 4, 6, 6, generator=torch.Generator().manual_seed(9))
            samplers[f"{name}/{guider}"] = getattr(RS, name)(**kw)(TS.toy_denoiser, x0.clone(), cond=c, uc=uc)
    g = torch.Generator().manual_seed(0)
    ts_in = [torch.rand(3, generator=g) * 30, torch.rand(2, 3, generator=g) * 5, torch.tensor([0.02])]
    ts_out = [ConcatTimestepEmbedderND(256)(x) for x in ts_in]
    vid = torch.arange(2 * 3 * 4 * 5 * 5, dtype=torch.float32).reshape(6, 4, 5, 5)
    vp = {f"{ncf}/{ncp}": VideoPredictionEmbedderWithEncoder(n_cond_frames=ncf, n_copies=ncp, encoder_config={"target": "torch.nn.Identity"},
                                                             scale_factor=0.5, disable_encoder_autocast=True)(vid.clone())
          for ncf, ncp in ((3, 1), (1, 4), (3, 2))}
    torch.save(dict(samplers=samplers, timestep_in=ts_in, timestep_out=ts_out, video_prediction=vp),
               os.path.join(OUT, "ref_cpu_surface.pt"))
    for name in ("inference-v01.yaml", "inference-v02.yaml"):
        shutil.copyfile(os.path.join(R.REF_ROOT, "configs", name), os.path.join(OUT, name))
    print("cpu surface fixtures", len(samplers))


@torch.no_grad()
def cpu_sampler_fixtures():
    """What tests/test_samplers_more_cpu.py compares against: the reference's ancestral, linear multistep and churned EDM
    samplers x every guider on the analytic toy denoiser, with the noise injected as that test injects it."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import test_samplers_more_cpu as TM
    R.setup()
    import sgm.modules.diffusionmodules.sampling as RS
    out = {}
    for case, (name, extra) in TM.CASES.items():
        for guider in TM.GUIDERS:
            smp = getattr(RS, name)(**TM.sampler_kwargs(guider), **extra)
            out[f"{case}/{guider}"] = TM.run(smp)
    torch.save(dict(samplers=out), os.path.join(OUT, "ref_cpu_samplers.pt"))
    print("cpu sampler fixtures", len(out))


@torch.no_grad()
def main():
    os.makedirs(OUT, exist_ok=True)
    if "--only-cpu-samplers" in sys.argv:
        cpu_sampler_fixtures()
        return
    if "--only-cpu-surface" in sys.argv:
        cpu_surface_fixtures()
        return
    if "--only-video" in sys.argv:
        video_decoder_fixture()
        return
    if "--only-oracle" in sys.argv:
        oracle_fixtures()
        return
    torch.manual_seed(0)
    # ---- stage-1 style UNet (8 input channels), T=4, 16x16 latents: denoiser outputs at 3 sigmas + 3-step sampler
    for tag, kw, cc, adm, scale in (("s1", UNET_KW, 4, 768, 2.5), ("s2", UNET2_KW, 13, 512, 2.0)):
        T, hw = 4, 16
        ref = R.build_unet(**kw)
        sd = spec.synth_state_dict(spec.unet_param_shapes(spec.UNetConfig.from_kwargs(**kw)), seed=1)
        ref.load_state_dict(sd, strict=True)
        net, den = R.wrap(ref), R.build_denoiser()
        x, c, uc = cond(T, cc, adm, hw, seed=11)
        kwm = dict(image_only_indicator=torch.zeros(2, T), num_video_frames=T)
        smp = R.build_sampler(num_steps=3, max_scale=scale, num_frames=T)
        fix = dict(unet_kwargs=kw, seed=1, T=T, hw=hw, x=x, c=c, uc=uc, max_scale=scale, denoised={}, euler={})
        for sigma in (700.0, 10.0, 0.5):
            xs = x * (1 + sigma ** 2) ** 0.5
            s = torch.full((T,), sigma)
            d = smp.denoise(xs, lambda i, sg, cc_: den(net, i, sg, cc_, **kwm), s, c, uc)     # CFG-combined D(x, sigma)
            fix["denoised"][sigma] = d
            fix["euler"][sigma] = smp.sampler_step(s, s * 0.7, lambda i, sg, cc_: den(net, i, sg, cc_, **kwm), xs, c, uc)
        fix["sampled3"] = smp(lambda i, sg, cc_: den(net, i, sg, cc_, **kwm), x.clone(), cond=c, uc=uc)
        torch.save(fix, os.path.join(OUT, f"unet_{tag}_mc64.pt"))
        print(tag, {k: float(v.abs().mean()) for k, v in fix["denoised"].items()}, float(fix["sampled3"].abs().mean()))
    # ---- VAE ch=64: mode-encode, sampled encode (CPU RNG, as the reference draws it), decode
    ae = R.build_vae(sample=True, **{k: v for k, v in VAE_DD.items()})
    sdv = spec.synth_state_dict(spec.vae_param_shapes(spec.VAEConfig.from_ddconfig(VAE_DD, 4)), seed=2)
    ae.load_state_dict(sdv, strict=True)
    g = torch.Generator().manual_seed(5)
    img = torch.rand(2, 3, 128, 128, generator=g) * 2 - 1
    z_in = torch.randn(2, 4, 16, 16, generator=g)
    torch.manual_seed(77)
    z_sampled = ae.encode(img)
    torch.manual_seed(77)
    noise = torch.randn(2, 4, 16, 16)
    ae.regularization.sample = False
    fix = dict(ddconfig=VAE_DD, seed=2, img=img, z_in=z_in, noise=noise, z_mode=ae.encode(img), z_sampled=z_sampled,
               dec=ae.decode(z_in))
    torch.save(fix, os.path.join(OUT, "vae_ch64.pt"))
    print("vae", float(fix["z_mode"].abs().mean()), float(fix["dec"].abs().mean()))
    video_decoder_fixture()
    oracle_fixtures()
    cpu_surface_fixtures()
    cpu_sampler_fixtures()


if __name__ == "__main__":
    main()
