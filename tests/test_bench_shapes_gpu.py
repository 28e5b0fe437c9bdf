"""Parity WHERE THE BENCHMARK RUNS (VERDICT r01, "What's weak" 1-3): the code paths `bench.py` times are only entered at
benchmark shapes -- tile pairs (`gemm_tc5_kernel<BN, 2>`: K >= 1920 and enough tiles), the wgmma FMHA inside the
network (L >= 512 with 5/10/20 heads), the full-width UNet at 64x64 (configs[1]) and 128x128 x 17 channels (configs[2])
latents, the stage-2 re-noise loop, and the VAE mid-block attention at L = 4096.

The oracle (oracle/hi3d_oracle.py, plain PyTorch) runs on the same GPU in fp32 with TF32 off (tests/conftest.py), so a
64x64 teacher-forced D(x, sigma) costs seconds.  Network-level bar = the north-star tolerance on the guided denoised
latents: rtol 1e-3, atol 1e-2, ZERO elements outside.  Every test prints its max|err| line.
"""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from hi3d_official_b200 import _native, configs, ops, pack, sampling, spec  # noqa: E402
from hi3d_official_b200.unet import VideoUNet  # noqa: E402
from oracle import hi3d_oracle as O  # noqa: E402
from test_kernels_gpu import DEV, H, close, nhwc, rnd  # noqa: E402


def _stats(a, b, name, rtol=1e-3, atol=1e-2):
    a, b = a.float(), b.float()
    err = (a - b).abs()
    frac = float((err > atol + rtol * b.abs()).float().mean())
    print(f"[bench-shape parity] {name}: max|err| {float(err.max()):.3e} mean|err| {float(err.mean()):.3e} "
          f"ref mean|x| {float(b.abs().mean()):.3e} max|x| {float(b.abs().max()):.3e} frac outside({atol:g},{rtol:g}) {frac:.2e}")
    return float(err.max()), frac


# ------------------------------------------------------------------------------------------------------------------
# (a) tile-pair GEMM: shapes the automatic rule sends to gemm_tc5_kernel<BN, 2>, plus every tc5 geometry with pairs forced
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def pair_mode():
    lib = _native.load()

    def set_(m):
        _native.check(lib.hi3d_gemm_tc5_set_pair_mode(m), "set_pair_mode")
    yield set_
    set_(-1)


@pytest.mark.parametrize("mode", [-1, 1, 0])
def test_pair_conv3x3_c320_64x64x32(pair_mode, mode):
    """stage-1 top level ResBlock conv: 32 images x 64 x 64, C = 320 -> K = 2880, 1024 row tiles (auto rule -> pairs)."""
    pair_mode(mode)
    n, c, hh = 32, 320, 64
    x = rnd(n, c, hh, hh, seed=11)
    w = rnd(c, c, 3, 3, scale=(9 * c) ** -0.5, seed=12)
    b = rnd(c, scale=0.1, seed=13)
    emb = rnd(n, c, scale=0.5, seed=14).to(H)
    xh = nhwc(x)
    M = n * hh * hh
    out = torch.zeros(M, c, dtype=H, device=DEV)
    ops.Gemm(ops.conv_taps([xh]), pack.pack_conv2d(w), out, M, mode=ops.ROWS_CONV2D, geom=dict(Ho=hh, Wo=hh, Hs=hh, Ws=hh),
             bias=b, rowbias=emb, rb_div=hh * hh, rb_mod=n, engine="tc5")()
    ref = F.conv2d(xh.permute(0, 3, 1, 2).float(), w.to(H).float(), b, padding=1) + emb.float()[:, :, None, None]
    close(out.view(n, hh, hh, c).permute(0, 3, 1, 2), ref, name=f"pair conv3x3 C=320 mode={mode}")


@pytest.mark.parametrize("mode", [-1, 1, 0])
def test_pair_temporal_conv_c640(pair_mode, mode):
    """temporal (3,1,1) conv at C = 640, 32x32 level: K = 1920, M = 32768 (auto rule -> pairs), with residual + blend."""
    pair_mode(mode)
    b_, c, T, hw = 2, 640, 16, 1024
    M = b_ * T * hw
    xh = rnd(M, c, seed=21).to(H)
    w = rnd(c, c, 3, 1, 1, scale=(3 * c) ** -0.5, seed=22)
    bias = rnd(c, scale=0.1, seed=23)
    res = rnd(M, c, seed=24).to(H)
    out = torch.zeros(M, c, dtype=H, device=DEV)
    ops.Gemm(ops.temporal_taps(xh), pack.pack_conv3d_t(w), out, M, mode=ops.ROWS_TEMPORAL, geom=dict(Ho=hw, Wo=1, T=T),
             bias=bias, residual=res, blend_x=res, alpha=0.4, engine="tc5")()
    xr = xh.view(b_, T, hw, 1, c).permute(0, 4, 1, 2, 3).float()
    conv = F.conv3d(xr, w.to(H).float(), bias, padding=(1, 0, 0)).permute(0, 2, 3, 4, 1).reshape(M, c)
    ref = 0.4 * res.float() + 0.6 * (conv.to(H).float() + res.float())
    close(out, ref, name=f"pair temporal conv C=640 mode={mode}")


@pytest.mark.parametrize("mode", [-1, 1, 0])
def test_pair_ff2_c640(pair_mode, mode):
    """FeedForward output projection at C = 640: [32768, 2560] x [640, 2560]^T + bias + residual (K = 2560 -> pairs)."""
    pair_mode(mode)
    M, K, N = 32768, 2560, 640
    a = rnd(M, K, seed=31).to(H)
    w = rnd(N, K, scale=K ** -0.5, seed=32).to(H)
    bias = rnd(N, scale=0.1, seed=33)
    res = rnd(M, N, seed=34).to(H)
    out = torch.zeros(M, N, dtype=H, device=DEV)
    ops.Gemm([ops.SegSpec(a)], w, out, M, bias=bias, residual=res, engine="tc5")()
    close(out, (a.float() @ w.float().t() + bias).to(H).float() + res.float(), name=f"pair ff2 C=640 mode={mode}")


@pytest.mark.parametrize("M,N,K", [(256, 256, 128), (300, 320, 320), (1000, 960, 640), (4096, 1280, 1280), (257, 2560, 320)])
def test_forced_pair_plain_epilogues(pair_mode, M, N, K):
    """The plain-rows tc5 cases of test_gemm_tc5_gpu.py re-run with tile pairs forced (ragged M, odd tile counts)."""
    pair_mode(1)
    a = rnd(M, K).to(H)
    w = rnd(N, K, scale=K ** -0.5).to(H)
    bias = rnd(N, scale=0.1)
    rb = rnd(5, N, scale=0.5).to(H)
    res = rnd(M, N).to(H)
    out = torch.zeros(M, N, dtype=H, device=DEV)
    ref0 = a.float() @ w.float().t()
    ops.Gemm([ops.SegSpec(a)], w, out, M, engine="tc5")()
    close(out, ref0, name="pair plain")
    ops.Gemm([ops.SegSpec(a)], w, out, M, bias=bias, rowbias=rb, rb_div=7, rb_mod=5, residual=res, engine="tc5")()
    idx = (torch.arange(M, device=DEV) // 7) % 5
    close(out, (ref0 + bias + rb.float()[idx]).to(H).float() + res.float(), name="pair bias+rowbias+res")
    ops.Gemm([ops.SegSpec(a)], w, out, M, bias=bias, act=ops.ACT_SILU, engine="tc5")()
    close(out, F.silu(ref0 + bias), name="pair silu")


def test_forced_pair_geglu_conv_concat_stride2(pair_mode):
    pair_mode(1)
    M, C = 513, 320
    a = rnd(M, C).to(H)
    w, b = rnd(8 * C, C, scale=C ** -0.5), rnd(8 * C, scale=0.1)
    wp, bp = pack.pack_geglu(w, b)
    out = torch.zeros(M, 4 * C, dtype=H, device=DEV)
    ops.Gemm([ops.SegSpec(a)], wp, out, M, bias=bp, act=ops.ACT_GEGLU, engine="tc5")()
    v, g = (a.float() @ w.to(H).float().t() + b).chunk(2, dim=-1)
    close(out, v * F.gelu(g), name="pair geglu")
    # conv over a virtual concat + fused 1x1 skip
    n, c1, c2, co, hh = 4, 64, 128, 64, 16
    x1, x2, hcur = rnd(n, c1, hh, hh), rnd(n, c2, hh, hh, seed=2), rnd(n, co, hh, hh, seed=3)
    w3 = rnd(co, co, 3, 3, scale=(9 * co) ** -0.5)
    ws_ = rnd(co, c1 + c2, 1, 1, scale=(c1 + c2) ** -0.5)
    b3 = rnd(co, scale=0.1)
    x1h, x2h, hh_ = nhwc(x1), nhwc(x2), nhwc(hcur)
    segs = ops.conv_taps([hh_]) + [ops.SegSpec(x1h), ops.SegSpec(x2h)]
    Wt = pack.cat_k(pack.pack_conv2d(w3), pack.pack_conv2d(ws_))
    Mc = n * hh * hh
    oc = torch.zeros(Mc, co, dtype=H, device=DEV)
    ops.Gemm(segs, Wt, oc, Mc, mode=ops.ROWS_CONV2D, geom=dict(Ho=hh, Wo=hh, Hs=hh, Ws=hh), bias=b3, engine="tc5")()
    xr = torch.cat([x1h, x2h], -1).permute(0, 3, 1, 2).float()
    ref = F.conv2d(hh_.permute(0, 3, 1, 2).float(), w3.to(H).float(), b3, padding=1) + F.conv2d(xr, ws_.to(H).float())
    close(oc.view(n, hh, hh, co).permute(0, 3, 1, 2), ref, name="pair conv+skip")
    # stride-2 conv (TMA element strides) and the parity-class up-conv
    n, ci, co, hs = 4, 128, 64, 32
    x, w = rnd(n, ci, hs, hs), rnd(co, ci, 3, 3, scale=(9 * ci) ** -0.5)
    bb = rnd(co, scale=0.1)
    xh = nhwc(x)
    ref = F.conv2d(xh.permute(0, 3, 1, 2).float(), w.to(H).float(), bb, stride=2, padding=1)
    ho = ref.shape[2]
    o2 = torch.zeros(n * ho * ho, co, dtype=H, device=DEV)
    ops.Gemm(ops.conv_taps([xh]), pack.pack_conv2d(w), o2, n * ho * ho, mode=ops.ROWS_CONV2D,
             geom=dict(Ho=ho, Wo=ho, Hs=hs, Ws=hs, stride=2), bias=bb, engine="tc5")()
    close(o2.view(n, ho, ho, co).permute(0, 3, 1, 2), ref, name="pair stride2")
    refu = F.conv2d(F.interpolate(xh.permute(0, 3, 1, 2).float(), scale_factor=2, mode="nearest"), w.to(H).float(), bb, padding=1)
    o3 = torch.zeros(n * 4 * hs * hs, co, dtype=H, device=DEV)
    for (py, px), (Wp, shifts) in pack.pack_upconv_parity(w).items():
        ops.Gemm([ops.SegSpec(xh, dy=sy, dx=sx) for sy, sx in shifts], Wp, o3, n * hs * hs, mode=ops.ROWS_CONV2D,
                 geom=dict(Ho=hs, Wo=hs, Hs=hs, Ws=hs, out_up=1, out_py=py, out_px=px), bias=bb, engine="tc5")()
    close(o3.view(n, 2 * hs, 2 * hs, co).permute(0, 3, 1, 2), refu, rtol=4e-3, name="pair upconv parity")


# ------------------------------------------------------------------------------------------------------------------
# (b) full-width teacher-forced D(x, sigma) at the benchmark latent sizes
# ------------------------------------------------------------------------------------------------------------------
_CACHE = {}


def _full_model(stage: int):
    """(engine, oracle state dict on the GPU) of the full-width stage-`stage` configuration, synthetic weights (seed 1)."""
    if stage not in _CACHE:
        _CACHE.clear()                                       # one 1.5 B-parameter model (+ fp32 oracle copy) at a time
        torch.cuda.empty_cache()
        model = configs.build_engine(stage, device=DEV)
        spec.synth_fill_(model, seed=1, fast=False)
        sd = {k: v.float() for k, v in model.model.diffusion_model.state_dict().items()}
        _CACHE[stage] = (model, sd)
    return _CACHE[stage]


def _cond(stage: int, h: int, T: int = 16, seed: int = 5):
    g = torch.Generator().manual_seed(seed)
    cc, adm = (4, 768) if stage == 1 else (13, 512)
    x = torch.randn(T, 4, h, h, generator=g).to(DEV)
    c = dict(crossattn=torch.randn(1, 1, 1024, generator=g).to(DEV), vector=torch.randn(1, adm, generator=g).to(DEV),
             concat=(torch.randn(T, cc, h, h, generator=g) * 0.18).to(DEV))
    uc = dict(crossattn=torch.zeros_like(c["crossattn"]), vector=c["vector"], concat=torch.zeros_like(c["concat"]))
    return x, c, uc


def _teacher_forced(stage: int, h: int, sigmas):
    model, sd = _full_model(stage)
    T = 16
    x, c, uc = _cond(stage, h)
    max_scale = 2.5 if stage == 1 else 2.0
    scale = O.guider_scale(T, max_scale)
    smp = model.sampler
    den = model.bind_denoiser(image_only_indicator=None, num_video_frames=T)
    worst = 0.0
    for sigma in sigmas:
        xs = (x * math.sqrt(1.0 + sigma ** 2)).contiguous()
        s = torch.full((T,), float(sigma), device=DEV)
        st = smp._fused_state(den, xs, c, uc, refresh=True)
        assert st is not None, "fused path not taken"
        x_next, d = st.step(xs, s, s * 0.7, want_denoised=True)
        with torch.no_grad():
            ref = O.cfg_denoise(sd, xs, s, c, uc, scale, num_video_frames=T)
        assert torch.isfinite(d).all()
        mx, frac = _stats(d, ref, f"stage {stage} full width, {h}x{h} latents, D(x, sigma={sigma})")
        ref_next = xs + (xs - ref) / sigma * (0.7 * sigma - sigma)
        _stats(x_next, ref_next, f"stage {stage} full width, {h}x{h} latents, euler(sigma={sigma})", atol=1e-2 * max(1.0, 0.3 * sigma))
        worst = max(worst, frac)
        del ref
    return worst


def test_full_width_stage1_64x64_teacher_forced():
    """Stage-1 benchmark shapes: CFG batch 32, 64x64 latents, 1.52 B parameters; wgmma FMHA at L = 4096 / 1024 with
    5 / 10 heads, tile pairs on the 3x3 and temporal convs.  0 elements outside rtol 1e-3 / atol 1e-2."""
    assert _teacher_forced(1, 64, (700.0, 10.0, 0.5)) == 0.0


@pytest.mark.slow
def test_full_width_stage2_128x128_teacher_forced():
    """Stage-2 benchmark shapes: 17 input channels, 128x128 latents (L = 16384 at the top level)."""
    assert _teacher_forced(2, 128, (10.0, 0.5)) == 0.0


# ------------------------------------------------------------------------------------------------------------------
# (c) stage-2 loop: VideoLDMStage2.sample_stage2 against O.sample_v02 (pipeline_i2v_eval_v02.py:86-135)
# ------------------------------------------------------------------------------------------------------------------
def test_sample_stage2_matches_oracle_v02_loop():
    T, h, steps = 8, 16, 3
    model = configs.build_engine(2, device=DEV, unet_overrides=dict(model_channels=64), vae_overrides=dict(ch=64),
                                 num_steps=steps, num_frames=T)
    spec.synth_fill_(model, seed=1, fast=False)
    sd = {k: v.float() for k, v in model.model.diffusion_model.state_dict().items()}
    g = torch.Generator().manual_seed(9)
    init = torch.randn(T, 4, h, h, generator=g).to(DEV)
    z = (torch.randn(T, 4, h, h, generator=g) * 0.18).to(DEV)
    c = dict(crossattn=torch.randn(1, 1, 1024, generator=g).to(DEV), vector=torch.randn(1, 512, generator=g).to(DEV),
             concat=(torch.randn(T, 13, h, h, generator=g) * 0.18).to(DEV))
    uc = dict(crossattn=torch.zeros_like(c["crossattn"]), vector=c["vector"], concat=torch.zeros_like(c["concat"]))
    lat = model.sample_stage2(c, uc, init.clone(), z, decode=False)
    with torch.no_grad():
        ref = O.sample_v02(sd, init.clone(), z, c, uc, num_steps=steps, max_scale=2.0, num_frames=T)
    # the alpha schedule is a known answer (SURVEY App. C): 1.0 at i = 0, then (0.5 (1 + cos(i / n)))^40
    assert O.v02_alpha(0, steps) == 1.0 and abs(O.v02_alpha(1, 25) - 0.98413) < 1e-4
    mx, frac = _stats(lat, ref, f"sample_stage2 free-running {steps} steps (width 64, {h}x{h})")
    assert torch.isfinite(lat).all()
    assert frac < 1e-3 and mx < 5e-2 * max(1.0, float(ref.abs().max()))


# ------------------------------------------------------------------------------------------------------------------
# (d) VAE decode at a 64x64 latent: mid-block AttnBlock at L = 4096 (model.py:180-201)
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ch,hw", [(64, 64), (128, 64)])
def test_vae_decode_64x64_latent(ch, hw):
    from hi3d_official_b200.vae import AutoencoderKL
    dd = dict(configs._VAE_DD, ch=ch)
    cfg = spec.VAEConfig.from_ddconfig(dd, 4)
    sd = spec.synth_state_dict(spec.vae_param_shapes(cfg), seed=3)
    ae = AutoencoderKL(embed_dim=4, ddconfig=dd)
    ae.load_state_dict(sd, strict=True)
    ae = ae.cuda().half()
    g = torch.Generator().manual_seed(4)
    z = torch.randn(1, 4, hw, hw, generator=g).to(DEV)
    dec = ae.decode(z.half(), scale=1.0 / 0.18215)
    with torch.no_grad():
        ref = O.vae_decode({k: v.to(DEV) for k, v in sd.items()}, z.half().float(), scale_factor=0.18215)
    mx, frac = _stats(dec, ref, f"VAE decode ch={ch}, {hw}x{hw} latent (AttnBlock L={hw * hw})", atol=2e-2)
    assert torch.isfinite(dec).all()
    assert frac == 0.0


def test_vae_encode_512_image():
    """Encoder at a 512 x 512 image: mid AttnBlock at L = 4096, asymmetric-pad stride-2 convs at full size."""
    from hi3d_official_b200.vae import AutoencoderKLModeOnly
    dd = dict(configs._VAE_DD)
    cfg = spec.VAEConfig.from_ddconfig(dd, 4)
    sd = spec.synth_state_dict(spec.vae_param_shapes(cfg), seed=3)
    ae = AutoencoderKLModeOnly(embed_dim=4, ddconfig=dd)
    ae.load_state_dict(sd, strict=True)
    ae = ae.cuda().half()
    g = torch.Generator().manual_seed(6)
    img = (torch.rand(1, 3, 512, 512, generator=g) * 2 - 1).to(DEV).half()
    zq = ae.encode(img)
    with torch.no_grad():
        ref = O.vae_encode({k: v.to(DEV) for k, v in sd.items()}, img.float(), scale_factor=1.0)
    mx, frac = _stats(zq, ref, "VAE encode (mode) 512x512 image", atol=2e-2)
    assert frac == 0.0


# ------------------------------------------------------------------------------------------------------------------
# ADVICE r01: reloading weights through the parent engine must invalidate packed weights / plans / graphs
# ------------------------------------------------------------------------------------------------------------------
def test_engine_reload_invalidates_packed_weights():
    T, h = 4, 16
    model = configs.build_engine(1, device=DEV, unet_overrides=dict(model_channels=64), vae_overrides=dict(ch=64),
                                 num_steps=2, num_frames=T)
    spec.synth_fill_(model, seed=1, fast=False)
    x, c, uc = _cond(1, h, T=T)
    a = model.sample_stage1(c, uc, x.clone(), decode=True)
    other = configs.build_engine(1, device=DEV, unet_overrides=dict(model_channels=64), vae_overrides=dict(ch=64),
                                 num_steps=2, num_frames=T)
    spec.synth_fill_(other, seed=2, fast=False)
    want = other.sample_stage1(c, uc, x.clone(), decode=True)
    sd_other = {k: v.clone() for k, v in other.state_dict().items()}
    missing, unexpected = model.load_state_dict(sd_other, strict=False)          # parent load: no override is called
    assert not missing and not unexpected
    b = model.sample_stage1(c, uc, x.clone(), decode=True)
    changed = float((a.float() - b.float()).abs().max())
    same = float((want.float() - b.float()).abs().max())
    print(f"[reload] |old - reloaded| {changed:.3e}   |fresh(new weights) - reloaded| {same:.3e}")
    assert changed > 0.2, "outputs did not change after loading different weights"
    # not bit-equal: the GroupNorm partial sums are combined with shared-memory float atomics (order varies run to run)
    assert same < 0.1 * changed, "reloaded engine differs from a fresh engine on the same weights"
