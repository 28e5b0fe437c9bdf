"""Per-kernel parity: every C-ABI entry point against a plain PyTorch fp32 computation of the same op on the
same (fp16-rounded) inputs.  Tolerances are fp16 output rounding (rtol 2e-3) plus a small atol scaled to the
output magnitude -- the kernels accumulate in fp32."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from hi3d_official_b200 import ops, pack  # noqa: E402

DEV = "cuda"
H = torch.float16


def rnd(*shape, scale=1.0, seed=None):
    g = torch.Generator(device="cpu")
    g.manual_seed(seed if seed is not None else (hash(shape) & 0xFFFF))
    return (torch.randn(*shape, generator=g) * scale).to(DEV)


def close(a, b, rtol=2e-3, atol=None, name=""):
    a, b = a.float(), b.float()
    if atol is None:
        atol = 2e-3 * float(b.abs().mean() + 1e-6) + 1e-4
    err = (a - b).abs()
    bad = err > (atol + rtol * b.abs())
    assert not bool(bad.any()), (f"{name}: {int(bad.sum())}/{bad.numel()} outside tol; max abs err {float(err.max()):.4e} "
                                 f"ref mean|x| {float(b.abs().mean()):.3e}")


def nhwc(x):  # NCHW fp32 -> NHWC fp16 contiguous
    return x.permute(0, 2, 3, 1).contiguous().to(H)


# ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,N,K", [(300, 320, 320), (128, 128, 64), (1000, 960, 640), (64, 8, 128), (257, 2560, 320)])
def test_gemm_plain_epilogues(M, N, K):
    a = rnd(M, K).to(H)
    w = rnd(N, K, scale=K ** -0.5).to(H)
    bias = rnd(N, scale=0.1)
    rb = rnd(5, N, scale=0.5).to(H)
    res = rnd(M, N).to(H)
    out = torch.zeros(M, N, dtype=H, device=DEV)
    ref0 = a.float() @ w.float().t()
    # plain
    ops.Gemm([ops.SegSpec(a)], w, out, M)()
    close(out, ref0, name="plain")
    # bias + rowbias(div 7, mod 5) + residual
    ops.Gemm([ops.SegSpec(a)], w, out, M, bias=bias, rowbias=rb, rb_div=7, rb_mod=5, residual=res)()
    idx = (torch.arange(M, device=DEV) // 7) % 5
    ref = (ref0 + bias + rb.float()[idx]).to(H).float() + res.float()
    close(out, ref, name="bias+rowbias+res")
    # silu
    ops.Gemm([ops.SegSpec(a)], w, out, M, bias=bias, act=ops.ACT_SILU)()
    close(out, F.silu(ref0 + bias), name="silu")
    # blend
    bx = rnd(M, N, seed=5).to(H)
    ops.Gemm([ops.SegSpec(a)], w, out, M, bias=bias, residual=res, blend_x=bx, alpha=0.3)()
    ref = 0.3 * bx.float() + 0.7 * ((ref0 + bias).to(H).float() + res.float())
    close(out, ref, name="blend")


@pytest.mark.parametrize("M,C", [(200, 64), (513, 320)])
def test_gemm_geglu(M, C):
    a = rnd(M, C).to(H)
    w = rnd(8 * C, C, scale=C ** -0.5)
    b = rnd(8 * C, scale=0.1)
    wp, bp = pack.pack_geglu(w, b)
    out = torch.zeros(M, 4 * C, dtype=H, device=DEV)
    ops.Gemm([ops.SegSpec(a)], wp, out, M, bias=bp, act=ops.ACT_GEGLU)()
    y = a.float() @ w.to(H).float().t() + b
    v, g = y.chunk(2, dim=-1)
    close(out, v * F.gelu(g), name="geglu")


def test_gemm_two_segment_k_concat():
    M = 200
    a1, a2 = rnd(M, 128).to(H), rnd(M, 64, seed=2).to(H)
    w = rnd(192, 192, scale=192 ** -0.5).to(H)
    out = torch.zeros(M, 192, dtype=H, device=DEV)
    ops.Gemm([ops.SegSpec(a1), ops.SegSpec(a2)], w, out, M)()
    close(out, torch.cat([a1, a2], 1).float() @ w.float().t(), name="kconcat")
    # channel sub-range of a wider tensor
    big = rnd(M, 256, seed=3).to(H)
    w2 = rnd(64, 128, scale=128 ** -0.5).to(H)
    out2 = torch.zeros(M, 64, dtype=H, device=DEV)
    ops.Gemm([ops.SegSpec(big, 128, c_off=64)], w2, out2, M)()
    close(out2, big[:, 64:192].float() @ w2.float().t(), name="c_off")


@pytest.mark.parametrize("stride,ups,asym", [(1, 0, False), (2, 0, False), (1, 1, False), (2, 0, True)])
def test_gemm_conv3x3(stride, ups, asym):
    n, ci, co, hs, ws = 3, 64, 128, 12, 10
    x = rnd(n, ci, hs, ws)
    w = rnd(co, ci, 3, 3, scale=(9 * ci) ** -0.5)
    b = rnd(co, scale=0.1)
    xh = nhwc(x)
    xr, wr = xh.permute(0, 3, 1, 2).float(), w.to(H).float()
    if ups:
        ref = F.conv2d(F.interpolate(xr, scale_factor=2, mode="nearest"), wr, b, padding=1)
    elif asym:
        ref = F.conv2d(F.pad(xr, (0, 1, 0, 1)), wr, b, stride=2)
    else:
        ref = F.conv2d(xr, wr, b, stride=stride, padding=1)
    ho, wo = ref.shape[2:]
    out = torch.zeros(n * ho * wo, co, dtype=H, device=DEV)
    segs = ops.conv_taps([xh], pad_lo=0 if asym else 1)
    ops.Gemm(segs, pack.pack_conv2d(w), out, n * ho * wo, mode=ops.ROWS_CONV2D,
             geom=dict(Ho=ho, Wo=wo, Hs=hs, Ws=ws, stride=stride, ups=ups), bias=b)()
    close(out.view(n, ho, wo, co).permute(0, 3, 1, 2), ref, name=f"conv s{stride} u{ups} a{asym}")


def test_gemm_conv_concat_skip_emb():
    """ResBlock second half as one GEMM: conv3x3(h) + 1x1 skip over the virtual concat [x1 | x2] + bias."""
    n, c1, c2, co, hh, ww = 4, 64, 128, 64, 8, 8
    x1, x2, hcur = rnd(n, c1, hh, ww), rnd(n, c2, hh, ww, seed=2), rnd(n, co, hh, ww, seed=3)
    w3 = rnd(co, co, 3, 3, scale=(9 * co) ** -0.5)
    ws_ = rnd(co, c1 + c2, 1, 1, scale=(c1 + c2) ** -0.5)
    b3, bs = rnd(co, scale=0.1), rnd(co, scale=0.1, seed=9)
    x1h, x2h, hh_ = nhwc(x1), nhwc(x2), nhwc(hcur)
    segs = ops.conv_taps([hh_]) + [ops.SegSpec(x1h), ops.SegSpec(x2h)]
    W = pack.cat_k(pack.pack_conv2d(w3), pack.pack_conv2d(ws_))
    M = n * hh * ww
    out = torch.zeros(M, co, dtype=H, device=DEV)
    ops.Gemm(segs, W, out, M, mode=ops.ROWS_CONV2D, geom=dict(Ho=hh, Wo=ww, Hs=hh, Ws=ww), bias=(b3 + bs))()
    xr = torch.cat([x1h, x2h], -1).permute(0, 3, 1, 2).float()
    ref = F.conv2d(hh_.permute(0, 3, 1, 2).float(), w3.to(H).float(), b3, padding=1) + \
        F.conv2d(xr, ws_.to(H).float(), bs)
    close(out.view(n, hh, ww, co).permute(0, 3, 1, 2), ref, name="conv+skip")
    # first half: conv over the concat with per-sample emb rowbias
    w1 = rnd(co, c1 + c2, 3, 3, scale=(9 * (c1 + c2)) ** -0.5)
    emb = rnd(n, co, scale=0.5).to(H)
    ops.Gemm(ops.conv_taps([x1h, x2h]), pack.pack_conv2d(w1), out, M, mode=ops.ROWS_CONV2D,
             geom=dict(Ho=hh, Wo=ww, Hs=hh, Ws=ww), bias=b3, rowbias=emb, rb_div=hh * ww, rb_mod=n)()
    ref = F.conv2d(xr, w1.to(H).float(), b3, padding=1) + emb.float()[:, :, None, None]
    close(out.view(n, hh, ww, co).permute(0, 3, 1, 2), ref, name="conv concat + emb")


@pytest.mark.parametrize("T", [16, 4])
def test_gemm_temporal_conv(T):
    b, c, co, hw = 2, 64, 64, 24
    x = rnd(b, c, T, hw, 1)
    w = rnd(co, c, 3, 1, 1, scale=(3 * c) ** -0.5)
    bias = rnd(co, scale=0.1)
    xh = x.permute(0, 2, 3, 4, 1).reshape(b * T * hw, c).contiguous().to(H)     # rows (b, t, s)
    M = b * T * hw
    out = torch.zeros(M, co, dtype=H, device=DEV)
    ops.Gemm(ops.temporal_taps(xh), pack.pack_conv3d_t(w), out, M, mode=ops.ROWS_TEMPORAL,
             geom=dict(Ho=hw, Wo=1, T=T), bias=bias)()
    xr = xh.view(b, T, hw, 1, c).permute(0, 4, 1, 2, 3).float()
    ref = F.conv3d(xr, w.to(H).float(), bias, padding=(1, 0, 0))
    close(out.view(b, T, hw, 1, co).permute(0, 4, 1, 2, 3), ref, name="temporal conv")


# ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,C", [(100, 320), (37, 1280), (64, 64), (20, 640), (9, 2560)])
def test_layernorm(M, C):
    x = (rnd(M, C) * 2 + 0.5).to(H)
    gamma, beta = 1 + 0.1 * rnd(C, seed=4), 0.1 * rnd(C, seed=5)
    y = torch.zeros(M, C, dtype=H, device=DEV)
    ops.layernorm(x, gamma, beta, y, M)
    close(y, F.layer_norm(x.float(), (C,), gamma, beta, 1e-5), name="layernorm")
    add = rnd(4, C, seed=8).to(H)
    ops.layernorm(x, gamma, beta, y, M, addvec=add, add_div=3, add_mod=4)
    idx = (torch.arange(M, device=DEV) // 3) % 4
    close(y, F.layer_norm(x.float() + add.float()[idx], (C,), gamma, beta, 1e-5), name="layernorm+add")


# ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_img,L,heads", [(3, 64, 2), (2, 100, 1), (2, 256, 5), (1, 1024, 2), (2, 4, 1), (1, 4096, 1)])
def test_attention_d64(n_img, L, heads):
    C = heads * 64
    qkv = rnd(n_img * L, 3 * C).to(H)
    out = torch.zeros(n_img * L, C, dtype=H, device=DEV)
    ops.attention_d64(qkv, n_img, L, heads, out)
    q, k, v = (t.view(n_img, L, heads, 64).transpose(1, 2).float() for t in qkv.view(n_img * L, 3, C).unbind(1))
    ref = torch.softmax(q @ k.transpose(-1, -2) * 0.125, -1) @ v
    close(out.view(n_img, L, heads, 64).transpose(1, 2), ref, atol=2e-3, name="fmha")


@pytest.mark.parametrize("B,T,S,heads", [(2, 16, 10, 5), (1, 4, 7, 1), (2, 16, 256, 1), (2, 3, 5, 2)])
def test_temporal_attention(B, T, S, heads):
    C = heads * 64
    qkv = rnd(B * T * S, 3 * C).to(H)
    out = torch.zeros(B * T * S, C, dtype=H, device=DEV)
    ops.temporal_attention_d64(qkv, B, T, S, heads, out)
    # rows (b, t, s) -> (b, s, h, t, d)
    q, k, v = (t.view(B, T, S, heads, 64).permute(0, 2, 3, 1, 4).float() for t in qkv.view(-1, 3, C).unbind(1))
    ref = torch.softmax(q @ k.transpose(-1, -2) * 0.125, -1) @ v
    close(out.view(B, T, S, heads, 64).permute(0, 2, 3, 1, 4), ref, atol=2e-3, name="temporal attn")


def test_softmax_rows_and_transpose():
    rows, L = 70, 1024
    s = rnd(rows, L, scale=3).to(H)
    ref = torch.softmax(s.float() * 0.2, -1)
    ops.softmax_rows(s, rows, L, 0.2)
    close(s, ref, atol=1e-5, name="softmax")
    x = rnd(100, 200).to(H)
    big = torch.zeros(100, 256, dtype=H, device=DEV)
    big[:, 32:232] = x
    out = torch.zeros(200, 100, dtype=H, device=DEV)
    ops.transpose(big[:, 32:], 100, 200, 256, out)
    assert torch.equal(out, x.t())


# ------------------------------------------------------------------------------------------------------
def test_timestep_embedding():
    t = torch.tensor([0.0, 1.6377701, -1.553652, 3.0, 15.0], device=DEV)
    out = torch.zeros(5, 320, dtype=H, device=DEV)
    ops.timestep_embedding(t, 320, out)
    half = 160
    freqs = torch.exp(-math.log(10000) * torch.arange(half, dtype=torch.float32, device=DEV) / half)
    args = t[:, None] * freqs[None]
    close(out, torch.cat([torch.cos(args), torch.sin(args)], -1), atol=1e-3, name="temb")


@pytest.mark.parametrize("cc_dtype", [torch.float32, torch.float16])
def test_sampler_pre_post(cc_dtype):
    Fn, Cx, Cc, Hh, Ww, T = 8, 4, 13, 6, 5, 4
    x = rnd(Fn, Cx, Hh, Ww) * 50
    sigma = torch.full((Fn,), 37.5, device=DEV)
    cc = (rnd(Fn, Cc, Hh, Ww, seed=2) * 0.2).to(cc_dtype)
    pre = torch.zeros(2 * Fn, Hh, Ww, 64, dtype=H, device=DEV)
    ops.sampler_pre(x, sigma, None, cc, pre)
    c_in = 1.0 / math.sqrt(37.5 ** 2 + 1)
    ref = torch.zeros(2 * Fn, 64, Hh, Ww, device=DEV)
    ref[:Fn, :Cx] = x * c_in
    ref[Fn:, :Cx] = x * c_in
    ref[Fn:, Cx:Cx + Cc] = cc.float()
    close(pre.permute(0, 3, 1, 2), ref, atol=1e-3, name="sampler_pre")
    # post
    net = rnd(2 * Fn, Hh, Ww, 8, seed=4).to(H)
    scale = torch.linspace(1.0, 2.5, T, device=DEV)
    sn = torch.full((Fn,), 20.0, device=DEV)
    x_out, den = torch.zeros_like(x), torch.zeros_like(x)
    ops.sampler_post(net, x, sigma, sn, scale, x_out, den)
    nn_ = net.float().permute(0, 3, 1, 2)[:, :Cx]
    c_skip, c_out = 1 / (37.5 ** 2 + 1), -37.5 / math.sqrt(37.5 ** 2 + 1)
    du, dc = nn_[:Fn] * c_out + x * c_skip, nn_[Fn:] * c_out + x * c_skip
    d_ref = du + scale.repeat(Fn // T).view(-1, 1, 1, 1) * (dc - du)
    torch.testing.assert_close(den, d_ref, rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(x_out, x + (x - d_ref) / 37.5 * (20.0 - 37.5), rtol=1e-5, atol=1e-4)


def test_layout_and_gaussian():
    x = rnd(3, 5, 9, 7)
    out = torch.zeros(3, 9, 7, 64, dtype=H, device=DEV)
    ops.nchw_to_nhwc(x, out, 2.0)
    ref = torch.zeros(3, 64, 9, 7, device=DEV)
    ref[:, :5] = x * 2
    close(out.permute(0, 3, 1, 2), ref, atol=1e-3, name="nchw->nhwc")
    back = torch.zeros(3, 5, 9, 7, device=DEV)
    ops.nhwc_to_nchw(out, back, 0.5)
    close(back, x, atol=1e-3, name="nhwc->nchw")
    backh = torch.zeros(3, 5, 9, 7, device=DEV, dtype=H)
    ops.nhwc_to_nchw(out, backh, 0.5)
    close(backh, x, atol=1e-3, name="nhwc->nchw fp16")
    mom = rnd(2, 6, 6, 8, seed=3).to(H)
    noise = rnd(2, 4, 6, 6, seed=4)
    o = torch.zeros(2, 4, 6, 6, device=DEV)
    ops.gaussian_sample(mom, noise, o, 0.18215)
    m = mom.float().permute(0, 3, 1, 2)
    ref = (m[:, :4] + torch.exp(0.5 * m[:, 4:].clamp(-30, 20)) * noise) * 0.18215
    torch.testing.assert_close(o, ref, rtol=1e-4, atol=1e-5)
    ops.gaussian_sample(mom, None, o, 1.0)
    torch.testing.assert_close(o, m[:, :4].contiguous(), rtol=0, atol=0)
    lat, init, z = rnd(100), rnd(100, seed=1), rnd(100, seed=2)
    ref = lat * 0.75 + (init * 3.0 + z) * 0.25
    ops.renoise_blend(lat, init, z, 0.25, 3.0)
    torch.testing.assert_close(lat, ref, rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_pack_weight_native_matches_pack_py(dtype):
    """hi3d_pack_weight / hi3d_pack_bias (C ABI) against the torch packing the plan uses (pack.py), bit for bit."""
    from hi3d_official_b200 import pack
    g = torch.Generator(device="cpu").manual_seed(5)
    w2 = torch.randn(24, 10, 3, 3, generator=g).to(DEV, dtype)
    assert torch.equal(ops.pack_weight_native(w2.contiguous(), 9, cin_pad=16, cout_pad=32), pack.pack_conv2d(w2, 16, 32))
    w3 = torch.randn(64, 64, 3, 1, 1, generator=g).to(DEV, dtype)
    assert torch.equal(ops.pack_weight_native(w3.contiguous(), 3), pack.pack_conv3d_t(w3))
    wl = torch.randn(40, 72, generator=g).to(DEV, dtype)
    assert torch.equal(ops.pack_weight_native(wl.contiguous(), 1, cout_pad=64), pack.pack_linear(wl, 64))
    wg, bg = torch.randn(128, 32, generator=g).to(DEV, dtype), torch.randn(128, generator=g).to(DEV, dtype)
    pw, pb = pack.pack_geglu(wg, bg)
    assert torch.equal(ops.pack_weight_native(wg.contiguous(), 1, geglu=True), pw)
    assert torch.equal(ops.pack_bias_native(bg, 128, geglu=True), pb)
    b = torch.randn(24, generator=g).to(DEV, dtype)
    assert torch.equal(ops.pack_bias_native(b, 24, 32), pack.pack_bias(b, 24, 32))
    assert torch.equal(ops.pack_bias_native(None, 24, 32, device=DEV), pack.pack_bias(None, 24, 32, device=DEV))


def test_pack_geglu_padded_rows_are_zero():
    """ADVICE r01: with cout_pad / n_pad > Co the interleaved GEGLU order must zero-fill the padding rows (they used to be
    filled with copies of real value / gate rows because the interleave was applied before the range check)."""
    from hi3d_official_b200 import pack
    g = torch.Generator(device="cpu").manual_seed(6)
    wg, bg = torch.randn(128, 32, generator=g).to(DEV), torch.randn(128, generator=g).to(DEV)
    pw, pb = pack.pack_geglu(wg, bg)
    got_w = ops.pack_weight_native(wg.contiguous(), 1, cin_pad=64, cout_pad=192, geglu=True)
    got_b = ops.pack_bias_native(bg, 128, 192, geglu=True)
    assert got_w.shape == (192, 64) and got_b.shape == (192,)
    assert torch.equal(got_w[:128, :32], pw) and not bool(got_w[128:].any()) and not bool(got_w[:, 32:].any())
    assert torch.equal(got_b[:128], pb) and not bool(got_b[128:].any())


def test_fused_heun_and_dpmpp2m_match_generic_path():
    """SURVEY 8f N4: HeunEDMSampler / DPMPP2MSampler with a fusable denoiser binding (network evaluations through
    sampler_pre -> launch plan -> sampler_post, solver algebra through hi3d_sampler_lincomb4) against the same samplers driven
    by the reference-style closure (generic path: OpenAIWrapper / Denoiser / guider in tensor expressions)."""
    from hi3d_official_b200 import configs, sampling, spec
    T, h = 4, 16
    model = configs.build_engine(1, device=DEV, unet_overrides=dict(model_channels=64), vae_overrides=dict(ch=64),
                                 num_steps=3, num_frames=T)
    spec.synth_fill_(model, seed=1, fast=False)
    g = torch.Generator().manual_seed(0)
    x = torch.randn(T, 4, h, h, generator=g).to(DEV)
    c = dict(crossattn=torch.randn(1, 1, 1024, generator=g).to(DEV), vector=torch.randn(1, 768, generator=g).to(DEV),
             concat=(torch.randn(T, 4, h, h, generator=g) * 0.18).to(DEV))
    uc = dict(crossattn=torch.zeros_like(c["crossattn"]), vector=c["vector"], concat=torch.zeros_like(c["concat"]))
    kw = dict(num_steps=3, device=DEV,
              discretization_config={"target": "sgm.modules.diffusionmodules.discretizer.EDMDiscretization", "params": {"sigma_max": 700.0}},
              guider_config={"target": "sgm.modules.diffusionmodules.guiders.LinearPredictionGuider",
                             "params": {"num_frames": T, "max_scale": 2.5, "min_scale": 1.0}})
    fused = model.bind_denoiser(image_only_indicator=None, num_video_frames=T)

    def closure(inp, sig, cc):
        return model.denoiser(model.model, inp, sig, cc, image_only_indicator=None, num_video_frames=T)
    for cls in (sampling.HeunEDMSampler, sampling.DPMPP2MSampler):
        smp = cls(**kw)
        n0 = N_launches()
        a = smp(fused, x.clone(), cond=c, uc=uc)
        used = N_launches() - n0
        b = cls(**kw)(closure, x.clone(), cond=c, uc=uc)
        err = float((a - b).abs().max())
        print(f"[{cls.__name__}] fused vs generic max|err| {err:.3e} (mean|x| {float(b.abs().mean()):.3e}); {used} hi3d launches")
        assert torch.isfinite(a).all() and err < 3e-2 * max(1.0, float(b.abs().max()))
        assert smp._fused, "the fused state was never built"


def N_launches():
    from hi3d_official_b200 import _native
    return _native.launch_count()


@pytest.mark.parametrize("n_img,L,qscale", [(2, 256, 1.0), (1, 4096, 1.0), (1, 16384, 1.0), (2, 1024, 4.0), (1, 512, 0.2)])
def test_attention_d512_flash(n_img, L, qscale):
    """hi3d_attention_d512_tc5 (VAE AttnBlock core, model.py:180-201): one head of dimension 512, fp32 scores inside the
    kernel, no L x L buffer -- against fp32 softmax(q k^T / sqrt(512)) v, up to L = 16384 (the 1024^2 VAE) and with logits
    large enough (|s| ~ 60) that fp16 scores would lose the parity."""
    qkv = rnd(n_img * L, 3, 512, seed=L + n_img)
    qkv[:, 0] *= qscale
    pos = torch.arange(n_img * L, device=DEV, dtype=torch.float32) % L / L
    qkv[:, 1] *= (0.5 + 1.5 * pos)[:, None]                 # keys grow along the sequence: the reference maximum moves
    qkv = qkv.reshape(n_img * L, 1536).to(H)
    out = torch.zeros(n_img * L, 512, dtype=H, device=DEV)
    ops.attention_d512(qkv, n_img, L, out)
    q, k, v = (t.reshape(n_img, L, 512).float() for t in qkv.view(n_img * L, 3, 512).unbind(1))
    ref = torch.empty(n_img, L, 512, device=DEV)
    for i in range(n_img):
        for r0 in range(0, L, 2048):
            s_ = q[i, r0:r0 + 2048] @ k[i].t() * 512 ** -0.5
            ref[i, r0:r0 + 2048] = torch.softmax(s_, -1) @ v[i]
    close(out.view(n_img, L, 512), ref, atol=2e-3, name=f"flash d512 L={L}")
