"""Every sampler x guider of hi3d_official_b200.sampling on the fused path (graph-replayed network evaluations through
hi3d_sampler_pre / hi3d_sampler_pre_ex -> VideoUNet launch plan -> hi3d_sampler_post / hi3d_sampler_post_ancestral, solver
algebra through hi3d_sampler_lincomb4 / hi3d_sampler_lincomb) on a model_channels = 64 UNet: against the generic path (the
reference-style closure, guider and torch algebra), graph replay against eager launches bit for bit, one object against
the same object inside batches of 2 and 3 bit for bit, and the new entry points against torch formulas.

Faults this file catches, one line each:
  * the ancestral noise added where sigma_next = 0 (`noise` in sampler_post_ancestral_kernel without the sigma_next test):
    test_post_ancestral_kernel (in a sampler, sigma_up is 0 wherever sigma_next is 0, so only the kernel check sees it);
  * the LMS coefficients taken one step off (`s[i + 1 - k]` for `s[i - k]` in lms_coefficients, or the newest (x, D) pair
    paired with the second coefficient): test_fused_lms_matches_quadrature_restatement;
  * the churn noise left out of the post step's x (`xp = x` in _FusedState._launch):
    test_fused_matches_generic[EulerEDMSampler_churn-*].
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from hi3d_official_b200 import _native, ops, sampling as S  # noqa: E402

DEV = "cuda"
T, HW = 4, 16
DISC = {"target": "sgm.modules.diffusionmodules.discretizer.EDMDiscretization", "params": {"sigma_max": 700.0}}
GUIDERS = {
    "none": None,
    "vanilla": {"target": "sgm.modules.diffusionmodules.guiders.VanillaCFG", "params": {"scale": 3.0}},
    "linear": {"target": "sgm.modules.diffusionmodules.guiders.LinearPredictionGuider",
               "params": {"num_frames": T, "max_scale": 2.5, "min_scale": 1.0}},
}
SAMPLERS = {
    "EulerEDMSampler": (S.EulerEDMSampler, {}),
    "HeunEDMSampler": (S.HeunEDMSampler, {}),
    "DPMPP2MSampler": (S.DPMPP2MSampler, {}),
    "EulerEDMSampler_churn": (S.EulerEDMSampler, dict(s_churn=2.0, s_noise=1.003)),
    "HeunEDMSampler_churn": (S.HeunEDMSampler, dict(s_churn=2.0)),
    "EulerAncestralSampler": (S.EulerAncestralSampler, {}),
    "DPMPP2SAncestralSampler": (S.DPMPP2SAncestralSampler, dict(eta=0.7)),
    "LinearMultistepSampler": (S.LinearMultistepSampler, {}),
}
STEPS = 5


@pytest.fixture(scope="module")
def model():
    from hi3d_official_b200 import configs, spec
    m = configs.build_engine(1, device=DEV, unet_overrides=dict(model_channels=64), vae_overrides=dict(ch=64),
                             num_steps=3, num_frames=T)
    spec.synth_fill_(m, seed=1, fast=False)
    return m


def _inputs(B=1, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B * T, 4, HW, HW, generator=g).to(DEV)
    c = dict(crossattn=torch.randn(B, 1, 1024, generator=g).to(DEV), vector=torch.randn(B, 768, generator=g).to(DEV),
             concat=(torch.randn(B * T, 4, HW, HW, generator=g) * 0.18).to(DEV))
    uc = dict(crossattn=torch.zeros_like(c["crossattn"]), vector=c["vector"].clone(), concat=torch.zeros_like(c["concat"]))
    return x, c, uc


def _sampler(name, guider, steps=STEPS):
    cls, extra = SAMPLERS[name]
    return cls(num_steps=steps, device=DEV, discretization_config=DISC, guider_config=GUIDERS[guider], **extra)


def _seeded_noise(smp, seed=17):
    g = torch.Generator(DEV).manual_seed(seed)
    smp.noise_sampler = lambda x: torch.randn(x.shape, generator=g, device=x.device)


def _closure(model):
    def f(inp, sig, cc):
        return model.denoiser(model.model, inp, sig, cc, image_only_indicator=None, num_video_frames=T)
    return f


@pytest.mark.parametrize("guider", list(GUIDERS))
@pytest.mark.parametrize("name", list(SAMPLERS))
def test_fused_matches_generic(model, name, guider):
    x, c, uc = _inputs()
    fused = model.bind_denoiser(image_only_indicator=None, num_video_frames=T)
    smp = _sampler(name, guider)
    _seeded_noise(smp)
    a = smp(fused, x.clone(), cond=c, uc=uc)
    assert smp._fused, "the fused state was never built"
    gen = _sampler(name, guider)
    _seeded_noise(gen)
    b = gen(_closure(model), x.clone(), cond=c, uc=uc)
    err = float((a - b).abs().max())
    print(f"[{name}/{guider}] fused vs generic max|err| {err:.3e} (max|x| {float(b.abs().max()):.3e})")
    assert torch.isfinite(a).all() and err < 3e-2 * max(1.0, float(b.abs().max()))


@pytest.mark.parametrize("name", ["HeunEDMSampler", "DPMPP2MSampler", "EulerEDMSampler_churn", "HeunEDMSampler_churn",
                                  "EulerAncestralSampler", "DPMPP2SAncestralSampler", "LinearMultistepSampler"])
def test_graph_replay_equals_eager(model, name, monkeypatch):
    x, c, uc = _inputs(seed=1)
    fused = model.bind_denoiser(image_only_indicator=None, num_video_frames=T)
    out = {}
    for mode in ("1", "0"):
        monkeypatch.setenv("HI3D_CUDA_GRAPH", mode)
        smp = _sampler(name, "linear")
        _seeded_noise(smp)
        n0 = _native.launch_count()
        out[mode] = smp(fused, x.clone(), cond=c, uc=uc)
        st = next(iter(smp._fused.values()))
        assert st.use_graph == (mode == "1") and bool(st._graphs) == (mode == "1")
        print(f"[{name}] graphs={mode}: {_native.launch_count() - n0} hi3d launches")
    assert torch.equal(out["1"], out["0"])


@pytest.mark.parametrize("name,guider", [("EulerAncestralSampler", "linear"), ("DPMPP2SAncestralSampler", "vanilla"),
                                         ("EulerEDMSampler_churn", "none"), ("LinearMultistepSampler", "linear")])
def test_object_alone_equals_object_in_batch(model, name, guider):
    """Object i draws its noise from its own generator: alone and inside batches of 2 and 3 it gets the same bits."""
    x, c, uc = _inputs(B=3, seed=2)
    fused = model.bind_denoiser(image_only_indicator=None, num_video_frames=T)
    seeds = [101, 202, 303]

    def run(objs):
        sl = lambda v, per_frame: torch.cat([v[o * T:(o + 1) * T] if per_frame else v[o:o + 1] for o in objs])  # noqa: E731
        cb = {k: sl(v, k == "concat").contiguous() for k, v in c.items()}
        ucb = {k: sl(v, k == "concat").contiguous() for k, v in uc.items()}
        smp = _sampler(name, guider)
        smp.noise_generators = [torch.Generator(DEV).manual_seed(seeds[o]) for o in objs]
        return smp(fused, sl(x, True).contiguous(), cond=cb, uc=ucb)
    batch3, batch2 = run([0, 1, 2]), run([2, 0])
    for o in range(3):
        alone = run([o])
        assert torch.equal(alone, batch3[o * T:(o + 1) * T]), o
    assert torch.equal(batch2[:T], batch3[2 * T:]) and torch.equal(batch2[T:], batch3[:T])


def test_identity_guider_plan_has_F_rows(model):
    x, c, uc = _inputs()
    fused = model.bind_denoiser(image_only_indicator=None, num_video_frames=T)
    for guider, rows in (("none", T), ("vanilla", 2 * T), ("linear", 2 * T)):
        smp = _sampler("EulerEDMSampler", guider)
        st = smp._fused_state(fused, x, c, uc, refresh=True)
        assert st is not None and st.plan.N == rows and st.guided == (guider != "none")


def test_fused_lms_matches_quadrature_restatement(model):
    """The fused LMS against a restatement written here: slopes d = (x - D)/sigma on the generic path, weights from scipy's
    adaptive quadrature of the Lagrange basis (as the reference integrates them)."""
    from scipy import integrate
    x, c, uc = _inputs(seed=3)
    fused = model.bind_denoiser(image_only_indicator=None, num_video_frames=T)
    steps = 7
    smp = _sampler("LinearMultistepSampler", "linear", steps)
    a = smp(fused, x.clone(), cond=c, uc=uc)
    gen = _sampler("LinearMultistepSampler", "linear", steps)
    sig = gen.discretization(steps, device="cpu").double().numpy()
    xr = x.clone() * math.sqrt(1.0 + sig[0] ** 2)
    ds = []
    for i in range(len(sig) - 1):
        s = torch.full((T,), float(sig[i]), device=DEV)
        den = gen.denoise(xr, _closure(model), s, c, uc)
        ds = (ds + [(xr - den) / float(sig[i])])[-4:]
        order = len(ds)
        for j, d in enumerate(reversed(ds)):
            def basis(tau, j=j):
                p = 1.0
                for k in range(order):
                    if k != j:
                        p *= (tau - sig[i - k]) / (sig[i - j] - sig[i - k])
                return p
            xr = xr + integrate.quad(basis, sig[i], sig[i + 1], epsrel=1e-10)[0] * d
    err = float((a - xr).abs().max())
    print(f"fused LMS vs quadrature restatement max|err| {err:.3e}")
    assert err < 3e-2 * max(1.0, float(xr.abs().max()))


# ---- the new entry points against torch formulas ---------------------------------------------------------------------------
def _rnd(*shape, seed):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)).to(DEV)


@pytest.mark.parametrize("guided", [True, False])
def test_pre_ex_kernel(guided):
    Fn, Cx, Cc, Hh, Ww = 8, 4, 13, 6, 5
    x, eps = _rnd(Fn, Cx, Hh, Ww, seed=1) * 30, _rnd(Fn, Cx, Hh, Ww, seed=2)
    sigma = torch.linspace(5.0, 40.0, Fn, device=DEV)
    sigma_hat = sigma * 1.3
    cc, cuc = _rnd(Fn, Cc, Hh, Ww, seed=3).half(), _rnd(Fn, Cc, Hh, Ww, seed=4).half()
    rows = 2 * Fn if guided else Fn
    out = torch.zeros(rows, Hh, Ww, 64, dtype=torch.float16, device=DEV)
    cn = torch.zeros(rows, device=DEV)
    x_hat = torch.zeros_like(x)
    ops.sampler_pre_ex(x, sigma_hat, cuc, cc, out, guided, c_noise_out=cn, churn=(sigma, eps, 1.1, x_hat))
    want_hat = x + (eps * 1.1) * (sigma_hat ** 2 - sigma ** 2).sqrt().view(-1, 1, 1, 1)
    torch.testing.assert_close(x_hat, want_hat, rtol=1e-6, atol=1e-4)
    c_in = (1.0 / (sigma_hat ** 2 + 1).sqrt()).view(-1, 1, 1, 1)
    ref = torch.zeros(rows, 64, Hh, Ww, device=DEV)
    ref[:, :Cx] = (want_hat * c_in).repeat(rows // Fn, 1, 1, 1)
    ref[rows - Fn:, Cx:Cx + Cc] = cc.float()
    if guided:
        ref[:Fn, Cx:Cx + Cc] = cuc.float()
    torch.testing.assert_close(out.permute(0, 3, 1, 2).float(), ref, rtol=2e-3, atol=2e-3)
    torch.testing.assert_close(cn, (0.25 * sigma_hat.log()).repeat(rows // Fn))
    # without churn the unguided pre step packs x itself
    ops.sampler_pre_ex(x, sigma, cuc, cc, out, guided)
    ref[:, :Cx] = (x / (sigma ** 2 + 1).sqrt().view(-1, 1, 1, 1)).repeat(rows // Fn, 1, 1, 1)
    torch.testing.assert_close(out.permute(0, 3, 1, 2).float(), ref, rtol=2e-3, atol=2e-3)


@pytest.mark.parametrize("guided", [True, False])
def test_post_ancestral_kernel(guided):
    Fn, Cx, Hh, Ww, Tn = 8, 4, 6, 5, 4
    rows = 2 * Fn if guided else Fn
    net = _rnd(rows, Hh, Ww, 8, seed=5).half()
    x, eps = _rnd(Fn, Cx, Hh, Ww, seed=6) * 20, _rnd(Fn, Cx, Hh, Ww, seed=7)
    sigma = torch.linspace(3.0, 30.0, Fn, device=DEV)
    sigma_next = sigma * 0.6
    sigma_next[::3] = 0.0                                  # noise must not be added there even though sigma_up != 0
    sigma_down, sigma_up = sigma * 0.5, sigma * 0.2
    scale = torch.linspace(1.0, 2.5, Tn, device=DEV) if guided else None
    x_out, den = torch.zeros_like(x), torch.zeros_like(x)
    ops.sampler_post_ancestral(net, x, sigma, sigma_down, scale, x_out, den, noise=(eps, 1.05, sigma_up, sigma_next))
    v = lambda t: t.view(-1, 1, 1, 1)                                                            # noqa: E731
    c_skip, c_out = v(1 / (sigma ** 2 + 1)), v(-sigma / (sigma ** 2 + 1).sqrt())
    nn_ = net.float().permute(0, 3, 1, 2)[:, :Cx]
    dc = nn_[rows - Fn:] * c_out + x * c_skip
    if guided:
        du = nn_[:Fn] * c_out + x * c_skip
        dc = du + v(scale.repeat(Fn // Tn)) * (dc - du)
    torch.testing.assert_close(den, dc, rtol=1e-5, atol=1e-5)
    euler = x + (x - dc) / v(sigma) * v(sigma_down - sigma)
    want = torch.where(v(sigma_next) > 0, euler + eps * 1.05 * v(sigma_up), euler)
    torch.testing.assert_close(x_out, want, rtol=1e-5, atol=1e-4)
    ops.sampler_post_ancestral(net, x, sigma, sigma_down, scale, x_out)
    torch.testing.assert_close(x_out, euler, rtol=1e-5, atol=1e-4)


@pytest.mark.parametrize("n", [1, 5, 8, 11])
def test_lincomb_kernel(n):
    Fn = 6
    xs = [_rnd(Fn, 4, 7, 3, seed=10 + k) for k in range(n)]
    cs = [_rnd(Fn, seed=40 + k) for k in range(n)]
    want = sum(c.view(-1, 1, 1, 1) * x for x, c in zip(xs, cs))
    got = S._lincomb(list(zip(xs, cs))) if n > 8 else ops.sampler_lincomb8(torch.empty_like(xs[0]), list(zip(xs, cs)))
    torch.testing.assert_close(got, want, rtol=1e-5, atol=1e-5)


def test_new_entry_points_reject_bad_geometry():
    lib = _native.load()
    x = torch.zeros(4, 4, 6, 6, device=DEV)
    s = torch.ones(4, device=DEV)
    out = torch.zeros(8, 6, 6, 16, dtype=torch.float16, device=DEV)
    p = lambda t: t.data_ptr()                                                                    # noqa: E731
    ok = dict(guided=1, F=4, Cx=4, Cc=0, H=6, W=6, Cpad=16)

    def pre(**kw):
        a = dict(ok, **kw)
        return lib.hi3d_sampler_pre_ex(p(x), p(s), kw.get("sigma_from"), kw.get("eps"), 1.0, None, None, 0, a["guided"],
                                       a["F"], a["Cx"], a["Cc"], a["H"], a["W"], a["Cpad"], p(out), None,
                                       kw.get("x_hat"), None)
    assert pre() == 0
    torch.cuda.synchronize()
    for bad in (dict(F=0), dict(Cx=0), dict(Cpad=12), dict(Cpad=8, Cx=4, Cc=8), dict(guided=2), dict(H=0),
                dict(Cc=4),                                   # concat channels without a concat tensor
                dict(eps=p(x)),                               # churn without sigma_from / x_hat_out
                dict(eps=p(x), sigma_from=p(s))):
        assert pre(**bad) == -2, bad
    assert b"hi3d_sampler_pre_ex" in lib.hi3d_last_error()

    def post(net_ld=8, F=4, Cx=4, H=6, W=6, scale=None, T=4, eps=None, su=None, sn=None):
        return lib.hi3d_sampler_post_ancestral(p(out), net_ld, p(x), p(s), p(s), scale, T, eps, 1.0, su, sn, F, Cx, H, W,
                                               p(x), None, None)
    for bad in (dict(net_ld=2), dict(F=0), dict(Cx=0), dict(H=0), dict(scale=p(s), T=0), dict(eps=p(x)),
                dict(eps=p(x), su=p(s))):
        assert post(**bad) == -2, bad
    import ctypes as C
    arr = (C.c_void_p * 9)(*([p(x)] * 9))
    carr = (C.c_void_p * 9)(*([p(s)] * 9))
    for nterms, F in ((0, 4), (9, 4), (2, 0)):
        assert lib.hi3d_sampler_lincomb(p(x), arr, carr, nterms, F, 144, None) == -2
    carr[1] = None
    assert lib.hi3d_sampler_lincomb(p(x), arr, carr, 2, 4, 144, None) == -2
    with pytest.raises(ValueError):
        ops.sampler_lincomb8(x, [(x, s)] * 9)
    with pytest.raises(_native.Hi3dError):
        ops.sampler_pre_ex(x, s, None, None, out[:, :, :, :0].contiguous(), True)


def test_frame_sharded_plans_refuse_the_new_samplers(model):
    x, c, uc = _inputs()
    den = model.bind_denoiser(shard=(0, 2), image_only_indicator=None, num_video_frames=T)
    for name, guider in (("EulerAncestralSampler", "linear"), ("EulerEDMSampler", "vanilla"), ("EulerEDMSampler", "none")):
        with pytest.raises(NotImplementedError, match="frame-sharded"):
            _sampler(name, guider)(den, x[:T // 2].clone(), cond=c, uc=uc)
