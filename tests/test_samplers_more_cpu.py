"""The ancestral, linear multistep and churned EDM samplers of hi3d_official_b200.sampling against the UNMODIFIED reference
classes (sgm/modules/diffusionmodules/sampling.py:150-302) on CPU with the analytic toy denoiser of test_samplers_cpu.py, for
every guider.  The noise is injected identically on both sides: the ancestral samplers' `noise_sampler` draws from a seeded
generator, the churned EDM samplers draw from the global generator seeded before the run.  The reference's results are
stored in tests/golden/ref_cpu_samplers.pt (tools/make_golden.py --only-cpu-samplers).  Also: the command-line sampler
choices (sampling.configure_sampler)."""
import os

import pytest
import torch

from hi3d_official_b200 import sampling as S
from test_samplers_cpu import DISC, GUIDERS, _cond, toy_denoiser

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "ref_cpu_samplers.pt")

CASES = {
    "EulerAncestralSampler": ("EulerAncestralSampler", {}),
    "EulerAncestralSampler_eta0.5": ("EulerAncestralSampler", dict(eta=0.5, s_noise=1.1)),
    "DPMPP2SAncestralSampler": ("DPMPP2SAncestralSampler", {}),
    "DPMPP2SAncestralSampler_eta0.5": ("DPMPP2SAncestralSampler", dict(eta=0.5)),
    "LinearMultistepSampler": ("LinearMultistepSampler", {}),
    "LinearMultistepSampler_order2": ("LinearMultistepSampler", dict(order=2)),
    "EulerEDMSampler_churn": ("EulerEDMSampler", dict(s_churn=2.0, s_tmin=0.05, s_tmax=50.0, s_noise=1.003)),
    "HeunEDMSampler_churn": ("HeunEDMSampler", dict(s_churn=2.0, s_noise=1.003)),
}


def sampler_kwargs(guider):
    return dict(num_steps=7, device="cpu", verbose=False, discretization_config=DISC, guider_config=GUIDERS[guider])


def run(smp):
    """One seeded run of `smp` (a reference or a hi3d sampler) on the toy problem with the noise injected."""
    g = torch.Generator().manual_seed(21)
    if hasattr(smp, "eta"):                       # the ancestral samplers draw through noise_sampler
        smp.noise_sampler = lambda x: torch.randn(x.shape, generator=g)
    c, uc = _cond()
    x0 = torch.randn(4, 4, 6, 6, generator=torch.Generator().manual_seed(9))
    torch.manual_seed(5)                          # EDMSampler draws its churn noise with torch.randn_like
    return smp(toy_denoiser, x0.clone(), cond=c, uc=uc)


@pytest.mark.parametrize("guider", list(GUIDERS))
@pytest.mark.parametrize("case", list(CASES))
def test_sampler_matches_reference(case, guider):
    name, extra = CASES[case]
    with torch.no_grad():
        b = run(getattr(S, name)(**sampler_kwargs(guider), **extra))
    a = torch.load(GOLDEN, weights_only=False)["samplers"][f"{case}/{guider}"]
    assert torch.isfinite(a).all()
    assert torch.allclose(a, b, rtol=1e-5, atol=1e-5), float((a - b).abs().max())


def test_churn_and_ancestral_noise_change_the_result():
    """The fixture is sensitive to the noise: without it (s_churn = 0, eta = 0) the results differ."""
    ref = torch.load(GOLDEN, weights_only=False)["samplers"]
    with torch.no_grad():
        b = run(S.EulerEDMSampler(**sampler_kwargs("linear")))
        e = run(S.EulerAncestralSampler(eta=0.0, **sampler_kwargs("linear")))
    assert (ref["EulerEDMSampler_churn/linear"] - b).abs().max() > 1e-2
    assert (ref["EulerAncestralSampler/linear"] - e).abs().max() > 1e-2


def test_lms_coefficients_integrate_the_lagrange_basis():
    """Gauss-Legendre weights against scipy's adaptive quadrature, as the reference integrates them, at every step."""
    from scipy import integrate
    sig = S.EDMDiscretization(sigma_max=700.0)(9).numpy()
    for i in range(len(sig) - 1):
        order = min(i + 1, 4)
        for j, c in enumerate(S.lms_coefficients(sig, i, order)):
            def basis(tau):
                p = 1.0
                for k in range(order):
                    if k != j:
                        p *= (tau - sig[i - k]) / (sig[i - j] - sig[i - k])
                return p
            want = integrate.quad(basis, sig[i], sig[i + 1], epsrel=1e-10)[0]
            assert abs(c - want) <= 1e-6 * max(1.0, abs(want)), (i, j, c, want)


def test_samplers_resolve_from_reference_target_strings():
    from hi3d_official_b200.util import instantiate_from_config
    for cls in ("EulerAncestralSampler", "DPMPP2SAncestralSampler", "LinearMultistepSampler"):
        s = instantiate_from_config({"target": f"sgm.modules.diffusionmodules.sampling.{cls}",
                                     "params": dict(num_steps=3, device="cpu", discretization_config=DISC)})
        assert type(s).__module__ == "hi3d_official_b200.sampling" and type(s).__name__ == cls


def _base():
    return S.EulerEDMSampler(num_steps=25, device="cpu", discretization_config=DISC,
                             guider_config={"target": "sgm.modules.diffusionmodules.guiders.LinearPredictionGuider",
                                            "params": {"num_frames": 16, "max_scale": 2.5, "min_scale": 1.0}})


def test_configure_sampler_defaults_keep_the_configuration():
    base = _base()
    assert S.configure_sampler(base) is base


@pytest.mark.parametrize("name", list(S.SAMPLER_CHOICES))
@pytest.mark.parametrize("guidance", S.GUIDANCE_CHOICES)
def test_configure_sampler_choices(name, guidance):
    base = _base()
    smp = S.configure_sampler(base, name, 10, guidance, None, num_frames=16)
    assert type(smp) is S.SAMPLER_CHOICES[name] and smp.num_steps == 10 and smp.discretization is base.discretization
    want = {"config": S.LinearPredictionGuider, "linear": S.LinearPredictionGuider, "vanilla": S.VanillaCFG,
            "none": S.IdentityGuider}[guidance]
    assert type(smp.guider) is want
    if guidance == "vanilla":
        assert smp.guider.scale == 2.5
    if guidance == "linear":
        assert smp.guider.max_scale == 2.5 and smp.guider.num_frames == 16


def test_configure_sampler_options():
    base = _base()
    assert S.configure_sampler(base, "heun", s_churn=0.5).s_churn == 0.5
    assert S.configure_sampler(base, "euler_ancestral", eta=0.3).eta == 0.3
    assert S.configure_sampler(base, "euler_ancestral").eta == 1.0
    assert S.configure_sampler(base, "lms").order == 4
    v = S.configure_sampler(base, guidance="vanilla", cfg_scale=4.0)
    assert type(v) is S.EulerEDMSampler and v.guider.scale == 4.0 and v.num_steps == 25
    for bad in (dict(sampler="lms", s_churn=1.0), dict(sampler="euler", eta=0.5), dict(guidance="none", cfg_scale=2.0),
                dict(cfg_scale=2.0)):
        with pytest.raises(ValueError):
            S.configure_sampler(base, **bad)
