"""Reproducible generation: the same inputs give the same bits on every run, and an object's result does not depend on the
other objects of its batch.  The GroupNorm statistics kernels sum in a fixed order that depends only on each image's own shape,
so the fused sampler step, the VAE, the MiDaS tower and both entry points are compared with torch.equal, not a tolerance."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

from hi3d_official_b200 import ops  # noqa: E402
from test_batch_gpu import _files, _fused_step, _run, _stage1_model  # noqa: E402
from test_kernels_gpu import DEV, H  # noqa: E402

B, T = 3, 16


# ---- unit statistics: the plans' channel counts and rows per image --------------------------------------------------------
def _images(n, rows, C, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    # a per-image, per-channel offset so that the sums do not cancel to noise
    off = torch.randn(n, 1, C, generator=g, device=DEV)
    return (torch.randn(n, rows, C, generator=g, device=DEV) * 1.5 + off).to(H)


def _unit_stats(x, unit, table=None):
    n, rows, C = x.shape
    t = torch.zeros(n * (C // unit) * 2, device=DEV) if table is None else table.clone()
    ops.groupnorm_unit_stats(x.view(n * rows, C), n, rows, unit, t)
    return t


STATS_SHAPES = [  # (C, unit, rows per image, n_images): VAE at 1024^2 / 512^2 (one frame per call), UNet at 2 x 16 frames
    (128, 4, 1 << 20, 1), (256, 4, 1 << 20, 1), (256, 4, 262147, 2), (512, 4, 1 << 16, 2),
    (320, 10, 16384, 32), (640, 10, 4096, 32), (1280, 10, 1024, 32), (1280, 10, 256, 96), (2560, 10, 64, 96), (320, 10, 4096, 96),
    (1280, 10, 64, 2), (320, 10, 16383, 3), (512, 16, 2304, 32),
]


@pytest.mark.parametrize("C,unit,rows,n", STATS_SHAPES)
def test_unit_stats_repeatable_batch_invariant_and_exact(C, unit, rows, n):
    x = _images(n, rows, C, seed=C + rows + n)
    nu = C // unit
    a, b = _unit_stats(x, unit), _unit_stats(x, unit)
    assert torch.equal(a, b), "two calls on the same tensor differ"
    # an accumulated table: each entry is written once, as old + this launch's sum
    base = torch.randn(n * nu * 2, generator=torch.Generator(device=DEV).manual_seed(1), device=DEV) * 100
    acc1, acc2 = _unit_stats(x, unit, base), _unit_stats(x, unit, base)
    assert torch.equal(acc1, acc2)
    assert torch.equal(acc1, base + a)
    # each image alone gives the bits it gets inside the batch
    for i in sorted({0, n // 2, n - 1}):
        one = _unit_stats(x[i:i + 1].contiguous(), unit)
        assert torch.equal(one, a.view(n, nu * 2)[i]), f"image {i} alone differs from image {i} of a batch of {n}"
    # against fp64
    xd = x.double().view(n, rows, nu, unit)
    ref = torch.stack([xd.sum((1, 3)), (xd * xd).sum((1, 3))], -1).view(n, nu, 2)
    scale = x.double().abs().view(n, rows, nu, unit).sum((1, 3))
    got = a.double().view(n, nu, 2)
    assert float(((got[..., 0] - ref[..., 0]).abs() / scale).max()) < 5e-5
    assert float(((got[..., 1] - ref[..., 1]).abs() / ref[..., 1]).max()) < 5e-5
    # every row is counted exactly once: ones on the first, the last and scattered rows, zeros elsewhere
    idx = torch.cat([torch.tensor([0, rows - 1]), torch.randperm(rows, generator=torch.Generator().manual_seed(3))[:97]]).unique()
    y = torch.zeros(n, rows, C, dtype=H, device=DEV)
    y[:, idx.to(DEV)] = 1.0
    assert torch.equal(_unit_stats(y, unit), torch.full((n * nu * 2,), float(len(idx) * unit), device=DEV))


def test_group_sums_repeatable_and_per_clip():
    unit, C1, C2, ns, ips = 10, 640, 320, 6, 16
    g = torch.Generator(device=DEV).manual_seed(2)
    s1 = torch.rand(ns * ips * (C1 // unit) * 2, generator=g, device=DEV) * 50
    s2 = torch.rand(ns * ips * (C2 // unit) * 2, generator=g, device=DEV) * 50
    for st2, c2 in ((None, 0), (s2, C2)):
        out = [torch.empty(ns * 64, device=DEV) for _ in range(2)]
        for o in out:
            ops.groupnorm_group_sums(s1, C1, st2, c2, unit, ns, ips, o)
        assert torch.equal(out[0], out[1])
        for b in range(ns):
            one = torch.empty(64, device=DEV)
            p1 = s1.view(ns, -1)[b].contiguous()
            p2 = st2.view(ns, -1)[b].contiguous() if st2 is not None else None
            ops.groupnorm_group_sums(p1, C1, p2, c2, unit, 1, ips, one)
            assert torch.equal(one, out[0].view(ns, 64)[b]), f"clip {b}"


# ---- the full-width stage-1 fused sampler step --------------------------------------------------------------------------------
def test_full_width_stage1_step_bit_exact():
    torch.manual_seed(0)
    model = _stage1_model()
    h = 64
    g = torch.Generator().manual_seed(31)
    x = (torch.randn(B * T, 4, h, h, generator=g) * 8).to(DEV)
    c = dict(crossattn=torch.randn(B, 1, 1024, generator=g).to(DEV), vector=torch.randn(B, 768, generator=g).to(DEV),
             concat=(torch.randn(B * T, 4, h, h, generator=g) * 0.18).half().to(DEV))
    uc = dict(crossattn=torch.zeros_like(c["crossattn"]), vector=c["vector"].clone(), concat=torch.zeros_like(c["concat"]))
    sigma = torch.full((B * T,), 8.0, device=DEV)
    sigma_next = torch.full((B * T,), 6.5, device=DEV)
    xb, db = _fused_step(model, x, c, uc, sigma, sigma_next)
    xb2, db2 = _fused_step(model, x, c, uc, sigma, sigma_next)
    assert torch.equal(xb, xb2) and torch.equal(db, db2), "two runs of the same batched step differ"
    model.sampler._fused.clear()
    for b in range(B):
        s = slice(b * T, (b + 1) * T)
        cb = {k: (v[s] if k == "concat" else v[b:b + 1]).contiguous() for k, v in c.items()}
        ucb = {k: (v[s] if k == "concat" else v[b:b + 1]).contiguous() for k, v in uc.items()}
        runs = [_fused_step(model, x[s].contiguous(), cb, ucb, sigma[s].contiguous(), sigma_next[s].contiguous())
                for _ in range(2)]
        assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1]), f"object {b}: two single runs differ"
        assert torch.equal(xb[s], runs[0][0]) and torch.equal(db[s], runs[0][1]), f"object {b}: batched differs from single"


# ---- the VAE: encode, 2-D decode and the temporal VideoDecoder ----------------------------------------------------------------
def _vae(kind):
    from hi3d_official_b200 import configs, spec
    from hi3d_official_b200.vae import AutoencoderKLModeOnly, AutoencoderKLTemporal
    dd = dict(configs._VAE_DD)
    cfg = spec.VAEConfig.from_ddconfig(dd, 4)
    sd = spec.synth_state_dict(spec.vae_param_shapes(cfg), seed=3)
    if kind == "video":
        ae = AutoencoderKLTemporal(embed_dim=4, ddconfig=dd, video_kernel_size=[3, 1, 1], time_mode="conv-only")
        sd = {k: v for k, v in sd.items() if not k.startswith("decoder.")}
        sd.update(spec.synth_state_dict(spec.video_decoder_param_shapes(cfg, (3, 1, 1)), seed=4))
    else:
        ae = AutoencoderKLModeOnly(embed_dim=4, ddconfig=dd)
    ae.load_state_dict(sd, strict=True)
    return ae.cuda().half()


def test_vae_encode_decode_bit_exact_per_object():
    ae = _vae("2d")
    g = torch.Generator().manual_seed(6)
    img = (torch.rand(B, 3, 256, 256, generator=g) * 2 - 1).to(DEV).half()
    z = ae.encode(img)
    assert torch.equal(z, ae.encode(img))
    for b in range(B):
        assert torch.equal(z[b:b + 1], ae.encode(img[b:b + 1].contiguous())), f"encode: object {b}"
    zl = torch.randn(B, 4, 32, 32, generator=g).to(DEV).half()
    dec = ae.decode(zl, scale=1.0 / 0.18215)
    assert torch.equal(dec, ae.decode(zl, scale=1.0 / 0.18215))
    for b in range(B):
        assert torch.equal(dec[b:b + 1], ae.decode(zl[b:b + 1].contiguous(), scale=1.0 / 0.18215)), f"decode: object {b}"


def test_video_decoder_bit_exact_per_clip():
    ae = _vae("video")
    Tc = 4
    g = torch.Generator().manual_seed(7)
    z = torch.randn(B * Tc, 4, 16, 16, generator=g).to(DEV).half()
    dec = ae.decode(z, timesteps=Tc)
    assert torch.equal(dec, ae.decode(z, timesteps=Tc))
    for b in range(B):
        s = slice(b * Tc, (b + 1) * Tc)
        assert torch.equal(dec[s], ae.decode(z[s].contiguous(), timesteps=Tc)), f"clip {b}"


# ---- the MiDaS DPT-Hybrid tower ---------------------------------------------------------------------------------------------------
def test_midas_tower_repeatable():
    import midas_oracle as MO
    from hi3d_official_b200.midas import DPTHybridTower
    tower = DPTHybridTower(MO.random_dpt_hybrid_sd(seed=44, device=DEV, **MO.SMALL), device=DEV)
    g = torch.Generator().manual_seed(8)
    x = (torch.rand(2, 3, 384, 384, generator=g) * 2 - 1).to(DEV)
    a, b = tower(x), tower(x)
    assert torch.equal(a, b)


# ---- the entry points: the same seed twice, and two images with --batch 2 against the single runs ---------------------------------
def test_pipelines_same_seed_same_bits_and_batch_invariant(tmp_path):
    import cv2
    import numpy as np
    names, seeds, elevs = ["cat", "dog"], ["3", "4"], ["0", "20"]
    towers = []
    for i, n in enumerate(names):
        cv2.imwrite(str(tmp_path / f"{n}.png"), (np.random.RandomState(i).rand(200, 160 + 40 * i, 3) * 255).astype("uint8"))
        g = torch.Generator().manual_seed(10 + i)
        towers.append(str(tmp_path / f"{n}.pt"))
        torch.save({"clip": torch.randn(1, 1024, generator=g), "aes": torch.tensor([[4.0 + i]]),
                    "depth": torch.rand(16, 24, 24, generator=g)}, towers[-1])
    imgs = [str(tmp_path / f"{n}.png") for n in names]
    batched = str(tmp_path / "batched")
    for script in ("pipeline_i2v_eval_v01.py", "pipeline_i2v_eval_v02.py"):
        _run(script, "--tiny", "--output_dir", batched, "--image_path", *imgs, "--seed", *seeds, "--elevation", *elevs,
             "--towers", *towers, "--batch", "2")
    for i, n in enumerate(names):
        singles = [str(tmp_path / f"single{k}" / n) for k in range(2)]
        for single in singles:
            for script in ("pipeline_i2v_eval_v01.py", "pipeline_i2v_eval_v02.py"):
                _run(script, "--tiny", "--output_dir", single, "--image_path", imgs[i], "--seed", seeds[i], "--elevation",
                     elevs[i], "--towers", towers[i])
        mine = os.path.join(batched, n)
        assert _files(mine) == _files(singles[0])
        for f in ("first_step/first.pt", "second_step_video/second.pt"):
            a, b, b2 = (torch.load(os.path.join(d, f)) for d in (mine, *singles))
            assert torch.equal(b, b2), f"{n}/{f}: two runs with seed {seeds[i]} differ"
            assert torch.equal(a, b), f"{n}/{f}: --batch 2 differs from the single-image run"
