"""Several objects in one batch: every kernel that sees B clips per CFG half gives each clip what a call over that clip alone
gives, and the stage-1 sampler step, the conditioner's towers, U^2-Net and the two entry points over B objects reproduce B
single-object runs.  Clips sit object-major inside each half: uncond clips 0..B-1, then cond clips 0..B-1."""
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from hi3d_official_b200 import ops, pack  # noqa: E402
from test_kernels_gpu import DEV, H, close, rnd  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
B, T = 3, 16


def clip_rows(x, b, rows, halves=1):
    """Rows of clip b (rows per clip) in each half of a [halves * B * rows, ...] tensor, halves stacked."""
    per = x.shape[0] // halves
    return torch.cat([x[k * per + b * rows:k * per + (b + 1) * rows] for k in range(halves)], 0)


# ---- sampler kernels -----------------------------------------------------------------------------------------------------
def test_sampler_pre_post_per_object():
    hw, Cx, Cc, Cpad, ld = 8, 4, 4, 64, 8
    F_ = B * T
    x = rnd(F_, Cx, hw, hw, seed=1)
    sigma = (torch.rand(F_, generator=torch.Generator().manual_seed(2)) * 10 + 0.1).to(DEV)
    cc, cuc = rnd(F_, Cc, hw, hw, seed=3).to(H), rnd(F_, Cc, hw, hw, seed=4).to(H)
    scale = torch.linspace(1.0, 2.5, T, device=DEV)
    out = torch.zeros(2 * F_, hw, hw, Cpad, dtype=H, device=DEV)
    cn = torch.zeros(2 * F_, device=DEV)
    ops.sampler_pre(x, sigma, cuc, cc, out, c_noise_out=cn)
    net = rnd(2 * F_ * hw * hw, ld, seed=5).to(H)
    xo, den = torch.empty_like(x), torch.empty_like(x)
    ops.sampler_post(net, x, sigma, sigma * 0.8, scale, xo, den)
    for b in range(B):
        s = slice(b * T, (b + 1) * T)
        o1, c1 = torch.zeros(2 * T, hw, hw, Cpad, dtype=H, device=DEV), torch.zeros(2 * T, device=DEV)
        ops.sampler_pre(x[s].contiguous(), sigma[s].contiguous(), cuc[s].contiguous(), cc[s].contiguous(), o1, c_noise_out=c1)
        assert torch.equal(clip_rows(out, b, T, 2), o1) and torch.equal(clip_rows(cn, b, T, 2), c1)
        xo1, den1 = torch.empty_like(x[s]), torch.empty_like(x[s])
        ops.sampler_post(clip_rows(net, b, T * hw * hw, 2).contiguous(), x[s].contiguous(), sigma[s].contiguous(),
                         (sigma[s] * 0.8).contiguous(), scale, xo1, den1)
        assert torch.equal(xo[s], xo1) and torch.equal(den[s], den1)


def test_renoise_blend_per_object():
    lat, init, z = rnd(B * T, 4, 16, 16, seed=6), rnd(B * T, 4, 16, 16, seed=7), rnd(B * T, 4, 16, 16, seed=8)
    one = [lat[b * T:(b + 1) * T].clone() for b in range(B)]
    ops.renoise_blend(lat, init, z, 0.3, 7.5)
    for b in range(B):
        s = slice(b * T, (b + 1) * T)
        ops.renoise_blend(one[b], init[s].contiguous(), z[s].contiguous(), 0.3, 7.5)
        assert torch.equal(lat[s], one[b])


# ---- temporal kernels of the UNet at 2 * B clips ---------------------------------------------------------------------------
def test_temporal_attention_per_clip():
    S, heads, C = 64, 5, 320
    nclip = 2 * B
    qkv = rnd(nclip * T * S, 3 * C, seed=9).to(H)
    out = torch.zeros(nclip * T * S, C, dtype=H, device=DEV)
    ops.temporal_attention_d64(qkv, nclip, T, S, heads, out)
    for b in range(nclip):
        r = slice(b * T * S, (b + 1) * T * S)
        o1 = torch.zeros(T * S, C, dtype=H, device=DEV)
        ops.temporal_attention_d64(qkv[r].contiguous(), 1, T, S, heads, o1)
        close(out[r], o1, rtol=1e-3, atol=1e-3, name=f"clip {b}")


@pytest.mark.parametrize("engine", ["mma", "tc5"])
def test_temporal_conv_clip_boundaries_zero_filled(engine):
    """(3,1,1) conv over 2B clips: frame 0 and frame T-1 of every clip see zeros, never the neighbouring clip."""
    hw, C, Co = 64, 320, 320
    nclip = 2 * B
    M = nclip * T * hw
    x = rnd(M, C, seed=10).to(H)
    w, bias = rnd(Co, C, 3, 1, 1, scale=1 / 30, seed=11), rnd(Co, scale=0.1, seed=12)
    emb = rnd(nclip * T, Co, scale=0.5, seed=13).to(H)
    out = torch.zeros(M, Co, dtype=H, device=DEV)
    wp = pack.pack_conv3d_t(w)
    ops.Gemm(ops.temporal_taps(x), wp, out, M, mode=ops.ROWS_TEMPORAL, geom=dict(Ho=hw, Wo=1, T=T), bias=bias, rowbias=emb,
             rb_div=hw, rb_mod=nclip * T, engine=engine)()
    xr = x.view(nclip, T, hw, 1, C).permute(0, 4, 1, 2, 3).float()
    ref = F.conv3d(xr, w.to(H).float(), bias, padding=(1, 0, 0)).permute(0, 2, 3, 4, 1).reshape(M, Co)
    ref = ref + emb.float().repeat_interleave(hw, 0)
    close(out, ref, name=f"temporal conv {nclip} clips")
    for b in range(nclip):
        r = slice(b * T * hw, (b + 1) * T * hw)
        o1 = torch.zeros(T * hw, Co, dtype=H, device=DEV)
        ops.Gemm(ops.temporal_taps(x[r].contiguous()), wp, o1, T * hw, mode=ops.ROWS_TEMPORAL, geom=dict(Ho=hw, Wo=1, T=T),
                 bias=bias, rowbias=emb[b * T:(b + 1) * T].contiguous(), rb_div=hw, rb_mod=T, engine=engine)()
        close(out[r], o1, rtol=1e-3, atol=1e-3, name=f"clip {b}")


@pytest.mark.parametrize("rb_div,rb_mod", [(64, T), (T * 64, 2 * B)])
def test_row_bias_per_clip(rb_div, rb_mod):
    """The time_pos_embed rows (frame of the clip: div HW, mod T) and the temporal cross-attention rows (clip: div T*HW,
    mod 2B) land on the rows of their own clip."""
    hw, C = 64, 320
    M = 2 * B * T * hw
    a, w, bias = rnd(M, C, seed=14).to(H), rnd(C, C, scale=1 / 18, seed=15).to(H), rnd(C, scale=0.1, seed=16)
    rb = rnd(rb_mod, C, scale=0.5, seed=17).to(H)
    out = torch.zeros(M, C, dtype=H, device=DEV)
    ops.Gemm([ops.SegSpec(a)], w, out, M, bias=bias, rowbias=rb, rb_div=rb_div, rb_mod=rb_mod, engine="tc5")()
    idx = (torch.arange(M, device=DEV) // rb_div) % rb_mod
    close(out, a.float() @ w.float().t() + bias + rb.float()[idx], name="rowbias")
    for b in range(2 * B):
        r = slice(b * T * hw, (b + 1) * T * hw)
        rb1 = rb if rb_mod == T else rb[b:b + 1].contiguous()
        o1 = torch.zeros(T * hw, C, dtype=H, device=DEV)
        ops.Gemm([ops.SegSpec(a[r].contiguous())], w, o1, T * hw, bias=bias, rowbias=rb1, rb_div=rb_div,
                 rb_mod=rb1.shape[0], engine="tc5")()
        close(out[r], o1, rtol=1e-3, atol=1e-3, name=f"clip {b}")


def test_temporal_groupnorm_sums_per_clip():
    """GroupNorm over (C/32, T, H, W): unit tables per frame, folded per clip of T frames."""
    hw, C, unit = 64, 320, 10
    nclip = 2 * B
    x = (rnd(nclip * T * hw, C, seed=18) * (1 + torch.arange(nclip * T * hw, device=DEV)[:, None] // (T * hw))).to(H)
    gam, bet = 1 + 0.1 * rnd(C, seed=19), 0.1 * rnd(C, seed=20)
    st = torch.zeros(nclip * T * (C // unit) * 2, device=DEV)
    ops.groupnorm_unit_stats(x, nclip * T, hw, unit, st)
    y = torch.zeros_like(x)
    ops.groupnorm_apply_stats(x, st, None, None, unit, nclip, T * hw, T, T * hw, gam, bet, 1e-5, True, y)
    ref = F.silu(F.group_norm(x.view(nclip, T * hw, C).permute(0, 2, 1).float(), 32, gam, bet, 1e-5))
    close(y, ref.permute(0, 2, 1).reshape(-1, C), name="temporal GroupNorm")
    for b in range(nclip):
        r = slice(b * T * hw, (b + 1) * T * hw)
        st1, y1 = torch.zeros(T * (C // unit) * 2, device=DEV), torch.zeros(T * hw, C, dtype=H, device=DEV)
        ops.groupnorm_unit_stats(x[r].contiguous(), T, hw, unit, st1)
        ops.groupnorm_apply_stats(x[r].contiguous(), st1, None, None, unit, 1, T * hw, T, T * hw, gam, bet, 1e-5, True, y1)
        close(y[r], y1, rtol=1e-3, atol=2e-3, name=f"clip {b}")


def test_vae_attention_d512_per_object():
    L = 256
    qkv = rnd(B * T * L, 1536, scale=0.5, seed=21).to(H)
    out = torch.zeros(B * T * L, 512, dtype=H, device=DEV)
    ops.attention_d512(qkv, B * T, L, out)
    for b in range(B):
        r = slice(b * T * L, (b + 1) * T * L)
        o1 = torch.zeros(T * L, 512, dtype=H, device=DEV)
        ops.attention_d512(qkv[r].contiguous(), T, L, o1)
        close(out[r], o1, rtol=1e-3, atol=1e-3, name=f"object {b}")


# ---- the full-width stage-1 UNet: a fused sampler step over B objects against B single-object steps ---------------------------
def _stage1_model():
    from hi3d_official_b200 import configs, spec
    model = configs.build_engine(1, device=DEV)
    spec.synth_fill_(model, seed=0, fast=True)
    return model


def _fused_step(model, x, c, uc, sigma, sigma_next):
    den = model.bind_denoiser(image_only_indicator=None, num_video_frames=T)
    st = model.sampler._fused_state(den, x, c, uc, refresh=True)
    assert st is not None
    return st.step(x, sigma, sigma_next, want_denoised=True)


def test_full_width_stage1_step_per_object():
    torch.manual_seed(0)
    model = _stage1_model()
    h = 64
    g = torch.Generator().manual_seed(31)
    x = (torch.randn(B * T, 4, h, h, generator=g) * 8).to(DEV)
    c = dict(crossattn=torch.randn(B, 1, 1024, generator=g).to(DEV), vector=torch.randn(B, 768, generator=g).to(DEV),
             concat=(torch.randn(B * T, 4, h, h, generator=g) * 0.18).half().to(DEV))
    # `vector` differs per object, as the elevation embedding inside it does
    uc = dict(crossattn=torch.zeros_like(c["crossattn"]), vector=c["vector"].clone(), concat=torch.zeros_like(c["concat"]))
    sigma = torch.full((B * T,), 8.0, device=DEV)
    sigma_next = torch.full((B * T,), 6.5, device=DEV)
    assert model.model.diffusion_model.get_plan(2 * B * T, h, h, T).B == 2 * B
    xb, db = _fused_step(model, x, c, uc, sigma, sigma_next)
    model.sampler._fused.clear()
    worst, spread = 0.0, 0.0
    for b in range(B):
        s = slice(b * T, (b + 1) * T)
        cb = {k: (v[s] if k == "concat" else v[b:b + 1]).contiguous() for k, v in c.items()}
        ucb = {k: (v[s] if k == "concat" else v[b:b + 1]).contiguous() for k, v in uc.items()}
        x1, d1 = _fused_step(model, x[s].contiguous(), cb, ucb, sigma[s].contiguous(), sigma_next[s].contiguous())
        x2, d2 = _fused_step(model, x[s].contiguous(), cb, ucb, sigma[s].contiguous(), sigma_next[s].contiguous())
        spread = max(spread, float((d1 - d2).abs().max()), float((x1 - x2).abs().max()))
        worst = max(worst, float((db[s] - d1).abs().max()), float((xb[s] - x1).abs().max()))
        torch.testing.assert_close(db[s], d1, rtol=1e-3, atol=1e-2)
        torch.testing.assert_close(xb[s], x1, rtol=1e-3, atol=1e-2)
    print(f"stage-1 step, {B} objects vs single: max|diff| {worst:.3e}; two single runs: max|diff| {spread:.3e}")


# ---- conditioner towers and U^2-Net over a batch ------------------------------------------------------------------------------
def _tiny_model_with_towers(stage):
    import clip_oracle as CO
    import midas_oracle as MO
    import pipeline_i2v_eval_v01 as P1
    from hi3d_official_b200 import conditioner as cond
    model = P1.load_model("none.yaml", "none.pt", stage, tiny=True)
    emb = model.conditioner.embedders
    sd = {}
    for i, e in enumerate(emb):
        if isinstance(e, cond.FrozenOpenCLIPImagePredictionEmbedder):
            sd.update({f"conditioner.embedders.{i}.open_clip.model.visual.{k}": v
                       for k, v in CO.random_visual_sd(320, 2, 80, 1024, seed=41).items()})
        elif isinstance(e, cond.AesEmbedder):
            sd.update({f"conditioner.embedders.{i}.aesthetic_model.visual.{k}": v
                       for k, v in CO.random_visual_sd(128, 2, 64, 768, seed=42).items()})
            sd.update({f"conditioner.embedders.{i}.aesthetic_mlp.{k}": v for k, v in CO.random_aesthetic_mlp(seed=43).items()})
        elif isinstance(e, cond.DepthEmbedder):
            sd.update({f"conditioner.embedders.{i}.model.model.{k}": v
                       for k, v in MO.random_dpt_hybrid_sd(seed=44, **MO.SMALL).items()})
    model.conditioner.load_tower_weights(sd)
    assert model.conditioner.missing_towers() == []
    return model


@pytest.mark.parametrize("stage", [1, 2])
def test_conditioning_per_object(stage):
    """CLIP ViT-H on B condition frames, the aesthetic tower on B images (stage 1), MiDaS on B*T frames (stage 2) and the VAE
    condition encode, once over the batch, with the condition-frame noise from each object's generator.  The noise is
    bit-identical to a single run's; the VAE encoder's GroupNorm statistics accumulate with float atomics, so `concat` may
    differ from a single run by as much as two single runs differ from each other."""
    import pipeline_i2v_eval_v01 as P1
    model = _tiny_model_with_towers(stage)
    size = 128 if stage == 1 else 256
    g = torch.Generator().manual_seed(45)
    video = (torch.rand(B, 3, T, size, size, generator=g) * 2 - 1).to(DEV)
    elevs, seeds = [0, 10, 20], [5, 6, 7]
    gens = lambda: [torch.Generator(DEV).manual_seed(s) for s in seeds]     # noqa: E731
    noisy = model.add_custom_cond({"video": video}, infer=True, generators=gens())["cond_frames"]
    c, uc = P1.cond_from_towers(model, video, None, elevs, stage, generators=gens())
    for b in range(B):
        torch.manual_seed(seeds[b])                    # a single-object run: the global generator, seeded
        noisy1 = model.add_custom_cond({"video": video[b:b + 1]}, infer=True)["cond_frames"]
        n = noisy1.shape[0]
        assert torch.equal(noisy[b * n:(b + 1) * n], noisy1)
        runs = []
        for _ in range(2):
            torch.manual_seed(seeds[b])
            runs.append(P1.cond_from_towers(model, video[b], None, elevs[b], stage))
        for i, d in enumerate((c, uc)):
            for k, v in runs[0][i].items():
                rows = v.shape[0] if k != "concat" else T
                got = d[k][b * rows:(b + 1) * rows]
                assert got.shape == v.shape, k
                diff = float((got.float() - v.float()).abs().max())
                spread = float((runs[1][i][k].float() - v.float()).abs().max())
                print(f"stage {stage} object {b} {'c' if i == 0 else 'uc'}[{k}]: batched vs single {diff:.2e}, two single runs {spread:.2e}")
                torch.testing.assert_close(got.float(), v.float(), rtol=1e-3, atol=max(2e-3, 2 * spread),
                                           msg=f"{k} of object {b}: {diff:.3e} (two single runs: {spread:.3e})")


def test_u2net_batch_per_image():
    import u2net_oracle as UO
    from PIL import Image
    from hi3d_official_b200 import rembg
    from hi3d_official_b200.u2net import U2NetTower
    session = rembg.U2netSession(U2NetTower(UO.random_u2net_sd(seed=46, variant="p", calib_hw=320), device=DEV))
    rs = torch.Generator().manual_seed(47)
    imgs = [Image.fromarray((torch.rand(hh, ww, 3, generator=rs) * 255).to(torch.uint8).numpy())
            for hh, ww in ((200, 160), (90, 300), (320, 320))]
    import numpy as np
    cut = rembg.remove_batch(imgs, session)
    for img, got in zip(imgs, cut):
        ref = rembg.remove(img, session)
        assert got.size == img.size
        diff = np.abs(np.asarray(got, dtype=np.int16) - np.asarray(ref, dtype=np.int16))
        assert diff.max() <= 2, f"cut-out differs by up to {diff.max()} levels"


# ---- the entry points: two images with --batch 2 against two single-image runs -------------------------------------------------
def _run(script, *args, cwd=ROOT):
    r = subprocess.run([sys.executable, os.path.join(ROOT, script), *args], capture_output=True, text=True, timeout=900, cwd=cwd)
    assert r.returncode == 0, r.stdout[-1500:] + r.stderr[-3000:]
    return r.stdout


def _files(root):
    return sorted(os.path.relpath(os.path.join(d, f), root) for d, _, fs in os.walk(root) for f in fs)


def test_pipelines_two_images_batched_match_single_runs(tmp_path):
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
        singles = [str(tmp_path / f"single{k}" / n) for k in range(2)]      # two runs: the spread of the float atomics
        for single in singles:
            for script in ("pipeline_i2v_eval_v01.py", "pipeline_i2v_eval_v02.py"):
                so = _run(script, "--tiny", "--output_dir", single, "--image_path", imgs[i], "--seed", seeds[i], "--elevation",
                          elevs[i], "--towers", towers[i])
                assert f"(seed {seeds[i]})" in so
        mine = os.path.join(batched, n)
        assert _files(mine) == _files(singles[0])
        for f in ("first_step/first.pt", "second_step_video/second.pt"):
            a, b, b2 = (torch.load(os.path.join(d, f)).float() for d in (mine, *singles))
            assert a.shape == b.shape == ((16, 3, 128, 128) if "first" in f else (16, 3, 256, 256))
            diff, spread = float((a - b).abs().max()), float((b2 - b).abs().max())
            print(f"{n}/{f}: batched vs single max|diff| {diff:.3e}, two single runs {spread:.3e}")
            # within the north-star tolerance, or within twice what two single runs of the same seed differ by
            assert bool(((a - b).abs() <= 1e-2 + 1e-3 * b.abs()).all()) or diff <= 2 * spread, f"{n}/{f}: {diff:.3e}"
