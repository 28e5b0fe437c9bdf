"""MiDaS DPT-Hybrid depth tower on the H100: the new kernels (ReLU epilogue, stem rows, "same" max-pool, GroupNorm apply with an
addend, bilinear x2, ReLU copy) against fp32 PyTorch with NaN-filled outputs and guard regions, then the full-size tower against
the fp32 oracle of tests/midas_oracle.py, the native stage-2 conditioner, and the stage-2 script with no tower outputs given."""
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

import midas_oracle as MO  # noqa: E402
from hi3d_official_b200 import ops  # noqa: E402
from test_kernels_gpu import DEV, H, close, rnd  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAN = float("nan")


def nan16(*shape):
    return torch.full(shape, NAN, dtype=H, device=DEV)


def untouched(t):
    return bool(torch.isnan(t.float()).all())


# ---- ReLU epilogue ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("engine", ["tc5", "mma"])
@pytest.mark.parametrize("n,N,K", [(1, 256, 128), (3, 64, 192), (2, 32, 64)])
def test_gemm_relu_epilogue(engine, n, N, K):
    M = 577 * n
    a, w, b = rnd(M, K, seed=1).to(H), rnd(N, K, scale=K ** -0.5, seed=2).to(H), rnd(N, scale=0.5, seed=3)
    res = rnd(M, N, seed=4).to(H)
    out = nan16(M + 8, N + 8)                                   # guard rows below and guard columns right of the output
    ops.Gemm([ops.SegSpec(a)], w, out, M, bias=b, act=ops.ACT_RELU, engine=engine)()
    ref = F.relu(a.float() @ w.float().t() + b).half().float()
    close(out[:M, :N], ref, name=f"{engine} relu")
    assert untouched(out[M:]) and untouched(out[:, N:])
    out2 = nan16(M, N)
    ops.Gemm([ops.SegSpec(a)], w, out2, M, bias=b, act=ops.ACT_RELU, residual=res, engine=engine)()
    close(out2, ref + res.float(), name=f"{engine} relu + residual")


@pytest.mark.parametrize("engine", ["tc5", "mma"])
def test_conv_relu_epilogue(engine):
    n, h, w, ci, co = 2, 12, 16, 64, 128
    x = rnd(n, h, w, ci, seed=5).to(H)
    wt = rnd(co, ci, 3, 3, scale=(9 * ci) ** -0.5, seed=6)
    b = rnd(co, scale=0.3, seed=7)
    out = nan16(n * h * w, co)
    ops.Gemm(ops.conv_taps([x.view(-1, ci)]), wt.permute(0, 2, 3, 1).reshape(co, -1).half().contiguous(), out, n * h * w,
             mode=ops.ROWS_CONV2D, geom=dict(Ho=h, Wo=w, Hs=h, Ws=w, stride=1), bias=b, act=ops.ACT_RELU, engine=engine)()
    ref = F.relu(F.conv2d(x.float().permute(0, 3, 1, 2), wt.half().float(), b, padding=1)).permute(0, 2, 3, 1).reshape(-1, co)
    close(out, ref.half().float(), name=f"{engine} conv relu")


# ---- stem rows, max-pool ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("hw", [(64, 96), (33, 50)])
def test_dpt_stem_rows(dtype, hw):
    n, (h, w), kpad = 2, hw, 192
    img = rnd(n, 3, h, w, seed=8).to(dtype)
    ho, wo = (h + 1) // 2, (w + 1) // 2
    out = nan16(n * ho * wo + 4, kpad)
    ops.dpt_stem_rows(img, out[:n * ho * wo])
    cols = F.unfold(MO.pad_same(img.float(), 7, 2), 7, stride=2)              # (n, 147, L), K ordered (c, ky, kx)
    ref = torch.zeros(n * ho * wo, kpad, device=DEV)
    ref[:, :147] = cols.transpose(1, 2).reshape(-1, 147)
    assert torch.equal(out[:n * ho * wo].float(), ref.half().float())
    assert untouched(out[n * ho * wo:])


@pytest.mark.parametrize("hw", [(48, 40), (17, 24), (6, 7)])
def test_maxpool3x3s2_same(hw):
    n, (h, w), c = 3, hw, 64
    x = rnd(n, h, w, c, seed=9).to(H)
    ho, wo = (h + 1) // 2, (w + 1) // 2
    y = nan16(n * ho * wo + 2, c)
    ops.maxpool3x3s2_same(x.view(-1, c), n, h, w, y[:n * ho * wo])
    ref = F.max_pool2d(MO.pad_same(x.float().permute(0, 3, 1, 2), 3, 2, value=float("-inf")), 3, 2)
    assert torch.equal(y[:n * ho * wo].float(), ref.permute(0, 2, 3, 1).reshape(-1, c))
    assert untouched(y[n * ho * wo:])


# ---- GroupNorm apply with an addend ------------------------------------------------------------------------------------------------
def _gn_case(n, rows, C, seed):
    x = (rnd(n * rows, C, seed=seed) * 2 + 0.5).to(H)
    st = torch.zeros(n, C // (C // 32), 2, device=DEV)
    ops.groupnorm_unit_stats(x, n, rows, C // 32, st)
    g, b = 1 + rnd(C, scale=0.2, seed=seed + 1), rnd(C, scale=0.2, seed=seed + 2)
    ref = F.group_norm(x.float().view(n, rows, C).permute(0, 2, 1), 32, g, b, eps=1e-5).permute(0, 2, 1).reshape(n * rows, C)
    return x, st, g, b, ref


@pytest.mark.parametrize("addend", ["none", "raw", "gn"])
@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("n,rows,C", [(2, 96 * 96, 64), (3, 577, 256), (2, 144, 1024)])
def test_groupnorm_apply_add(addend, relu, n, rows, C):
    x, st, g, b, ref = _gn_case(n, rows, C, seed=10)
    kw = {}
    if addend == "raw":
        a = rnd(n * rows, C, seed=20).to(H)
        kw, ref = dict(add=a), ref + a.float()
    elif addend == "gn":
        a, sa, ga, ba, ra = _gn_case(n, rows, C, seed=30)
        kw, ref = dict(add=a, add_stats=sa, add_gamma=ga, add_beta=ba), ref + ra
    if relu:
        ref = F.relu(ref)
    y = nan16(n * rows + 8, C)
    ops.groupnorm_apply_add(x, st, g, b, C // 32, n, y[:n * rows], relu=relu, **kw)
    close(y[:n * rows], ref, atol=4e-3, name=f"gn apply {addend} relu={relu}")
    assert untouched(y[n * rows:])


def test_groupnorm_apply_add_haloed_output():
    """The trunk's last apply writes image i at rows i * (1 + P) + 1 .. : the class-token rows between stay untouched."""
    n, rows, C = 3, 36, 256
    x, st, g, b, ref = _gn_case(n, rows, C, seed=40)
    y = nan16(n * (rows + 1), C)
    ops.groupnorm_apply_add(x, st, g, b, C // 32, n, y, relu=True, y_sample_rows=rows + 1, y_row_off=1)
    yv = y.view(n, rows + 1, C)
    close(yv[:, 1:].reshape(-1, C), F.relu(ref), atol=4e-3, name="haloed gn apply")
    assert untouched(yv[:, 0])


# ---- bilinear x2, ReLU copy ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hw", [(5, 7), (12, 8), (1, 3)])
@pytest.mark.parametrize("with_add", [False, True])
def test_upsample2x_bilinear_ac(hw, with_add):
    n, (h, w), c = 2, hw, 128
    x = rnd(n, h, w, c, seed=50).to(H)
    ref = F.interpolate(x.float().permute(0, 3, 1, 2), scale_factor=2, mode="bilinear", align_corners=True)
    ref = ref.permute(0, 2, 3, 1).reshape(-1, c)
    add = None
    if with_add:
        add = rnd(n * 4 * h * w, c, seed=51).to(H)
        ref = ref + add.float()
    y = nan16(n * 4 * h * w + 3, c)
    ops.upsample2x_bilinear_ac(x.view(-1, c), n, h, w, y[:n * 4 * h * w], add=add)
    close(y[:n * 4 * h * w], ref, name="upsample2x")
    assert untouched(y[n * 4 * h * w:])


def test_relu_copy():
    x = rnd(1000, 64, seed=60).to(H)
    y = nan16(1008, 64)
    ops.relu_copy(x, y[:1000])
    assert torch.equal(y[:1000], F.relu(x)) and untouched(y[1000:])


# ---- the full-size tower against the fp32 oracle (SURVEY §8c: native error <= 2x the oracle's own error under autocast) --------
def test_tower_full_size_384():
    from hi3d_official_b200.conditioner import depth_to_concat
    from hi3d_official_b200.midas import DPTHybridTower
    sd = MO.random_dpt_hybrid_sd(seed=11, device=DEV, **MO.FULL)
    g = torch.Generator().manual_seed(12)
    x = (torch.rand(4, 3, 384, 384, generator=g) * 2 - 1).to(DEV)
    with torch.no_grad():
        ref = MO.dpt_forward(sd, x)
        with torch.autocast("cuda", dtype=torch.float16):
            amp = MO.dpt_forward(sd, x).float()
    got = DPTHybridTower(sd, device=DEV)(x)
    assert got.shape == ref.shape == (4, 384, 384) and got.dtype == torch.float32
    e, e_amp = MO.relerr(got, ref), MO.relerr(amp, ref)
    cat = lambda y: depth_to_concat(y, 1024, 1024)            # noqa: E731  (the stage-2 size: 9 x 128 x 128)
    ce, ce_amp = MO.relerr(cat(got), cat(ref)), MO.relerr(cat(amp), cat(ref))
    print(f"DPT-Hybrid 4 x 384^2: rel-L2 native {e:.3e}, autocast {e_amp:.3e} (ratio {e / e_amp:.2f}); depth_to_concat native "
          f"{ce:.3e}, autocast {ce_amp:.3e} (ratio {ce / ce_amp:.2f})")
    assert e <= 2 * e_amp, f"depth: native error {e:.3e} > 2 x autocast error {e_amp:.3e}"
    assert ce <= 2 * ce_amp, f"depth_to_concat: native error {ce:.3e} > 2 x autocast error {ce_amp:.3e}"


# ---- the stage-2 conditioner and script with native towers (reduced widths) -------------------------------------------------
def _small_clip(seed):
    import clip_oracle as CO
    return CO.random_visual_sd(320, 2, 80, 1024, seed=seed)


def test_stage2_conditioning_native_vs_oracle():
    import pipeline_i2v_eval_v01 as P1
    from hi3d_official_b200 import conditioner as cond
    model = P1.load_model("none.yaml", "none.pt", 2, tiny=True)
    emb = model.conditioner.embedders
    i_clip = next(i for i, e in enumerate(emb) if isinstance(e, cond.FrozenOpenCLIPImagePredictionEmbedder))
    i_depth = next(i for i, e in enumerate(emb) if isinstance(e, cond.DepthEmbedder))
    dsd = MO.random_dpt_hybrid_sd(seed=51, **MO.SMALL)
    sd = {f"conditioner.embedders.{i_clip}.open_clip.model.visual.{k}": v for k, v in _small_clip(52).items()}
    sd.update({f"conditioner.embedders.{i_depth}.model.model.{k}": v for k, v in dsd.items()})
    assert sorted(model.conditioner.load_tower_weights(sd)) == ["clip", "depth"]
    assert model.conditioner.missing_towers() == []
    T = model.num_samples
    g = torch.Generator().manual_seed(53)
    frames = (torch.rand(3, T, 256, 256, generator=g) * 2 - 1).to(DEV)
    torch.manual_seed(5)
    c, uc = P1.cond_from_towers(model, frames, None, 10, 2)
    # the oracle's depth maps of the very frames the depth tower saw, passed in the batch as `cond_frames:depth`
    tower, seen = emb[i_depth].model, []
    sd_dev = {k: v.to(DEV) for k, v in dsd.items()}
    tower.set_fn(lambda y: seen.append(MO.dpt_forward(sd_dev, y.float())) or seen[-1])
    torch.manual_seed(5)
    P1.cond_from_towers(model, frames, None, 10, 2)
    tower.set_fn(None)
    assert len(seen) == 2 and seen[0].shape == (T, 96, 96)
    torch.manual_seed(5)
    c_ref, uc_ref = P1.cond_from_towers(model, frames, {"depth": seen[0]}, 10, 2)
    nd = 9
    e = MO.relerr(c["concat"][:, :nd].float(), c_ref["concat"][:, :nd].float())
    print(f"stage-2 conditioning: depth channels of concat rel-L2 {e:.2e}")
    assert c["concat"].shape == c_ref["concat"].shape and c["concat"].shape[1] == 13
    assert e < 2e-2
    torch.testing.assert_close(c["concat"][:, nd:].float(), c_ref["concat"][:, nd:].float(), atol=1e-2, rtol=1e-2)
    torch.testing.assert_close(c["crossattn"], c_ref["crossattn"])
    torch.testing.assert_close(c["vector"], c_ref["vector"])


def test_stage2_script_with_native_towers(tmp_path):
    os.makedirs(tmp_path / "ckpts")
    os.makedirs(tmp_path / "out" / "first_step")
    torch.save({"visual." + k: v for k, v in _small_clip(61).items()}, tmp_path / "ckpts" / "open_clip_pytorch_model.bin")
    torch.save(MO.random_dpt_hybrid_sd(seed=62, **MO.SMALL), tmp_path / "ckpts" / "dpt_hybrid_384.pt")
    g = torch.Generator().manual_seed(63)
    torch.save(torch.rand(16, 3, 128, 128, generator=g) * 2 - 1, tmp_path / "out" / "first_step" / "first.pt")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "pipeline_i2v_eval_v02.py"), "--tiny", "--seed", "0", "--output_dir", "out"],
                       capture_output=True, text=True, timeout=900, cwd=str(tmp_path))
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    frames = torch.load(tmp_path / "out" / "second_step_video" / "second.pt")
    assert frames.shape[0] == 16 and bool(torch.isfinite(frames.float()).all())
