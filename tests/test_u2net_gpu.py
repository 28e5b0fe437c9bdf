"""U^2-Net background removal on the H100: dilated taps on both GEMM engines, the ceil-mode pool, the bilinear resize and the
side fusion against PyTorch with NaN-filled outputs and guard regions, the full-size tower and the `p` variant against the fp32
oracle of tests/u2net_oracle.py, and the two pipeline scripts with background removal."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

import u2net_oracle as UO  # noqa: E402
from hi3d_official_b200 import ops  # noqa: E402
from test_kernels_gpu import DEV, H, close, rnd  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAN = float("nan")


def nan16(*shape):
    return torch.full(shape, NAN, dtype=H, device=DEV)


def untouched(t):
    return bool(torch.isnan(t.float()).all())


# ---- dilated 3x3 convs, written into a channel slice ---------------------------------------------------------------------------
@pytest.mark.parametrize("engine", ["tc5", "mma"])
@pytest.mark.parametrize("n", [1, 8])
@pytest.mark.parametrize("hw", [10, 20, 40])
@pytest.mark.parametrize("d", [1, 2, 4, 8])
def test_dilated_conv(engine, n, hw, d):
    ci, co = 64, 32
    x = rnd(n, hw, hw, ci, seed=1).to(H)
    wt = rnd(co, ci, 3, 3, scale=(9 * ci) ** -0.5, seed=2)
    b = rnd(co, scale=0.3, seed=3)
    M = n * hw * hw
    out = nan16(M + 8, 64)                                        # the conv writes columns 16..47 of the first M rows only
    ops.Gemm(ops.conv_taps([x.view(-1, ci)], dilation=d), wt.permute(0, 2, 3, 1).reshape(co, -1).half().contiguous(),
             out[:M, 16:16 + co], M, mode=ops.ROWS_CONV2D, geom=dict(Ho=hw, Wo=hw, Hs=hw, Ws=hw, stride=1), bias=b,
             act=ops.ACT_RELU, engine=engine)()
    ref = F.relu(F.conv2d(x.float().permute(0, 3, 1, 2), wt.half().float(), b, padding=d, dilation=d))
    close(out[:M, 16:16 + co], ref.permute(0, 2, 3, 1).reshape(M, co).half().float(), name=f"{engine} d={d} {n}x{hw}^2")
    assert untouched(out[:, :16]) and untouched(out[:, 16 + co:]) and untouched(out[M:])


@pytest.mark.parametrize("engine", ["tc5", "mma"])
@pytest.mark.parametrize("co", [16, 32])
def test_conv_into_channel_slice_with_residual(engine, co):
    n, hw, ci, d = 2, 20, 64, 2
    x = rnd(n, hw, hw, ci, seed=4).to(H)
    wt = rnd(co, ci, 3, 3, scale=(9 * ci) ** -0.5, seed=5)
    b = rnd(co, scale=0.3, seed=6)
    res = rnd(n * hw * hw, co, seed=7).to(H)
    M = n * hw * hw
    out = nan16(M, 64)
    ops.Gemm(ops.conv_taps([x.view(-1, ci)], dilation=d), wt.permute(0, 2, 3, 1).reshape(co, -1).half().contiguous(),
             out[:, co:2 * co], M, mode=ops.ROWS_CONV2D, geom=dict(Ho=hw, Wo=hw, Hs=hw, Ws=hw, stride=1), bias=b,
             act=ops.ACT_RELU, residual=res, engine=engine)()
    ref = F.relu(F.conv2d(x.float().permute(0, 3, 1, 2), wt.half().float(), b, padding=d, dilation=d))
    ref = ref.permute(0, 2, 3, 1).reshape(M, co).half().float() + res.float()
    close(out[:, co:2 * co], ref, name=f"{engine} N={co} slice + residual")
    assert untouched(out[:, :co]) and untouched(out[:, 2 * co:])


# ---- pool, resize, side fusion -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hw", [(20, 20), (13, 21), (7, 11), (1, 3)])
def test_maxpool2x2_ceil_reads_a_channel_slice(hw):
    n, (h, w), c = 2, hw, 32
    buf = rnd(n * h * w, 96, seed=8).to(H)
    ho, wo = (h + 1) // 2, (w + 1) // 2
    y = nan16(n * ho * wo + 2, 64)
    ops.maxpool2x2_ceil(buf[:, 32:64], n, h, w, y[:n * ho * wo, 16:48])
    ref = F.max_pool2d(buf[:, 32:64].float().reshape(n, h, w, c).permute(0, 3, 1, 2), 2, 2, ceil_mode=True)
    assert torch.equal(y[:n * ho * wo, 16:48].float(), ref.permute(0, 2, 3, 1).reshape(-1, c))
    assert untouched(y[:, :16]) and untouched(y[:, 48:]) and untouched(y[n * ho * wo:])


@pytest.mark.parametrize("src,dst", [((10, 10), (320, 320)), ((13, 13), (25, 25)), ((7, 11), (13, 21)), ((1, 1), (5, 5)),
                                     ((40, 40), (13, 17))])
def test_resize_bilinear(src, dst):
    n, c = 2, 16
    x = rnd(n * src[0] * src[1], 48, seed=9).to(H)
    y = nan16(n * dst[0] * dst[1] + 3, 64)
    M = n * dst[0] * dst[1]
    ops.resize_bilinear(x[:, 16:32], n, *src, y[:M, :c], *dst)
    ref = F.interpolate(x[:, 16:32].float().reshape(n, *src, c).permute(0, 3, 1, 2), size=dst, mode="bilinear",
                        align_corners=False).permute(0, 2, 3, 1).reshape(M, c)
    err = (y[:M, :c].float() - ref).abs()
    assert bool((err <= ref.abs() * 2 ** -11 + 1e-6).all()), f"max err {float(err.max()):.3e}"   # one fp16 rounding
    assert untouched(y[:, c:]) and untouched(y[M:])


def test_fuse_sides():
    n, H_, W_ = 2, 97, 131
    sizes = [(97, 131), (49, 66), (25, 33), (13, 17), (7, 9), (4, 5)]
    sides, ref = [], torch.full((n, 1, H_, W_), 0.3, device=DEV)
    for k, (h, w) in enumerate(sizes):
        s = rnd(n * h * w, 8, scale=2.0, seed=10 + k).to(H)
        sides.append((s, h, w))
        ref = ref + F.interpolate(s[:, :1].float().reshape(n, h, w, 1).permute(0, 3, 1, 2), size=(H_, W_), mode="bilinear",
                                  align_corners=False)
    out = torch.full((n, H_, W_), NAN, device=DEV)
    ops.u2net_fuse_sides(sides, 0.3, n, H_, W_, out)
    torch.testing.assert_close(out, torch.sigmoid(ref[:, 0]), atol=2e-6, rtol=1e-5)


# ---- the tower against the fp32 oracle -----------------------------------------------------------------------------------------
def _mask_u8(p):
    """rembg's uint8 mask of each image: min-max normalised, truncated."""
    p = p.double()
    mi = p.amin(dim=(1, 2), keepdim=True)
    ma = p.amax(dim=(1, 2), keepdim=True)
    return ((p - mi) / (ma - mi) * 255).to(torch.uint8)


def _image_like(n, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, 3, h, w, generator=g) * 0.6
    x[:, :, h // 4:3 * h // 4, w // 5:3 * w // 5] += 1.2          # a bright object on a darker background
    return x.to(DEV)


@pytest.mark.parametrize("variant,n,hw", [("full", 1, (320, 320)), ("full", 2, (200, 328)), ("p", 1, (320, 320))])
def test_tower_against_oracle(variant, n, hw):
    from hi3d_official_b200.u2net import U2NetTower
    sd = {k: v.to(DEV) for k, v in UO.random_u2net_sd(seed=21, variant=variant).items()}
    x = _image_like(n, *hw, seed=22)
    with torch.no_grad():
        ref = UO.u2net_forward(sd, x)
        with torch.autocast("cuda", dtype=torch.float16):
            amp = UO.u2net_forward(sd, x).float()
    got = U2NetTower(sd, device=DEV)(x)
    assert got.shape == ref.shape == (n, *hw) and got.dtype == torch.float32
    e, e_amp = UO.relerr(got, ref), UO.relerr(amp, ref)
    m, m_ref, m_amp = _mask_u8(got), _mask_u8(ref), _mask_u8(amp)
    bad = int(((m.int() - m_ref.int()).abs() > 1).sum())
    bad_amp = int(((m_amp.int() - m_ref.int()).abs() > 1).sum())
    print(f"U^2-Net {variant} {n} x {hw}: rel-L2 native {e:.3e}, autocast {e_amp:.3e}; mask levels off by > 1: native {bad}, "
          f"autocast {bad_amp} of {m.numel()}")
    assert e <= 2 * e_amp, f"native error {e:.3e} > 2 x autocast error {e_amp:.3e}"
    assert bad <= max(2 * bad_amp, 0.001 * m.numel())


def test_tower_reuses_its_plan():
    """Buffers and launches are kept per input shape: repeated calls, a shape change and a return to the first shape give what
    a fresh tower gives, and the returned maps are not overwritten by later calls."""
    from hi3d_official_b200.u2net import U2NetTower
    sd = UO.random_u2net_sd(seed=24, variant="p", calib_hw=96)
    tower = U2NetTower(sd, device=DEV)
    xa, xb, xc = _image_like(1, 96, 96, seed=25), _image_like(1, 96, 96, seed=26), _image_like(2, 61, 75, seed=27)
    ya = tower(xa)
    ya_kept = ya.clone()
    yb, yc, ya2 = tower(xb), tower(xc), tower(xa)
    assert torch.equal(ya, ya_kept) and torch.equal(ya2, ya)
    for x, y in ((xb, yb), (xc, yc)):
        assert torch.equal(U2NetTower(sd, device=DEV)(x), y)


@pytest.mark.parametrize("view", ["contiguous", "column slice"])
def test_gemm_rejects_an_fp32_output(view):
    x, w = rnd(128, 64, seed=28).to(H), rnd(32, 64, seed=29).to(H)
    out = torch.full((128, 64), NAN, device=DEV)
    with pytest.raises(ValueError, match="out"):
        ops.Gemm([ops.SegSpec(x)], w, out if view == "contiguous" else out[:, :32], 128, engine="tc5")
    assert bool(torch.isnan(out).all())


def test_tower_rejects_bad_input():
    from hi3d_official_b200.u2net import U2NetTower
    tower = U2NetTower(UO.random_u2net_sd(seed=23, variant="p", calib_hw=32), device=DEV)
    for shape in [(3, 64, 64), (1, 4, 64, 64), (1, 1, 64, 64)]:
        with pytest.raises(ValueError):
            tower(torch.zeros(*shape, device=DEV))


# ---- the pipelines with background removal --------------------------------------------------------------------------------------
def test_pipelines_with_background_removal(tmp_path):
    import cv2
    from PIL import Image
    from hi3d_official_b200 import rembg
    os.makedirs(tmp_path / "ckpts")
    sd = UO.random_u2net_sd(seed=31, variant="p")
    torch.save(sd, tmp_path / "ckpts" / "u2net.pth")
    rs = np.random.RandomState(0)
    a = (rs.rand(200, 160, 3) * 80).astype("uint8")
    a[50:150, 40:120] = (150 + rs.rand(100, 80, 3) * 100).astype("uint8")
    cv2.imwrite(str(tmp_path / "in.png"), a)
    g = torch.Generator().manual_seed(0)
    torch.save({"clip": torch.randn(1, 1024, generator=g), "aes": torch.tensor([[5.2]]),
                "depth": torch.rand(16, 24, 24, generator=g)}, str(tmp_path / "towers.pt"))
    common = ["--tiny", "--output_dir", "out", "--seed", "1", "--towers", "towers.pt"]
    r = subprocess.run([sys.executable, os.path.join(ROOT, "pipeline_i2v_eval_v01.py"), *common, "--image_path", "in.png"],
                       capture_output=True, text=True, timeout=900, cwd=str(tmp_path))
    assert r.returncode == 0, r.stdout[-1500:] + r.stderr[-3000:]
    assert "removed the background" in r.stdout
    rgba = Image.open(tmp_path / "out" / "temp_image" / "rgba.png")
    white = Image.open(tmp_path / "out" / "temp_image" / "white.png")
    assert rgba.mode == "RGBA" and white.mode == "RGB" and rgba.size == white.size == (160, 200)
    # the same cut-out through the fp32 oracle, and through the oracle under fp16 autocast for the error bar
    sd_dev = {k: v.to(DEV) for k, v in sd.items()}

    def oracle(x, amp):
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16, enabled=amp):
            return UO.u2net_forward(sd_dev, torch.from_numpy(x).to(DEV)).float().cpu().numpy()
    ref = UO.rembg_remove(Image.open(tmp_path / "in.png"), lambda x: oracle(x, False))
    ref_amp = UO.rembg_remove(Image.open(tmp_path / "in.png"), lambda x: oracle(x, True))
    with torch.no_grad():
        got = rembg.remove(Image.open(tmp_path / "in.png"), session=rembg.new_session(sd, device=DEV))
    assert np.array_equal(np.array(got), np.array(rgba))          # the script's file is what the session computes
    alpha = lambda im: np.array(im)[..., 3].astype(int)           # noqa: E731
    bad = int((np.abs(alpha(rgba) - alpha(ref)) > 1).sum())
    bad_amp = int((np.abs(alpha(ref_amp) - alpha(ref)) > 1).sum())
    bound = max(2 * bad_amp, 0.001 * alpha(ref).size)
    print(f"cut-out alpha off by > 1: native {bad}, autocast {bad_amp} of {alpha(ref).size}")
    assert bad <= bound
    ref_white = Image.new("RGB", ref.size, "WHITE")
    ref_white.paste(ref, mask=ref.split()[3])
    off = np.abs(np.array(white).astype(int) - np.array(ref_white).astype(int)).max(-1)
    assert int((off > 2).sum()) <= bound
    # stage 2: frame 0 from white.png
    r = subprocess.run([sys.executable, os.path.join(ROOT, "pipeline_i2v_eval_v02.py"), *common],
                       capture_output=True, text=True, timeout=900, cwd=str(tmp_path))
    assert r.returncode == 0, r.stdout[-1500:] + r.stderr[-3000:]
    assert "frame 0 replaced by" in r.stdout
    second = torch.load(tmp_path / "out" / "second_step_video" / "second.pt")
    assert second.shape == (16, 3, 256, 256) and bool(torch.isfinite(second.float()).all())


def test_replace_first_frame(tmp_path):
    import cv2
    from pipeline_i2v_eval_v02 import replace_first_frame
    frames = torch.zeros(4, 3, 64, 64)
    assert not replace_first_frame(frames, str(tmp_path), 64)
    os.makedirs(tmp_path / "temp_image")
    a = (np.random.RandomState(1).rand(90, 70, 3) * 255).astype("uint8")
    cv2.imwrite(str(tmp_path / "temp_image" / "white.png"), a)
    assert replace_first_frame(frames, str(tmp_path), 64)
    ref = cv2.cvtColor(cv2.resize(a, [64, 64]), cv2.COLOR_BGR2RGB)
    torch.testing.assert_close(frames[0], (torch.from_numpy(ref).permute(2, 0, 1).float() / 255 - 0.5) * 2)
    assert not frames[1:].any()
