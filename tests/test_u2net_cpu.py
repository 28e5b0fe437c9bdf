"""U^2-Net background removal without a GPU: the graph's size (parameters, state-dict keys, FLOPs), the loader, the load-time
folding of BatchNorm and outconv (fp64 against the unfolded oracle), and the rembg surface with the network replaced by the fp32
oracle, bit for bit against the literal restatement of rembg's host steps."""
import io

import numpy as np
import pytest
import torch

import u2net_oracle as UO
from hi3d_official_b200 import rembg, u2net


@pytest.fixture(scope="module")
def sds():
    return {v: UO.random_u2net_sd(seed=1, variant=v) for v in ("full", "p")}


@pytest.mark.parametrize("variant,params", [("full", 44_009_869), ("p", 1_131_181)])
def test_parameter_and_key_counts(sds, variant, params):
    sd = sds[variant]
    assert u2net.param_count(sd) == params
    assert len(sd) == 798
    assert sum(1 for k, v in sd.items() if k.endswith("weight") and v.dim() == 4) == 119
    assert set(u2net.live_state_dict(sd)) == u2net.expected_keys()


def test_flops_at_320():
    from torch.utils.flop_counter import FlopCounterMode
    for variant, gflop in (("full", 117.2), ("p", 39.5)):
        sd = UO.random_u2net_sd(seed=2, variant=variant, calib_hw=32)
        with FlopCounterMode(display=False) as fc, torch.no_grad():
            UO.u2net_forward(sd, torch.zeros(1, 3, 320, 320))
        assert abs(fc.get_total_flops() / 1e9 - gflop) < 0.05, (variant, fc.get_total_flops())


@pytest.mark.parametrize("hw", [(200, 328), (97, 131)])
def test_odd_sizes_run(sds, hw):
    with torch.no_grad():
        y = UO.u2net_forward(sds["p"], torch.randn(1, 3, *hw))
    assert y.shape == (1, *hw) and bool(torch.isfinite(y).all())


# ---- loader ---------------------------------------------------------------------------------------------------------------------
def _roundtrip(tmp_path, sd):
    p = tmp_path / "u2net.pth"
    torch.save(sd, p)
    return u2net.load_u2net(str(p))


def test_loader_plain_and_prefixed(tmp_path, sds):
    sd = sds["p"]
    got = _roundtrip(tmp_path, sd)
    assert set(got) == u2net.expected_keys()                       # num_batches_tracked dropped
    assert all(torch.equal(got[k], sd[k]) for k in got)
    got = _roundtrip(tmp_path, {"module." + k: v for k, v in sd.items()})
    assert set(got) == u2net.expected_keys()


def test_loader_rejects_missing_and_unexpected(tmp_path, sds):
    sd = dict(sds["p"])
    del sd["stage3d.rebnconv2d.bn_s1.running_var"]
    with pytest.raises(KeyError, match="missing"):
        _roundtrip(tmp_path, sd)
    sd = dict(sds["p"])
    sd["stage7.rebnconvin.conv_s1.weight"] = torch.zeros(1)
    with pytest.raises(KeyError, match="unexpected"):
        _roundtrip(tmp_path, sd)


def test_loader_ignores_num_batches_tracked(sds):
    sd = {k: v for k, v in sds["p"].items() if not k.endswith("num_batches_tracked")}
    assert set(u2net.live_state_dict(sd)) == u2net.expected_keys()


# ---- folding ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", ["full", "p"])
def test_folding_equals_unfolded_fp64(sds, variant):
    sd = {k: v.double() if v.is_floating_point() else v for k, v in sds[variant].items()}
    x = torch.randn(1, 3, 64, 80, generator=torch.Generator().manual_seed(3), dtype=torch.float64)
    with torch.no_grad():
        ref = UO.u2net_d0(sd, x)
        got = UO.folded_d0(u2net.fold(sd), x)
    assert UO.relerr(got, ref) < 1e-12
    assert float(ref.std()) > 2.0, "d0 spread too small for a meaningful min-max normalised mask"


# ---- the rembg surface ------------------------------------------------------------------------------------------------------------
def _oracle_session(sd):
    return rembg.U2netSession(lambda x: UO.u2net_forward(sd, x.float()))


def _rgb(w, h, seed):
    from PIL import Image
    rs = np.random.RandomState(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    blob = ((yy - h / 2) ** 2 / (h / 3) ** 2 + (xx - w / 2) ** 2 / (w / 3) ** 2 < 1)[..., None]
    a = np.where(blob, rs.randint(120, 255, (h, w, 3)), rs.randint(0, 90, (h, w, 3))).astype("uint8")
    return Image.fromarray(a, "RGB")


def test_remove_matches_literal_rgb(sds):
    img = _rgb(173, 121, seed=4)
    with torch.no_grad():
        got = rembg.remove(img, session=_oracle_session(sds["p"]))
        ref = UO.rembg_remove(img, lambda a: UO.u2net_forward(sds["p"], torch.from_numpy(a)).numpy())
    assert got.mode == "RGBA" and got.size == img.size
    assert np.array_equal(np.array(got), np.array(ref))
    alpha = np.array(got)[..., 3]
    assert alpha.min() < 64 and alpha.max() > 192


def test_remove_matches_literal_rgba_exif_rotated(sds):
    from PIL import Image
    base = _rgb(150, 96, seed=5).convert("RGBA")
    base.putalpha(200)
    exif = Image.Exif()
    exif[0x0112] = 6                                               # orientation: rotate 90 degrees clockwise to display
    buf = io.BytesIO()
    base.save(buf, format="PNG", exif=exif)
    img = Image.open(io.BytesIO(buf.getvalue()))
    with torch.no_grad():
        got = rembg.remove(img, session=_oracle_session(sds["p"]))
        img2 = Image.open(io.BytesIO(buf.getvalue()))
        ref = UO.rembg_remove(img2, lambda a: UO.u2net_forward(sds["p"], torch.from_numpy(a)).numpy())
    assert got.size == (96, 150)                                  # transposed by the EXIF orientation
    assert np.array_equal(np.array(got), np.array(ref))


def test_new_session_without_weights(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    with pytest.raises(FileNotFoundError):
        rembg.new_session()


# ---- the graph table against the oracle's own, and the GEMM wrapper's output checks -----------------------------------------------
def test_graph_table_matches_u2net():
    """The module's stage kinds and dilations against the table the oracle states from U-2-Net's model/u2net.py."""
    assert {s: (L, pooled) for s, L, pooled in u2net.STAGES} == UO.STAGE_KIND
    for stage, (L, pooled) in UO.STAGE_KIND.items():
        assert u2net.rsu_convs(L, pooled) == list(UO.DILATIONS[(L, pooled)].items()), stage
    f = u2net.fold(UO.random_u2net_sd(seed=6, variant="p", calib_hw=32))
    for stage, kind in UO.STAGE_KIND.items():
        for name, d in UO.DILATIONS[kind].items():
            assert f[f"{stage}.{name}"][2] == d, (stage, name)


@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
@pytest.mark.parametrize("view", ["contiguous", "column slice"])
def test_gemm_rejects_an_output_off_the_gpu(dtype, view):
    """ops.Gemm takes a contiguous CUDA fp16 output or a column slice of one; anything else is refused before any launch."""
    from hi3d_official_b200 import ops
    out = torch.zeros(128, 64, dtype=dtype)
    if view == "column slice":
        out = out[:, 16:48]
    with pytest.raises(ValueError, match="out"):
        ops.Gemm([], torch.zeros(32, 64, dtype=torch.float16), out, 128)
