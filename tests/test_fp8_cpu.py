"""FP8 sampling without a GPU: the e4m3 weight packing, the --precision flag of the entry points, and the plan refusing fp8 with
frame sharding before anything is packed or allocated."""
import argparse

import pytest
import torch

import pipeline_i2v_eval_v01 as P1
from hi3d_official_b200 import pack

E4M3 = torch.float8_e4m3fn


def test_pack_e4m3_scales_rounding_and_zero_rows():
    w = torch.zeros(4, 6, dtype=torch.float16)
    # row 0: amax 448 -> scale 1; 1.0625 and 1.1875 lie halfway between e4m3 neighbours (steps of 1/8 in [1, 2)): nearest even
    w[0, :4] = torch.tensor([448.0, 1.0625, 1.1875, -1.0625])
    w[1, :3] = torch.tensor([0.5, -2.0, 1.0])           # amax 2 -> scale 2/448, the amax element becomes exactly -448
    w[3, 0] = 1000.0                                    # 1000 / (1000 / 448) may round above 448 in fp32: saturates, no NaN
    q, sc = pack.pack_e4m3(w)
    assert q.dtype == E4M3 and sc.dtype == torch.float32 and q.shape == w.shape and sc.shape == (4,)
    assert sc[0] == 1.0 and sc[2] == 1.0                # row 2 is all zero: scale 1
    assert torch.allclose(sc[1], torch.tensor(2.0 / 448)) and torch.allclose(sc[3], torch.tensor(1000.0 / 448))
    assert q[0, :4].float().tolist() == [448.0, 1.0, 1.25, -1.0]
    assert float(q[1, 1]) == -448.0
    assert float(q[3, 0]) == 448.0 and not torch.isnan(q.float()).any()
    assert (q[2].float() == 0).all() and (q[:, 4:].float() == 0).all()
    # dequantised weights are within half an e4m3 step (2^-4 relative) of the fp16 ones
    deq = q.float() * sc[:, None]
    assert ((deq - w.float()).abs() <= w.float().abs() / 16 + 1e-12).all()


def test_pack_e4m3_keeps_k_padding_zero():
    g = torch.Generator().manual_seed(0)
    w16 = pack.pack_conv2d(torch.randn(8, 5, 3, 3, generator=g), cin_pad=64)       # [8, 9 * 64], 59 zero columns per tap
    q, sc = pack.pack_e4m3(w16)
    pad = torch.ones(9, 64, dtype=torch.bool)
    pad[:, :5] = False
    assert (q.float().view(8, 9, 64)[:, pad] == 0).all()
    assert (q.float().view(8, 9, 64)[:, ~pad] != 0).any()
    with pytest.raises(ValueError):
        pack.pack_e4m3(w16.float())


@pytest.mark.parametrize("stage", [1, 2])
def test_precision_flag(stage):
    ap = argparse.ArgumentParser()
    P1.add_cli_args(ap, stage)
    assert ap.parse_args([]).precision == "fp16"
    assert ap.parse_args(["--precision", "fp8"]).precision == "fp8"
    with pytest.raises(SystemExit):
        ap.parse_args(["--precision", "bf16"])


def test_fp8_with_frame_sharding_refused_before_packing():
    from hi3d_official_b200.unet import VideoUNet
    kw = dict(adm_in_channels=768, num_classes="sequential", in_channels=8, out_channels=4, model_channels=64,
              attention_resolutions=[4, 2, 1], num_res_blocks=2, channel_mult=[1, 2, 4, 4], num_head_channels=64,
              use_linear_in_transformer=True, transformer_depth=1, context_dim=1024, extra_ff_mix_layer=True,
              use_spatial_context=True, merge_strategy="learned_with_images", video_kernel_size=[3, 1, 1])
    net = VideoUNet(**kw)                               # CPU parameters: packing would refuse them, so reaching it would fail
    with pytest.raises(ValueError):
        net.set_precision("bf16")
    net.set_precision("fp8")
    with pytest.raises(NotImplementedError, match="frame-sharded"):
        net.get_plan(16, 16, 16, 8, shard=(0, 2))
    assert net._packed is None and net._plans == {}


def test_fp8_coverage_query():
    """hi3d_gemm_tc5_fp8_covers answers from the geometry alone (no device), with the engine's own tiling rules."""
    from hi3d_official_b200 import ops
    T = ops.ROWS_TEMPORAL
    assert ops.fp8_covers(T, 32 * 1024, 320, dict(Ho=1024, Wo=1, T=16))
    assert not ops.fp8_covers(T, 32 * 4, 256, dict(Ho=4, Wo=1, T=16))         # 4 pixels x 32 frames per tile > 16 frames
    assert ops.fp8_covers(ops.ROWS_CONV2D, 32 * 4, 256, dict(Ho=2, Wo=2))     # 2 x 2 x 32 images
    assert not ops.fp8_covers(ops.ROWS_CONV2D, 8 * 4, 256, dict(Ho=2, Wo=2))  # 8 images < 32 per tile
    assert not ops.fp8_covers(ops.ROWS_CONV2D, 32 * 64, 256, dict(Ho=8, Wo=8, ups=1))
    assert ops.fp8_covers(ops.ROWS_PLAIN, 77, 64) and not ops.fp8_covers(ops.ROWS_PLAIN, 77, 16)
