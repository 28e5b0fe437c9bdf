"""FP8 spatial attention without a GPU: the --precision fp8_attn flag, the plan's frame-sharding refusal, the size and the key
permutation of the transposed V buffer, and the kernel's register budget."""
import argparse
import os
import re
import shutil
import subprocess

import pytest

import pipeline_i2v_eval_v01 as P1
from hi3d_official_b200 import _native, build, ops

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("stage", [1, 2])
def test_precision_flag_takes_fp8_attn(stage):
    ap = argparse.ArgumentParser()
    P1.add_cli_args(ap, stage)
    assert ap.parse_args(["--precision", "fp8_attn"]).precision == "fp8_attn"
    assert ap.parse_args(["--precision", "fp8"]).precision == "fp8"
    with pytest.raises(SystemExit):
        ap.parse_args(["--precision", "bf16"])


def test_fp8_attn_with_frame_sharding_refused_before_packing():
    from hi3d_official_b200.unet import PRECISIONS, VideoUNet
    assert PRECISIONS == ("fp16", "fp8", "fp8_attn")
    kw = dict(adm_in_channels=768, num_classes="sequential", in_channels=8, out_channels=4, model_channels=64,
              attention_resolutions=[4, 2, 1], num_res_blocks=2, channel_mult=[1, 2, 4, 4], num_head_channels=64,
              use_linear_in_transformer=True, transformer_depth=1, context_dim=1024, extra_ff_mix_layer=True,
              use_spatial_context=True, merge_strategy="learned_with_images", video_kernel_size=[3, 1, 1])
    net = VideoUNet(**kw)                               # CPU parameters: packing would refuse them, so reaching it would fail
    net.set_precision("fp8_attn")
    with pytest.raises(NotImplementedError, match="frame-sharded"):
        net.get_plan(16, 16, 16, 8, shard=(0, 2))
    assert net._packed is None and net._plans == {}


@pytest.mark.parametrize("n_img,L,heads", [(1, 1, 1), (3, 77, 2), (2, 128, 5), (32, 16384, 5), (32, 1000, 20), (1, 129, 1)])
def test_vt_bytes(n_img, L, heads):
    assert ops.attention_vt_bytes(n_img, L, heads) == n_img * heads * 64 * ((L + 127) // 128 * 128)


def test_vt_bytes_refuses_bad_arguments():
    with pytest.raises(_native.Hi3dError):
        ops.attention_vt_bytes(0, 128, 1)


def pi(k: int) -> int:
    """Key held by column k of a 32-block of vt, as include/hi3d_b200.h states it."""
    return (k & 16) + 8 * ((k >> 1) & 1) + 2 * ((k >> 2) & 3) + (k & 1)


def test_pi_is_a_bijection_that_maps_s_fragments_to_a_fragments():
    assert sorted(pi(k) for k in range(32)) == list(range(32))
    hdr = open(os.path.join(ROOT, "include", "hi3d_b200.h")).read()
    assert "pi(k) = (k & 16) + 8*((k >> 1) & 1) + 2*((k >> 2) & 3) + (k & 1)" in hdr
    # lane t4 of a quad holds S columns 8 i + 2 t4 + {0, 1} (f32 accumulator) and A columns 4 t4 + 0..3, 16 + 4 t4 + 0..3 (8-bit
    # k32 A fragment): with keys permuted by pi both name the same eight keys, in register byte order
    for t4 in range(4):
        s_keys = [8 * i + 2 * t4 + e for i in range(4) for e in range(2)]
        a_keys = [pi(k) for k in list(range(4 * t4, 4 * t4 + 4)) + list(range(16 + 4 * t4, 20 + 4 * t4))]
        assert a_keys == s_keys


@pytest.mark.skipif(shutil.which("nvcc") is None and not os.path.exists("/usr/local/cuda/bin/nvcc"), reason="needs nvcc")
def test_fp8_attention_kernel_compiles_without_spills(tmp_path):
    nvcc = build._nvcc()
    src = os.path.join(build.CSRC, "attn_fp8_tc5.cu")
    r = subprocess.run([nvcc] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "a.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    kernels = re.findall(r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads",
                         r.stderr)
    assert {k for k, *_ in kernels} >= {"_ZN4hi3d15fmha_fp8_kernelENS_9Fa8ParamsE", "_ZN4hi3d14vt_e4m3_kernelEPKhiiiPh"}, r.stderr
    for name, frame, st, ld in kernels:
        assert (int(frame), int(st), int(ld)) == (0, 0, 0), f"{name}: stack {frame}, spill stores {st}, spill loads {ld}"
