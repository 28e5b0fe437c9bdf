"""TMA + wgmma spatial attention (hi3d_attention_d64_tc5) against PyTorch fp32 softmax(QK^T/8)V and against the
mma.sync kernel, incl. sequence lengths that are not a multiple of the key tile."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from hi3d_official_b200 import _native, ops  # noqa: E402
from test_kernels_gpu import DEV, H, close, rnd  # noqa: E402


@pytest.fixture(params=[(0, 0), (0, 1), (0, 2), (1, 0), (1, 1), (1, 2), (2, 0), (2, 1), (2, 2), (2, 4), (2, 5), (2, 6), (3, 0), (3, 1), (3, 3), (4, 0), (4, 1), (4, 2), (6, 0), (6, 1), (6, 5)],
                ids=["shared-mufu", "shared-emu25", "shared-emu50", "split-mufu", "split-emu25", "split-emu50",
                     "lean-mufu", "lean-emu25", "lean-emu50", "lean-emu100", "lean-emu37", "lean-emu12", "anyorder-mufu", "anyorder-emu25", "anyorder-emu75",
                     "pingpong-mufu", "pingpong-emu25", "pingpong-emu50",
                     "blocks-mufu", "blocks-emu25", "blocks-emu37"],
                autouse=True)
def kernel_variant(request):
    """Every case runs on several kernel variants (key tile 64 / 128, K/V ring depth 2 .. 5; the ids keep the names of the
    project's earlier kernel variants) with part of the softmax exponentials on the FMA pipe (cubic polynomial) -- the
    production default is one of them (attn_tc5.cu FA_VARIANT_DEFAULT, FA_EMU_DEFAULT)."""
    lib = _native.load()
    variant, emu = request.param
    _native.check(lib.hi3d_attention_tc5_set_variant(variant), "set_variant")
    _native.check(lib.hi3d_attention_tc5_set_exp_emulation(emu), "set_exp_emulation")
    yield request.param
    _native.check(lib.hi3d_attention_tc5_set_variant(6), "set_variant")            # back to the production defaults
    _native.check(lib.hi3d_attention_tc5_set_exp_emulation(0), "set_exp_emulation")


def ref_attn(qkv, n_img, L, heads):
    C = heads * 64
    q, k, v = (t.view(n_img, L, heads, 64).transpose(1, 2).float() for t in qkv.view(n_img * L, 3, C).unbind(1))
    return torch.softmax(q @ k.transpose(-1, -2) * 0.125, -1) @ v


@pytest.mark.parametrize("n_img,L,heads,scale", [(1, 128, 1, 1.0), (2, 256, 2, 1.0), (3, 1024, 5, 1.0), (1, 4096, 2, 1.0),
                                                 (2, 1024, 3, 3.0), (1, 384, 1, 0.3), (1, 512, 1, 1.0), (2, 16384, 1, 1.0),
                                                 (1, 640, 2, 6.0)])
def test_attention_tc5(n_img, L, heads, scale):
    C = heads * 64
    qkv = (rnd(n_img * L, 3 * C) * scale).to(H)
    out = torch.zeros(n_img * L, C, dtype=H, device=DEV)
    ops.attention_d64(qkv, n_img, L, heads, out, engine="tc5")
    ref = ref_attn(qkv, n_img, L, heads)
    # P is fp16 (2^-11 relative) against fp32 softmax weights: the error bound scales with max |v| (~ 4 * scale)
    close(out.view(n_img, L, heads, 64).transpose(1, 2), ref, atol=2e-3 * max(1.0, scale), name="fmha tc5")
    out2 = torch.zeros_like(out)
    ops.attention_d64(qkv, n_img, L, heads, out2, engine="mma")
    close(out, out2, atol=8e-3, name="tc5 vs mma")     # two fp16 results: one ulp at |x| ~ 8 is 7.8e-3


def test_attention_tc5_ragged_forwards():
    n_img, L, heads = 2, 100, 2
    qkv = rnd(n_img * L, 3 * heads * 64).to(H)
    out = torch.zeros(n_img * L, heads * 64, dtype=H, device=DEV)
    ops.attention_d64(qkv, n_img, L, heads, out, engine="tc5")
    close(out.view(n_img, L, heads, 64).transpose(1, 2), ref_attn(qkv, n_img, L, heads), atol=2e-3, name="ragged")


@pytest.mark.parametrize("ramp", ["up", "down", "spike"])
def test_attention_tc5_moving_maximum(ramp):
    """Keys whose scores rise, fall or spike along the sequence: the running maximum of the online softmax moves (and the
    accumulator is rescaled) many times inside one call."""
    n_img, L, heads = 1, 1024, 2
    C = heads * 64
    qkv = rnd(n_img * L, 3, C)
    pos = torch.arange(L, device=DEV, dtype=torch.float32) / L
    if ramp == "up":
        gain = 0.2 + 4.0 * pos                      # later key tiles dominate: the maximum keeps moving
    elif ramp == "down":
        gain = 4.2 - 4.0 * pos                      # first tile holds the maximum: single-read path afterwards
    else:
        gain = torch.full_like(pos, 0.5)
        gain[L // 2 + 7] = 12.0                     # one huge key in the middle of the sequence
    qkv[:, 1] *= gain[:, None]
    qkv = qkv.reshape(n_img * L, 3 * C).to(H)
    out = torch.zeros(n_img * L, C, dtype=H, device=DEV)
    ops.attention_d64(qkv, n_img, L, heads, out, engine="tc5")
    close(out.view(n_img, L, heads, 64).transpose(1, 2), ref_attn(qkv, n_img, L, heads), atol=3e-3, name=f"fmha tc5 {ramp}")
