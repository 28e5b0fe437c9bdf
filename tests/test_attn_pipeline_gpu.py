"""The warp-specialised, software-pipelined d = 64 attention kernel (hi3d_attention_d64_tc5) where test_attn_tc5_gpu.py does
not reach: the benchmark's full ds1 shape (sampled against fp32 softmax(QK^T/8)V, and bit-identical across two runs, which a
barrier race in the K / V rings or the intra-warpgroup pipeline would break) and sequence lengths at and around the query
tiles of every variant with several images, where the masked key tail of one image reads the next image's rows."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from hi3d_official_b200 import _native, ops  # noqa: E402
from test_kernels_gpu import DEV, H, close, rnd  # noqa: E402


def ref_slice(qkv, n_img, L, heads, img, head, q0, nq):
    """fp32 softmax(QK^T/8)V of queries q0 .. q0 + nq - 1 of one (image, head)."""
    C = heads * 64
    x = qkv.view(n_img, L, 3, C)[img, :, :, head * 64:(head + 1) * 64].float()
    q, k, v = x[q0:q0 + nq, 0], x[:, 1], x[:, 2]
    return torch.softmax(q @ k.t() * 0.125, -1) @ v


def test_bench_shape_sampled_and_deterministic():
    n_img, L, heads = 32, 16384, 5
    C = heads * 64
    qkv = rnd(n_img * L, 3 * C, seed=11).to(H)
    out = torch.zeros(n_img * L, C, dtype=H, device=DEV)
    ops.attention_d64(qkv, n_img, L, heads, out, engine="tc5")
    out2 = torch.full_like(out, float("nan"))
    ops.attention_d64(qkv, n_img, L, heads, out2, engine="tc5")
    torch.cuda.synchronize()
    assert torch.equal(out, out2), f"two runs differ in {int((out != out2).sum())} elements"
    o = out.view(n_img, L, heads, 64)
    for img, head, blk in [(0, 0, 0), (0, 4, 127), (7, 2, 64), (13, 1, 5), (21, 3, 100), (31, 0, 33), (31, 4, 127)]:
        q0 = blk * 128
        close(o[img, q0:q0 + 128, head], ref_slice(qkv, n_img, L, heads, img, head, q0, 128), atol=2e-3,
              name=f"ds1 image {img} head {head} queries {q0}..")


@pytest.mark.parametrize("variant", range(7))
@pytest.mark.parametrize("L", [191, 192, 193, 4097])
def test_tile_edges_several_images(L, variant):
    lib = _native.load()
    _native.check(lib.hi3d_attention_tc5_set_variant(variant), "set_variant")
    try:
        n_img, heads = 3, 2
        C = heads * 64
        qkv = rnd(n_img * L, 3 * C, seed=L).to(H)
        guard = 256                                        # rows past the last image must stay untouched
        buf = torch.full(((n_img * L + guard), C), float("nan"), dtype=H, device=DEV)
        ops.attention_d64(qkv, n_img, L, heads, buf[:n_img * L], engine="tc5")
        torch.cuda.synchronize()
        assert bool(buf[n_img * L:].isnan().all()), "stores past the last image's rows"
        out = buf[:n_img * L].view(n_img, L, heads, 64)
        for img in range(n_img):
            for head in range(heads):
                close(out[img, :, head], ref_slice(qkv, n_img, L, heads, img, head, 0, L), atol=2e-3,
                      name=f"L {L} variant {variant} image {img} head {head}")
    finally:
        _native.check(lib.hi3d_attention_tc5_set_variant(6), "set_variant")
