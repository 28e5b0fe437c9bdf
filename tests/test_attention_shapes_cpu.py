"""ops.attention_shapes without a GPU: the size, frame-count and L % 128 checks that every fp16 / e4m3 attention entry point runs
before it launches, on meta tensors (nothing is allocated or launched)."""
import pytest
import torch

from hi3d_official_b200 import ops

META = dict(device="meta", dtype=torch.float16)


def _t(rows, cols):
    return torch.empty(rows, cols, **META)


@pytest.mark.parametrize("d", [64, 80])
def test_spatial_sizes_fit_exactly(d):
    n_img, L, heads = 3, 193, 5
    C = heads * d
    ops.attention_shapes("a", _t(n_img * L, 3 * C), _t(n_img * L, C), n_img, L, heads, d)
    ops.attention_shapes("a", _t(n_img * L + 7, 3 * C), _t(n_img * L + 256, C), n_img, L, heads, d)     # larger buffers are fine
    with pytest.raises(ValueError, match="qkv"):
        ops.attention_shapes("a", _t(n_img * L - 1, 3 * C), _t(n_img * L, C), n_img, L, heads, d)
    with pytest.raises(ValueError, match="out"):
        ops.attention_shapes("a", _t(n_img * L, 3 * C), _t(n_img * L - 1, C), n_img, L, heads, d)
    with pytest.raises(ValueError, match="qkv"):                        # row stride of another head count
        ops.attention_shapes("a", _t(n_img * L * 2, 3 * (heads - 1) * d), _t(n_img * L, C), n_img, L, heads, d)
    with pytest.raises(ValueError, match="out"):
        ops.attention_shapes("a", _t(n_img * L, 3 * C), _t(n_img * L * 2, C - d), n_img, L, heads, d)
    with pytest.raises(ValueError, match="qkv"):                        # a flat buffer has no row stride of 3C
        ops.attention_shapes("a", torch.empty(n_img * L * 3 * C, **META), _t(n_img * L, C), n_img, L, heads, d)


@pytest.mark.parametrize("n_img,L,heads", [(0, 64, 1), (1, 0, 1), (1, 64, 0), (-1, -64, 1)])
def test_nonpositive_geometry_refused(n_img, L, heads):
    with pytest.raises(ValueError, match="geometry"):
        ops.attention_shapes("a", _t(64, 192), _t(64, 64), n_img, L, heads, 64)


@pytest.mark.parametrize("T", [1, 5, 16])
def test_temporal_rows_count_frames(T):
    B, S, heads = 2, 37, 3
    C = heads * 64
    rows = B * T * S
    ops.attention_shapes("t", _t(rows, 3 * C), _t(rows, C), B, S, heads, 64, T=T)
    with pytest.raises(ValueError, match="qkv"):
        ops.attention_shapes("t", _t(rows - 1, 3 * C), _t(rows, C), B, S, heads, 64, T=T)
    with pytest.raises(ValueError, match="out"):
        ops.attention_shapes("t", _t(rows, 3 * C), _t(B * S * max(T - 1, 0) + S - 1, C), B, S, heads, 64, T=T)


@pytest.mark.parametrize("T", [0, 17, 64])
def test_temporal_frame_count_limited_to_16(T):
    B, S = 1, 8
    with pytest.raises(ValueError, match="T must be 1 .. 16"):
        ops.attention_shapes("t", _t(B * max(T, 1) * S, 192), _t(B * max(T, 1) * S, 64), B, S, 1, 64, T=T)


@pytest.mark.parametrize("L,ok", [(128, True), (4096, True), (64, False), (200, False), (16448, False)])
def test_d512_needs_l_multiple_of_128(L, ok):
    n_img = 2
    qkv, out = _t(n_img * L, 1536), _t(n_img * L, 512)
    if ok:
        ops.attention_shapes("d512", qkv, out, n_img, L, 1, 512, L_multiple=128)
    else:
        with pytest.raises(ValueError, match="multiple of 128"):
            ops.attention_shapes("d512", qkv, out, n_img, L, 1, 512, L_multiple=128)


def test_entry_points_check_before_any_launch(monkeypatch):
    """Every attention entry point hands its geometry to attention_shapes after the dtype / device checks and before it touches
    the library: with those checks passed by a stub and the library replaced by one that fails when called, an undersized
    buffer must raise ValueError, not reach the library."""
    seen = []

    class NoLib:
        def __getattr__(self, name):
            raise AssertionError(f"{name} was called for a geometry that does not fit")

    monkeypatch.setattr(ops, "_chk16", lambda t, name: None)
    monkeypatch.setattr(ops, "_chk8", lambda t, name: None)
    monkeypatch.setattr(ops.N, "load", lambda *a, **k: NoLib())
    real = ops.attention_shapes

    def spy(name, *a, **k):
        seen.append(name)
        return real(name, *a, **k)

    monkeypatch.setattr(ops, "attention_shapes", spy)
    small = _t(10, 192), _t(10, 64)
    with pytest.raises(ValueError):
        ops.attention_d64(small[0], 2, 10, 1, small[1], engine="tc5")
    with pytest.raises(ValueError):
        ops.attention_d64(small[0], 2, 10, 1, small[1], engine="mma")
    with pytest.raises(ValueError):
        ops.attention_d80(_t(10, 240), 2, 10, 1, _t(10, 80))
    with pytest.raises(ValueError):
        ops.attention_d512(_t(128, 1536), 2, 128, _t(256, 512))
    with pytest.raises(ValueError):
        ops.attention_d512(_t(200, 1536), 1, 200, _t(200, 512))
    with pytest.raises(ValueError):
        ops.temporal_attention_d64(_t(16 * 4, 192), 1, 17, 4, 1, _t(17 * 4, 64))
    with pytest.raises(ValueError):
        ops.temporal_attention_d64(small[0], 1, 2, 10, 1, small[1])
    e4m3 = torch.empty(10, 192, device="meta", dtype=torch.float8_e4m3fn)
    with pytest.raises(ValueError):
        ops.attention_d64_fp8(e4m3, e4m3, 2, 10, 1, small[1])
    assert seen == ["attention_d64", "attention_d64", "attention_d80", "attention_d512", "attention_d512",
                    "temporal_attention_d64", "temporal_attention_d64", "attention_d64_fp8"]
