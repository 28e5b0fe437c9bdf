"""The wgmma engine's ping-pong schedule (hi3d_gemm_tc5 on short-K fp16 GEMMs with at least one tile per SM) against its
single-tile schedule (hi3d_gemm_tc5_set_pair_mode(0)), bit for bit.

Both run the same k16 wgmma sequence in the same K order for every output element, and the same epilogue arithmetic in the
same order, so the outputs must be equal, not merely close.  Every case first asks hi3d_gemm_tc5_schedule which kernel runs,
so that no case can pass without the ping-pong kernel having run (or, for the cases below its tile-count rule, without the
single-tile kernel having been chosen).  Outputs are written into buffers pre-filled with a sentinel, with extra rows and,
where the layout allows, extra columns: nothing outside the result may change."""
import ctypes

import pytest
import torch

pytestmark = pytest.mark.gpu

from hi3d_official_b200 import _native, ops, pack  # noqa: E402

DEV, H = "cuda", torch.float16
PINGPONG, SINGLE = 3, 1
SENTINEL = 7.0


def _lib():
    return _native.load()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(*shape, generator=g, device=DEV) * scale).to(H)


def _schedule(g):
    r = _lib().hi3d_gemm_tc5_schedule(ctypes.byref(g.p))
    assert r >= 0, _lib().hi3d_last_error()
    return r // 1000, r % 1000


def _plain(M, N, K, *, act=ops.ACT_NONE, residual=False, blend=False, rowbias=False, seed=0):
    a = _rnd(M, K, seed=seed)
    bias = torch.randn(N, device=DEV) * 0.1
    if act == ops.ACT_GEGLU:
        w, bias = pack.pack_geglu(torch.randn(N, K, device=DEV) * K ** -0.5, bias)
    else:
        w = _rnd(N, K, scale=K ** -0.5, seed=seed + 1)
    n_out = N // 2 if act == ops.ACT_GEGLU else N
    res = _rnd(M, n_out, seed=seed + 2) if residual else None
    bx = _rnd(M, n_out, seed=seed + 3) if blend else None
    rb = _rnd(2, N, scale=0.5, seed=seed + 4) if rowbias else None

    def make(out):
        return ops.Gemm([ops.SegSpec(a)], w, out[:M, :n_out], M, bias=bias, act=act, residual=res, blend_x=bx,
                        alpha=0.3 if blend else 0.0, rowbias=rb, rb_div=M // 2 if rowbias else 1, rb_mod=2 if rowbias else 1,
                        engine="tc5")
    return make, M, n_out


def _check(make, rows, cols, want=PINGPONG):
    """make(out) -> ops.Gemm writing into out[:rows, :cols] of a sentinel-filled buffer with 64 more rows and 16 more columns.
    The automatic choice must be `want`; its output must equal the single-tile kernel's, border included.  Returns the
    automatic choice's tile width."""
    lib = _lib()
    outs, widths = [], []
    for mode in (-1, 0):
        _native.check(lib.hi3d_gemm_tc5_set_pair_mode(mode), "set_pair_mode")
        try:
            out = torch.full((rows + 64, cols + 16), SENTINEL, dtype=H, device=DEV)
            g = make(out)
            sched, bn = _schedule(g)
            assert sched == (want if mode == -1 else SINGLE), (mode, sched, bn)
            widths.append(bn)
            g()
            torch.cuda.synchronize()
            outs.append(out)
        finally:
            _native.check(lib.hi3d_gemm_tc5_set_pair_mode(-1), "set_pair_mode")
    a, b = outs
    assert torch.isfinite(a[:rows, :cols]).all()
    assert torch.equal(a, b), f"max |diff| {(a.float() - b.float()).abs().max().item()}"
    assert (a[rows:] == SENTINEL).all() and (a[:, cols:] == SENTINEL).all()
    return widths[0]


# the stage-2 UNet's short-K GEMMs at full size (2 x 16 frames of 128 x 128 latents at ds1 = 524288 rows, C = 320)
ROWS = 2 * 16 * 128 * 128


def test_ff1_geglu():
    _check(*_plain(ROWS, 2560, 320, act=ops.ACT_GEGLU))


def test_qkv():
    _check(*_plain(ROWS, 960, 320, seed=1))


def test_to_out_residual_rowbias():
    _check(*_plain(ROWS, 320, 320, residual=True, rowbias=True, seed=2))


def test_ff2_residual():
    _check(*_plain(ROWS, 320, 1280, residual=True, seed=3))


def test_temporal_ff2_residual_blend():
    _check(*_plain(ROWS, 320, 1280, residual=True, blend=True, seed=4))


def test_temporal_conv_residual_blend():
    b, T, hw, c = 2, 16, 128 * 128, 320
    M = b * T * hw
    xh = _rnd(M, c, seed=5)
    w = pack.pack_conv3d_t(torch.randn(c, c, 3, 1, 1, device=DEV) * (3 * c) ** -0.5)
    bias = torch.randn(c, device=DEV) * 0.1
    res, bx = _rnd(M, c, seed=6), _rnd(M, c, seed=7)

    def make(out):
        return ops.Gemm(ops.temporal_taps(xh), w, out[:M, :c], M, mode=ops.ROWS_TEMPORAL, geom=dict(Ho=hw, Wo=1, T=T),
                        bias=bias, residual=res, blend_x=bx, alpha=0.4, engine="tc5")
    _check(make, M, c)


def _conv(n, hs, ci, co, *, stride=1, seed=0):
    ho = hs // stride
    xh = _rnd(n, hs, hs, ci, seed=seed)
    w = pack.pack_conv2d(torch.randn(co, ci, 3, 3, device=DEV) * (9 * ci) ** -0.5)
    bias = torch.randn(co, device=DEV) * 0.1
    M = n * ho * ho

    def make(out):
        return ops.Gemm(ops.conv_taps([xh]), w, out[:M, :co], M, mode=ops.ROWS_CONV2D,
                        geom=dict(Ho=ho, Wo=ho, Hs=hs, Ws=hs, stride=stride), bias=bias, engine="tc5")
    return make, M, co


def test_conv_in():
    """input_blocks.0.0: 3x3 conv of the 64-channel padded input, K = 576."""
    _check(*_conv(32, 128, 64, 320, seed=8))


def test_conv_stride2():
    _check(*_conv(32, 128, 64, 320, stride=2, seed=9))


def test_upsample_parity_conv():
    """out_up: one parity class of nearest x2 + conv3x3, rows written to the x2 grid."""
    n, hs, ci, co = 32, 64, 64, 320
    xh = _rnd(n, hs, hs, ci, seed=10)
    (py, px), (Wt, shifts) = next(iter(pack.pack_upconv_parity(torch.randn(co, ci, 3, 3, device=DEV) * (9 * ci) ** -0.5).items()))
    M = n * hs * hs

    def make(out):
        return ops.Gemm([ops.SegSpec(xh, dy=sy, dx=sx) for sy, sx in shifts], Wt, out[:4 * M, :co], M, mode=ops.ROWS_CONV2D,
                        geom=dict(Ho=hs, Wo=hs, Hs=hs, Ws=hs, out_up=1, out_py=py, out_px=px), engine="tc5")
    _check(make, 4 * M, co)


def test_ragged_m_and_n():
    _check(*_plain(131 * 128 * 3 + 37, 200, 256, residual=True, seed=11))


def test_odd_tiles_per_cta():
    """A tile count that gives most CTAs an odd number of tiles: the last tile of a CTA falls to its first consumer."""
    sms = _sms()
    m_tiles = 3 * sms + 1          # N = 128 -> one 128-wide n-tile
    make, M, n = _plain(m_tiles * 128 - 5, 128, 320, residual=True, seed=12)
    assert _check(make, M, n) == 128


@pytest.mark.parametrize("M,N", [(128, 64), (1000, 320), (64 * 128, 128)], ids=["one-tile", "few-tiles", "tiles-below-sms"])
def test_fewer_tiles_than_sms(M, N):
    """Below one tile per SM the engine keeps its single-tile kernel."""
    if M == 64 * 128:
        M = (_sms() - 8) * 128
    _check(*_plain(M, N, 320, residual=True, seed=13), want=SINGLE)
