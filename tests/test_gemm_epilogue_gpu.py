"""The ping-pong schedule's epilogue: TMA stores of the staged tile (plain, conv and temporal output maps, column slices of wider
buffers, the parity-class upsample rows) and the chunk pass that adds residual and blend in shared memory.

Each case writes into a column slice of a sentinel-filled buffer that is wider and longer than the result, checks that the
engine picked the ping-pong kernel, that its output equals the single-tile kernel's bit for bit (border included), that
nothing outside the slice changed, and that the result is close to an fp32 torch computation (the tolerance of
test_gemm_tc5_gpu.py)."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from hi3d_official_b200 import _native, ops, pack  # noqa: E402

DEV, H = "cuda", torch.float16
PINGPONG, SINGLE = 3, 1
SENTINEL = -5.0
COL0, EXTRA = 24, 40          # the result starts at column COL0 of a buffer EXTRA columns wider than it


def _rnd(*shape, scale=1.0, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(*shape, generator=g, device=DEV) * scale).to(H)


def _close(got, ref):
    err = (got.float() - ref).abs()
    tol = 2e-3 * ref.abs() + 2e-3 * ref.abs().mean()
    assert bool((err <= tol).all()), f"max err {float(err.max()):.3e} (ref mean {float(ref.abs().mean()):.3e})"


def _run(make, rows, cols, ref, inplace=None, col0=COL0, extra=EXTRA):
    """make(out_slice) -> ops.Gemm writing out_slice = buffer[:rows, col0:col0 + cols].  inplace(out_slice) fills the slice
    with the residual before each run (an in-place residual add)."""
    lib = _native.load()
    outs = []
    for mode in (-1, 0):
        _native.check(lib.hi3d_gemm_tc5_set_pair_mode(mode), "set_pair_mode")
        try:
            buf = torch.full((rows + 64, col0 + cols + extra), SENTINEL, dtype=H, device=DEV)
            if inplace is not None:
                inplace(buf[:rows, col0:col0 + cols])
            g = make(buf[:rows, col0:col0 + cols])
            r = lib.hi3d_gemm_tc5_schedule(ctypes.byref(g.p))
            assert r // 1000 == (PINGPONG if mode == -1 else SINGLE), (mode, r)
            g()
            torch.cuda.synchronize()
            outs.append(buf)
        finally:
            _native.check(lib.hi3d_gemm_tc5_set_pair_mode(-1), "set_pair_mode")
    a, b = outs
    assert torch.equal(a, b), f"max |diff| {(a.float() - b.float()).abs().max().item()}"
    assert (a[rows:] == SENTINEL).all() and (a[:, :col0] == SENTINEL).all() and (a[:, col0 + cols:] == SENTINEL).all()
    _close(a[:rows, col0:col0 + cols], ref)


M_RAGGED = 300 * 128 + 77     # ragged M, more tiles than SMs


@pytest.mark.parametrize("N", [320, 200], ids=["N320", "N200"])
def test_plain_slice(N):
    K = 320
    a, w = _rnd(M_RAGGED, K, seed=1), _rnd(N, K, scale=K ** -0.5, seed=2)
    bias = torch.randn(N, device=DEV) * 0.1
    ref = a.float() @ w.float().t() + bias
    _run(lambda o: ops.Gemm([ops.SegSpec(a)], w, o, M_RAGGED, bias=bias, engine="tc5"), M_RAGGED, N, ref)


@pytest.mark.parametrize("N", [2 * 320, 2 * 200, 2 * 96], ids=["Nout320", "Nout200", "Nout96"])
def test_geglu_slice(N):
    K = 320
    a = _rnd(M_RAGGED, K, seed=3)
    w0, b0 = torch.randn(N, K, device=DEV) * K ** -0.5, torch.randn(N, device=DEV) * 0.1
    w, bias = pack.pack_geglu(w0, b0)
    h = a.float() @ w0.to(H).float().t() + b0
    v, gate = h[:, : N // 2], h[:, N // 2:]
    ref = v * F.gelu(gate)
    _run(lambda o: ops.Gemm([ops.SegSpec(a)], w, o, M_RAGGED, bias=bias, act=ops.ACT_GEGLU, engine="tc5"), M_RAGGED, N // 2, ref)


def test_rowbias_and_residual():
    M, N, K = M_RAGGED, 320, 320
    a, w = _rnd(M, K, seed=4), _rnd(N, K, scale=K ** -0.5, seed=5)
    bias = torch.randn(N, device=DEV) * 0.1
    rb = _rnd(3, N, scale=0.5, seed=6)
    res = _rnd(M, N, seed=7)
    rows = (torch.arange(M, device=DEV) // 2000) % 3
    h = (a.float() @ w.float().t() + bias + rb.float()[rows]).half().float()
    ref = h + res.float()
    _run(lambda o: ops.Gemm([ops.SegSpec(a)], w, o, M, bias=bias, rowbias=rb, rb_div=2000, rb_mod=3, residual=res, engine="tc5"),
         M, N, ref)


def test_inplace_residual():
    """out is the residual (a residual must be contiguous, so the whole width of the buffer)."""
    M, N, K = M_RAGGED, 320, 640
    a, w = _rnd(M, K, seed=8), _rnd(N, K, scale=K ** -0.5, seed=9)
    bias = torch.randn(N, device=DEV) * 0.1
    res = _rnd(M, N, seed=10)
    ref = (a.float() @ w.float().t() + bias).half().float() + res.float()

    def fill(o):
        o.copy_(res)

    _run(lambda o: ops.Gemm([ops.SegSpec(a)], w, o, M, bias=bias, residual=o, engine="tc5"), M, N, ref, inplace=fill, col0=0, extra=0)


@pytest.mark.parametrize("same", [True, False], ids=["blend_is_residual", "blend_separate"])
def test_blend(same):
    M, N, K, alpha = M_RAGGED, 320, 320, 0.3
    a, w = _rnd(M, K, seed=11), _rnd(N, K, scale=K ** -0.5, seed=12)
    bias = torch.randn(N, device=DEV) * 0.1
    res = _rnd(M, N, seed=13)
    bx = res if same else _rnd(M, N, seed=14)
    h = ((a.float() @ w.float().t() + bias).half().float() + res.float()).half().float()
    ref = alpha * bx.float() + (1 - alpha) * h
    _run(lambda o: ops.Gemm([ops.SegSpec(a)], w, o, M, bias=bias, residual=res, blend_x=bx, alpha=alpha, engine="tc5"), M, N, ref)


def test_conv_slice_residual():
    n, hs, ci, co = 16, 64, 64, 200
    xh = _rnd(n, hs, hs, ci, seed=15)
    wt = torch.randn(co, ci, 3, 3, device=DEV) * (9 * ci) ** -0.5
    bias = torch.randn(co, device=DEV) * 0.1
    M = n * hs * hs
    res = _rnd(M, co, seed=16)
    ref = F.conv2d(xh.permute(0, 3, 1, 2).float(), wt.to(H).float(), bias, padding=1).permute(0, 2, 3, 1).reshape(M, co)
    ref = ref.half().float() + res.float()
    _run(lambda o: ops.Gemm(ops.conv_taps([xh]), pack.pack_conv2d(wt), o, M, mode=ops.ROWS_CONV2D,
                            geom=dict(Ho=hs, Wo=hs, Hs=hs, Ws=hs), bias=bias, residual=res, engine="tc5"), M, co, ref)


def test_upsample_parity_slice():
    n, hs, ci, co = 16, 32, 64, 200
    xh = _rnd(n, hs, hs, ci, seed=17)
    wt = torch.randn(co, ci, 3, 3, device=DEV) * (9 * ci) ** -0.5
    (py, px), (Wt, shifts) = next(iter(pack.pack_upconv_parity(wt).items()))
    M = n * hs * hs
    up = F.interpolate(xh.permute(0, 3, 1, 2).float(), scale_factor=2, mode="nearest")
    full = F.conv2d(up, wt.to(H).float(), padding=1).permute(0, 2, 3, 1)            # n, 2hs, 2hs, co
    lib = _native.load()
    outs = []
    for mode in (-1, 0):
        _native.check(lib.hi3d_gemm_tc5_set_pair_mode(mode), "set_pair_mode")
        try:
            buf = torch.full((4 * M + 64, COL0 + co + EXTRA), SENTINEL, dtype=H, device=DEV)
            g = ops.Gemm([ops.SegSpec(xh, dy=sy, dx=sx) for sy, sx in shifts], Wt, buf[:4 * M, COL0:COL0 + co], M,
                         mode=ops.ROWS_CONV2D, geom=dict(Ho=hs, Wo=hs, Hs=hs, Ws=hs, out_up=1, out_py=py, out_px=px), engine="tc5")
            assert lib.hi3d_gemm_tc5_schedule(ctypes.byref(g.p)) // 1000 == (PINGPONG if mode == -1 else SINGLE)
            g()
            torch.cuda.synchronize()
            outs.append(buf)
        finally:
            _native.check(lib.hi3d_gemm_tc5_set_pair_mode(-1), "set_pair_mode")
    a, b = outs
    assert torch.equal(a, b)
    grid = a[:4 * M].view(n, 2 * hs, 2 * hs, -1)
    cls = grid[:, py::2, px::2, COL0:COL0 + co]
    _close(cls, full[:, py::2, px::2])
    # every row outside the parity class, and every column outside the slice, keeps the sentinel
    mask = torch.ones(n, 2 * hs, 2 * hs, dtype=torch.bool, device=DEV)
    mask[:, py::2, px::2] = False
    assert (grid[mask] == SENTINEL).all()
    assert (a[:, :COL0] == SENTINEL).all() and (a[:, COL0 + co:] == SENTINEL).all() and (a[4 * M:] == SENTINEL).all()


def test_temporal_slice_blend():
    b, T, hw, c, co = 2, 16, 32 * 32, 320, 200
    M = b * T * hw
    xh = _rnd(M, c, seed=18)
    wt = torch.randn(co, c, 3, 1, 1, device=DEV) * (3 * c) ** -0.5
    bias = torch.randn(co, device=DEV) * 0.1
    res, bx, alpha = _rnd(M, co, seed=19), _rnd(M, co, seed=20), 0.4
    x5 = xh.view(b, T, hw, c).permute(0, 3, 1, 2).unsqueeze(-1).float()           # b, c, T, hw, 1
    h = F.conv3d(x5, wt.to(H).float(), bias, padding=(1, 0, 0)).squeeze(-1).permute(0, 2, 3, 1).reshape(M, co)
    h = (h.half().float() + res.float()).half().float()
    ref = alpha * bx.float() + (1 - alpha) * h
    _run(lambda o: ops.Gemm(ops.temporal_taps(xh), pack.pack_conv3d_t(wt), o, M, mode=ops.ROWS_TEMPORAL,
                            geom=dict(Ho=hw, Wo=1, T=T), bias=bias, residual=res, blend_x=bx, alpha=alpha, engine="tc5"),
         M, co, ref)
