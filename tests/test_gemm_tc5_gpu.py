"""TMA + wgmma implicit-GEMM engine (hi3d_gemm_tc5) against PyTorch fp32 and against the mma.sync engine,
on every geometry it claims (plain rows, 3x3 conv patches with OOB padding, temporal taps, K-concat, skip
segments) and every epilogue."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from hi3d_official_b200 import ops, pack  # noqa: E402
from test_kernels_gpu import DEV, H, close, nhwc, rnd  # noqa: E402

E = "tc5"


@pytest.fixture(params=[-1, 8, 16], ids=["ew-auto", "ew8", "ew16"], autouse=True)
def epilogue_warps(request):
    """Every case runs with the automatic choice and with 8 / 16 MMA + epilogue warps forced (one 128-row tile per CTA, or a
    pair of row tiles sharing each B tile)."""
    from hi3d_official_b200 import _native
    lib = _native.load()
    _native.check(lib.hi3d_gemm_tc5_set_epilogue_warps(request.param), "set_epilogue_warps")
    yield request.param
    _native.check(lib.hi3d_gemm_tc5_set_epilogue_warps(-1), "set_epilogue_warps")


@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (256, 256, 128), (300, 320, 320), (1000, 960, 640), (4096, 1280, 1280),
                                   (257, 2560, 320), (128, 64, 1024)])
def test_tc5_plain(M, N, K):
    a = rnd(M, K).to(H)
    w = rnd(N, K, scale=K ** -0.5).to(H)
    bias = rnd(N, scale=0.1)
    rb = rnd(5, N, scale=0.5).to(H)
    res = rnd(M, N).to(H)
    out = torch.zeros(M, N, dtype=H, device=DEV)
    ref0 = a.float() @ w.float().t()
    ops.Gemm([ops.SegSpec(a)], w, out, M, engine=E)()
    close(out, ref0, name="plain")
    ops.Gemm([ops.SegSpec(a)], w, out, M, bias=bias, rowbias=rb, rb_div=7, rb_mod=5, residual=res, engine=E)()
    idx = (torch.arange(M, device=DEV) // 7) % 5
    close(out, (ref0 + bias + rb.float()[idx]).to(H).float() + res.float(), name="bias+rowbias+res")
    bx = rnd(M, N, seed=5).to(H)
    ops.Gemm([ops.SegSpec(a)], w, out, M, bias=bias, residual=res, blend_x=bx, alpha=0.3, act=ops.ACT_NONE, engine=E)()
    close(out, 0.3 * bx.float() + 0.7 * ((ref0 + bias).to(H).float() + res.float()), name="blend")
    ops.Gemm([ops.SegSpec(a)], w, out, M, bias=bias, act=ops.ACT_SILU, engine=E)()
    close(out, F.silu(ref0 + bias), name="silu")


def test_tc5_geglu_and_kconcat():
    M, C = 513, 320
    a = rnd(M, C).to(H)
    w, b = rnd(8 * C, C, scale=C ** -0.5), rnd(8 * C, scale=0.1)
    wp, bp = pack.pack_geglu(w, b)
    out = torch.zeros(M, 4 * C, dtype=H, device=DEV)
    ops.Gemm([ops.SegSpec(a)], wp, out, M, bias=bp, act=ops.ACT_GEGLU, engine=E)()
    v, g = (a.float() @ w.to(H).float().t() + b).chunk(2, dim=-1)
    close(out, v * F.gelu(g), name="geglu")
    a1, a2 = rnd(M, 128).to(H), rnd(M, 64, seed=2).to(H)
    w2 = rnd(192, 192, scale=192 ** -0.5).to(H)
    o2 = torch.zeros(M, 192, dtype=H, device=DEV)
    ops.Gemm([ops.SegSpec(a1), ops.SegSpec(a2)], w2, o2, M, engine=E)()
    close(o2, torch.cat([a1, a2], 1).float() @ w2.float().t(), name="kconcat")


@pytest.mark.parametrize("n,ci,co,hh,ww", [(4, 64, 128, 16, 16), (2, 128, 320, 32, 32), (8, 64, 64, 8, 8), (32, 64, 64, 4, 4),
                                           (2, 64, 128, 64, 64)])
def test_tc5_conv3x3(n, ci, co, hh, ww):
    x = rnd(n, ci, hh, ww)
    w = rnd(co, ci, 3, 3, scale=(9 * ci) ** -0.5)
    b = rnd(co, scale=0.1)
    emb = rnd(n, co, scale=0.5).to(H)
    xh = nhwc(x)
    ref = F.conv2d(xh.permute(0, 3, 1, 2).float(), w.to(H).float(), b, padding=1) + emb.float()[:, :, None, None]
    M = n * hh * ww
    out = torch.zeros(M, co, dtype=H, device=DEV)
    ops.Gemm(ops.conv_taps([xh]), pack.pack_conv2d(w), out, M, mode=ops.ROWS_CONV2D, geom=dict(Ho=hh, Wo=ww, Hs=hh, Ws=ww),
             bias=b, rowbias=emb, rb_div=hh * ww, rb_mod=n, engine=E)()
    close(out.view(n, hh, ww, co).permute(0, 3, 1, 2), ref, name="conv3x3")


def test_tc5_conv_concat_skip():
    n, c1, c2, co, hh, ww = 4, 64, 128, 64, 16, 16
    x1, x2, hcur = rnd(n, c1, hh, ww), rnd(n, c2, hh, ww, seed=2), rnd(n, co, hh, ww, seed=3)
    w3 = rnd(co, co, 3, 3, scale=(9 * co) ** -0.5)
    ws_ = rnd(co, c1 + c2, 1, 1, scale=(c1 + c2) ** -0.5)
    b3 = rnd(co, scale=0.1)
    x1h, x2h, hh_ = nhwc(x1), nhwc(x2), nhwc(hcur)
    segs = ops.conv_taps([hh_]) + [ops.SegSpec(x1h), ops.SegSpec(x2h)]
    W = pack.cat_k(pack.pack_conv2d(w3), pack.pack_conv2d(ws_))
    M = n * hh * ww
    out = torch.zeros(M, co, dtype=H, device=DEV)
    ops.Gemm(segs, W, out, M, mode=ops.ROWS_CONV2D, geom=dict(Ho=hh, Wo=ww, Hs=hh, Ws=ww), bias=b3, engine=E)()
    xr = torch.cat([x1h, x2h], -1).permute(0, 3, 1, 2).float()
    ref = F.conv2d(hh_.permute(0, 3, 1, 2).float(), w3.to(H).float(), b3, padding=1) + F.conv2d(xr, ws_.to(H).float())
    close(out.view(n, hh, ww, co).permute(0, 3, 1, 2), ref, name="conv+skip")
    w1 = rnd(co, c1 + c2, 3, 3, scale=(9 * (c1 + c2)) ** -0.5)
    ops.Gemm(ops.conv_taps([x1h, x2h]), pack.pack_conv2d(w1), out, M, mode=ops.ROWS_CONV2D,
             geom=dict(Ho=hh, Wo=ww, Hs=hh, Ws=ww), bias=b3, engine=E)()
    close(out.view(n, hh, ww, co).permute(0, 3, 1, 2), F.conv2d(xr, w1.to(H).float(), b3, padding=1), name="conv concat")


@pytest.mark.parametrize("T,hw", [(16, 256), (16, 64), (16, 16), (8, 128)])
def test_tc5_temporal_conv(T, hw):
    b, c, co = 2, 64, 128
    x = rnd(b, c, T, hw, 1)
    w = rnd(co, c, 3, 1, 1, scale=(3 * c) ** -0.5)
    bias = rnd(co, scale=0.1)
    xh = x.permute(0, 2, 3, 4, 1).reshape(b * T * hw, c).contiguous().to(H)
    M = b * T * hw
    res = rnd(M, co, seed=7).to(H)
    out = torch.zeros(M, co, dtype=H, device=DEV)
    ops.Gemm(ops.temporal_taps(xh), pack.pack_conv3d_t(w), out, M, mode=ops.ROWS_TEMPORAL, geom=dict(Ho=hw, Wo=1, T=T),
             bias=bias, residual=res, blend_x=res, alpha=0.4, engine=E)()
    xr = xh.view(b, T, hw, 1, c).permute(0, 4, 1, 2, 3).float()
    conv = F.conv3d(xr, w.to(H).float(), bias, padding=(1, 0, 0)).permute(0, 2, 3, 4, 1).reshape(M, co)
    ref = 0.4 * res.float() + 0.6 * (conv.to(H).float() + res.float())
    close(out, ref, name="temporal conv + blend")


def test_tc5_unsupported_geometry_forwards_to_mma_engine():
    n, ci, co, hs = 2, 64, 64, 12
    x, w = rnd(n, ci, hs, hs), rnd(co, ci, 3, 3, scale=(9 * ci) ** -0.5)
    xh = nhwc(x)
    ref = F.conv2d(xh.permute(0, 3, 1, 2).float(), w.to(H).float(), stride=2, padding=1)
    ho = ref.shape[2]
    out = torch.zeros(n * ho * ho, co, dtype=H, device=DEV)
    ops.Gemm(ops.conv_taps([xh]), pack.pack_conv2d(w), out, n * ho * ho, mode=ops.ROWS_CONV2D,
             geom=dict(Ho=ho, Wo=ho, Hs=hs, Ws=hs, stride=2), engine=E)()
    close(out.view(n, ho, ho, co).permute(0, 3, 1, 2), ref, name="stride-2 via fallback")


@pytest.mark.parametrize("engine", ["mma", "tc5"])
@pytest.mark.parametrize("n,ci,co,hs", [(2, 64, 128, 16), (4, 128, 64, 32), (1, 64, 64, 64)])
def test_stride2_conv_both_paddings(engine, n, ci, co, hs):
    """UNet Downsample (pad 1, stride 2) and VAE Downsample (pad (0,1,0,1), stride 2): TMA element strides on tc5."""
    x, w = rnd(n, ci, hs, hs), rnd(co, ci, 3, 3, scale=(9 * ci) ** -0.5)
    b = rnd(co, scale=0.1)
    xh = nhwc(x)
    xr, wr = xh.permute(0, 3, 1, 2).float(), w.to(H).float()
    for asym in (False, True):
        ref = F.conv2d(F.pad(xr, (0, 1, 0, 1)), wr, b, stride=2) if asym else F.conv2d(xr, wr, b, stride=2, padding=1)
        ho = ref.shape[2]
        out = torch.zeros(n * ho * ho, co, dtype=H, device=DEV)
        ops.Gemm(ops.conv_taps([xh], pad_lo=0 if asym else 1), pack.pack_conv2d(w), out, n * ho * ho, mode=ops.ROWS_CONV2D,
                 geom=dict(Ho=ho, Wo=ho, Hs=hs, Ws=hs, stride=2), bias=b, engine=engine)()
        close(out.view(n, ho, ho, co).permute(0, 3, 1, 2), ref, name=f"stride2 asym={asym} {engine}")


@pytest.mark.parametrize("engine", ["mma", "tc5"])
@pytest.mark.parametrize("n,ci,co,hs", [(2, 64, 128, 16), (4, 128, 64, 8), (1, 64, 64, 32)])
def test_upsample_conv_as_parity_convs(engine, n, ci, co, hs):
    """nearest x2 + conv3x3 == four parity-class 2x2 convs with pre-summed taps, written through out_up."""
    x, w = rnd(n, ci, hs, hs), rnd(co, ci, 3, 3, scale=(9 * ci) ** -0.5)
    b = rnd(co, scale=0.1)
    xh = nhwc(x)
    ref = F.conv2d(F.interpolate(xh.permute(0, 3, 1, 2).float(), scale_factor=2, mode="nearest"), w.to(H).float(), b, padding=1)
    out = torch.zeros(n * 4 * hs * hs, co, dtype=H, device=DEV)
    for (py, px), (Wt, shifts) in pack.pack_upconv_parity(w).items():
        ops.Gemm([ops.SegSpec(xh, dy=sy, dx=sx) for sy, sx in shifts], Wt, out, n * hs * hs, mode=ops.ROWS_CONV2D,
                 geom=dict(Ho=hs, Wo=hs, Hs=hs, Ws=hs, out_up=1, out_py=py, out_px=px), bias=b, engine=engine)()
    # pre-summed fp16 taps add one more fp16 rounding of the weights: slightly wider tolerance
    close(out.view(n, 2 * hs, 2 * hs, co).permute(0, 3, 1, 2), ref, rtol=4e-3, name=f"upconv parity {engine}")


# ---- GroupNorm statistics from the epilogue (hi3d_gemm_params::gn_stats) and the one-launch apply that consumes them ------
def _unit_sums(out2d, n_img, rows, unit):
    """(sum, sumsq) per image and per `unit` channels of the STORED fp16 tensor."""
    o = out2d.float().view(n_img, rows, -1, unit)
    return torch.stack([o.sum((1, 3)), (o * o).sum((1, 3))], -1)            # [n_img, units, 2]


def _close_stats(got, ref, name):
    err = (got - ref).abs()
    tol = 2e-3 * ref.abs() + 2e-3 * ref.abs().mean()
    assert bool((err <= tol).all()), f"{name}: max err {float(err.max()):.3e} (ref mean {float(ref.abs().mean()):.3e})"


@pytest.mark.parametrize("engine", ["tc5", "mma"])
@pytest.mark.parametrize("n,ci,co,hh,unit", [(4, 64, 320, 32, 10), (8, 64, 64, 8, 2), (32, 64, 64, 4, 2), (2, 128, 640, 16, 10)])
def test_gemm_epilogue_gn_stats_conv(engine, n, ci, co, hh, unit):
    x, w, b = rnd(n, ci, hh, hh), rnd(co, ci, 3, 3, scale=(9 * ci) ** -0.5), rnd(co, scale=0.1)
    res = rnd(n * hh * hh, co, seed=9).to(H)
    xh = nhwc(x)
    M = n * hh * hh
    out = torch.zeros(M, co, dtype=H, device=DEV)
    stats = torch.zeros(n, co // unit, 2, device=DEV)
    ops.Gemm(ops.conv_taps([xh]), pack.pack_conv2d(w), out, M, mode=ops.ROWS_CONV2D, geom=dict(Ho=hh, Wo=hh, Hs=hh, Ws=hh),
             bias=b, residual=res, engine=engine, gn_stats=stats.view(-1), gn_unit=unit, gn_rows=hh * hh)()
    ref = F.conv2d(xh.permute(0, 3, 1, 2).float(), w.to(H).float(), b, padding=1)
    close(out.view(n, hh, hh, co).permute(0, 3, 1, 2), ref.to(H).float() + res.view(n, hh, hh, co).permute(0, 3, 1, 2).float(),
          name="conv + residual (with stats)")
    _close_stats(stats, _unit_sums(out, n, hh * hh, unit), f"epilogue stats conv {engine}")
    # accumulate semantics: a second launch adds
    ops.Gemm(ops.conv_taps([xh]), pack.pack_conv2d(w), out, M, mode=ops.ROWS_CONV2D, geom=dict(Ho=hh, Wo=hh, Hs=hh, Ws=hh),
             bias=b, residual=res, engine=engine, gn_stats=stats.view(-1), gn_unit=unit, gn_rows=hh * hh)()
    _close_stats(stats, 2 * _unit_sums(out, n, hh * hh, unit), f"epilogue stats accumulate {engine}")


@pytest.mark.parametrize("pair", [-1, 1])
def test_gemm_epilogue_gn_stats_temporal_plain_upconv(pair):
    lib = __import__("hi3d_official_b200._native", fromlist=["x"]).load()
    lib.hi3d_gemm_tc5_set_pair_mode(pair)
    try:
        # temporal taps, T = 8, 64 px frames (two frames per tile) and 256 px frames
        for hw in (64, 256):
            b_, c, co, T, unit = 2, 64, 320, 8, 10
            M = b_ * T * hw
            xh = rnd(M, c, seed=3).to(H)
            w = rnd(co, c, 3, 1, 1, scale=(3 * c) ** -0.5)
            out = torch.zeros(M, co, dtype=H, device=DEV)
            stats = torch.zeros(b_ * T, co // unit, 2, device=DEV)
            ops.Gemm(ops.temporal_taps(xh), pack.pack_conv3d_t(w), out, M, mode=ops.ROWS_TEMPORAL, geom=dict(Ho=hw, Wo=1, T=T),
                     engine="tc5", gn_stats=stats.view(-1), gn_unit=unit, gn_rows=hw)()
            _close_stats(stats, _unit_sums(out, b_ * T, hw, unit), f"epilogue stats temporal hw={hw}")
        # plain rows (proj_out-like), ragged last tile, images of 100 rows
        M, K, N, rows, unit = 700, 320, 320, 100, 10
        a, w = rnd(M, K).to(H), rnd(N, K, scale=K ** -0.5).to(H)
        out = torch.zeros(M, N, dtype=H, device=DEV)
        stats = torch.zeros(M // rows, N // unit, 2, device=DEV)
        ops.Gemm([ops.SegSpec(a)], w, out, M, engine="tc5", gn_stats=stats.view(-1), gn_unit=unit, gn_rows=rows)()
        _close_stats(stats, _unit_sums(out, M // rows, rows, unit), "epilogue stats plain")
        # nearest x2 + conv as four parity launches accumulating into one table
        n, ci, co, hs, unit = 2, 64, 64, 16, 2
        x, w = rnd(n, ci, hs, hs), rnd(co, ci, 3, 3, scale=(9 * ci) ** -0.5)
        xh = nhwc(x)
        out = torch.zeros(n * 4 * hs * hs, co, dtype=H, device=DEV)
        stats = torch.zeros(n, co // unit, 2, device=DEV)
        for (py, px), (Wt, shifts) in pack.pack_upconv_parity(w).items():
            ops.Gemm([ops.SegSpec(xh, dy=sy, dx=sx) for sy, sx in shifts], Wt, out, n * hs * hs, mode=ops.ROWS_CONV2D,
                     geom=dict(Ho=hs, Wo=hs, Hs=hs, Ws=hs, out_up=1, out_py=py, out_px=px), engine="tc5",
                     gn_stats=stats.view(-1), gn_unit=unit, gn_rows=hs * hs)()
        _close_stats(stats, _unit_sums(out, n, 4 * hs * hs, unit), "epilogue stats upconv")
    finally:
        lib.hi3d_gemm_tc5_set_pair_mode(-1)


@pytest.mark.parametrize("silu,eps", [(True, 1e-5), (False, 1e-6)])
def test_groupnorm_apply_from_unit_stats(silu, eps):
    """hi3d_groupnorm_apply_stats: spatial (per image), temporal (T images per sample) and the two-source concat whose groups
    straddle the source boundary (C1 = 1280 / 128, C2 = 640 / 64 -> 60 / 6 channels per group), against F.group_norm."""
    for (n, rows, c1, c2, unit, ips) in ((4, 256, 320, 0, 10, 1), (4, 64, 128, 64, 2, 1), (8, 64, 64, 0, 2, 4), (2, 128, 1280, 640, 10, 1)):
        C = c1 + c2
        x1 = rnd(n * rows, c1, seed=1).to(H) * 1.5 + 0.3
        x2 = (rnd(n * rows, c2, seed=2).to(H) * 0.7 - 0.2) if c2 else None
        s1 = torch.zeros(n, c1 // unit, 2, device=DEV)
        ops.groupnorm_unit_stats(x1, n, rows, unit, s1.view(-1))
        _close_stats(s1, _unit_sums(x1, n, rows, unit), "unit stats")
        s2 = None
        if c2:
            s2 = torch.zeros(n, c2 // unit, 2, device=DEV)
            ops.groupnorm_unit_stats(x2, n, rows, unit, s2.view(-1))
        gam, bet = 1 + 0.1 * rnd(C, seed=3), 0.1 * rnd(C, seed=4)
        y = torch.zeros(n * rows, C, dtype=H, device=DEV)
        ns = n // ips
        ops.groupnorm_apply_stats(x1, s1.view(-1), x2, None if s2 is None else s2.view(-1), unit, ns, rows * ips, ips, rows * ips,
                                  gam, bet, eps, silu, y)
        xc = x1 if x2 is None else torch.cat([x1, x2], 1)
        ref = F.group_norm(xc.view(ns, rows * ips, C).permute(0, 2, 1).float(), 32, gam, bet, eps)
        if silu:
            ref = F.silu(ref)
        close(y.view(ns, rows * ips, C).permute(0, 2, 1), ref, name=f"apply from stats n={n} C={c1}+{c2} ips={ips}")
        if ips > 1 or c2 == 0:
            sums = torch.zeros(ns, 32, 2, device=DEV)
            ops.groupnorm_group_sums(s1.view(-1), c1, None, 0, unit, ns, ips, sums)
            g = xc.float().view(ns, rows * ips, 32, C // 32)
            _close_stats(sums, torch.stack([g.sum((1, 3)), (g * g).sum((1, 3))], -1), "group sums")
