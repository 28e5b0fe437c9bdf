"""FP8 sampling (VideoUNet.set_precision("fp8")): the e4m3 producers against the fp16 kernels bit for bit, the e4m3 wgmma GEMM
against an fp32 product of its dequantised operands, every GEMM of the fp8 UNet plan against its state-dict layer on the plan's own
inputs, the whole plan against fp32 oracles, and the reproducibility and entry points of the mode.

GEMM tolerance (_check), per output: 2e-3 |ref| + 2^-10 sum_k |a_k w_k| + 1e-3 mean |ref|.  The first and last terms are the fp16
rounding of the output and of the fp16 epilogue steps.  The middle one is accumulation order: Hopper's e4m3 MMA adds products into
an accumulator of reduced precision before the fp32 accumulate, so its error scales with sum |a w|, not with fp32 rounding.  An
e4m3 output must lie within one e4m3 step of e4m3(reference) wherever that accumulation term is below 1/16 of |ref|; smaller
results are dominated by it either way."""
import os
import re
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from hi3d_official_b200 import _native, ops, pack, spec  # noqa: E402
from oracle import hi3d_oracle as O  # noqa: E402

DEV = "cuda"
E4M3 = torch.float8_e4m3fn
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def e4m3_ref(x16: torch.Tensor) -> torch.Tensor:
    """The rule every e4m3 store follows: the fp16 value, saturated to +-448, rounded to nearest even."""
    return x16.float().clamp(-448, 448).to(E4M3)


def assert_bits(y8: torch.Tensor, y16: torch.Tensor, what: str):
    ref = e4m3_ref(y16)
    same = y8.view(torch.uint8) == ref.view(torch.uint8)
    assert bool(same.all()), f"{what}: {int((~same).sum())} of {same.numel()} e4m3 values differ from e4m3(fp16 output)"


# ---- producers ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C1,C2,unit,ips", [(320, 0, 10, 1), (320, 320, 10, 1), (640, 0, 20, 4), (320, 640, 10, 4),
                                           (64, 0, 2, 1), (128, 64, 2, 8)])
@pytest.mark.parametrize("silu", [True, False])
def test_groupnorm_apply_stats_fp8_bit_exact(C1, C2, unit, ips, silu):
    g = torch.Generator().manual_seed(C1 + C2 + ips)
    n_samples, rows_img = 2, 96
    rows = ips * rows_img
    xs = [(torch.randn(n_samples * rows, c, generator=g) * 3 + 1).half().to(DEV) for c in (C1, C2) if c]
    C = C1 + C2
    gamma = (torch.randn(C, generator=g) * 150).to(DEV)         # some outputs beyond +-448: the saturation is tested too
    beta = torch.randn(C, generator=g).to(DEV)
    stats = []
    for x in xs:
        st = torch.zeros(n_samples * ips * (x.shape[1] // unit) * 2, device=DEV)
        ops.groupnorm_unit_stats(x, n_samples * ips, rows_img, unit, st)
        stats.append(st)
    x2, st2 = (xs[1], stats[1]) if C2 else (None, None)
    y16 = torch.empty(n_samples * rows, C, dtype=torch.float16, device=DEV)
    y8 = torch.empty(n_samples * rows, C, dtype=E4M3, device=DEV)
    for y in (y16, y8):
        ops.groupnorm_apply_stats(xs[0], stats[0], x2, st2, unit, n_samples, rows, ips, rows, gamma, beta, 1e-5, silu, y)
    torch.cuda.synchronize()
    assert float(y16.float().abs().max()) > 448
    assert_bits(y8, y16, f"groupnorm C={C1}+{C2} ips={ips}")


@pytest.mark.parametrize("C", [320, 640, 1280, 64, 96, 2560])
@pytest.mark.parametrize("with_add", [False, True])
def test_layernorm_fp8_bit_exact(C, with_add):
    g = torch.Generator().manual_seed(C)
    M, T, HW = 8 * 37, 8, 37
    x = (torch.randn(M, C, generator=g) * 2 + 0.5).half().to(DEV)
    gamma, beta = (torch.randn(C, generator=g) * 60).to(DEV), torch.randn(C, generator=g).to(DEV)
    add = torch.randn(T, C, generator=g).half().to(DEV) if with_add else None
    y16 = torch.empty(M, C, dtype=torch.float16, device=DEV)
    y8 = torch.empty(M, C, dtype=E4M3, device=DEV)
    for y in (y16, y8):
        ops.layernorm(x, gamma, beta, y, M, addvec=add, add_div=HW, add_mod=T)
    torch.cuda.synchronize()
    assert_bits(y8, y16, f"layernorm C={C} add={with_add}")


# ---- the e4m3 GEMM --------------------------------------------------------------------------------------------------------------
def _a8(rows, C, g):
    return e4m3_ref(torch.randn(rows, C, generator=g).half()).to(DEV)


def _w8(N, K, g):
    w = (torch.randn(N, K, generator=g) / K ** 0.5).half()
    w[3] = 0                                                  # an all-zero row: scale 1
    W8, sc = pack.pack_e4m3(w)
    return W8.to(DEV), sc.to(DEV), W8.float().to(DEV) * sc.to(DEV)[:, None]


def _check(out, ref, absprod, what, fp8_out=False):
    """ref: the fp32 result; absprod: sum_k |a_k w_k| per output, the scale of the accumulation error.  Hopper's e4m3 MMA adds
    products into an accumulator of reduced precision before the fp32 accumulate, so the accumulation-order term is
    2^-10 of that sum rather than fp32 rounding.  Returns the worst error / tolerance (fp16 output) or the most e4m3 steps
    from e4m3(reference) (e4m3 output): 1 at most."""
    torch.cuda.synchronize()
    if fp8_out:
        # at most one e4m3 step from e4m3(reference): compare the codes as signed magnitudes
        def ordered(t):
            c = t.view(torch.uint8).int()
            return torch.where(c >= 128, -(c - 128), c)
        d = (ordered(out) - ordered(e4m3_ref(ref.half()))).abs()
        # where the accumulation error is below 1/16 of |result|, it is below one e4m3 step (results smaller than that are
        # dominated by the accumulation error, and the fp16-output cases bound it)
        d = d[ref.abs() > 2 ** -6 * absprod]
        steps = int(d.max()) if d.numel() else 0
        assert steps <= 1, f"{what}: e4m3 output {steps} steps from e4m3(reference)"
        return float(steps)
    err = (out.float() - ref).abs()
    tol = 2e-3 * ref.abs() + 2 ** -10 * absprod + 1e-3 * float(ref.abs().mean())   # fp16 rounding of output and epilogue
    bad = err > tol
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} outside, max err {float(err.max()):.3e}"
    return float((err / tol.clamp_min(1e-30)).max())


def _epilogue(acc, bias, rowbias, rb_div, act, residual, blend_x, alpha):
    v = acc + bias
    if rowbias is not None:
        v = v + rowbias.float()[torch.arange(v.shape[0], device=DEV) // rb_div % rowbias.shape[0]]
    if act == ops.ACT_GEGLU:
        v = v[:, 0::2] * F.gelu(v[:, 1::2])
    if residual is not None:
        v = v + residual.float()
    if blend_x is not None:
        v = alpha * blend_x.float() + (1 - alpha) * v
    return v


# ---- which tile the engine runs -------------------------------------------------------------------------------------------------
def sm_count() -> int:
    return torch.cuda.get_device_properties(0).multi_processor_count


def tc5_m_tiles(mode: int, M: int, Ho: int = 1, Wo: int = 1, T: int = 1) -> int:
    """Row tiles of a GEMM on the wgmma engine (tc5_geometry in gemm_tc5.cu): 128 rows, a (tn x th x tw) conv patch or a
    (tf frames x ts pixels) temporal patch per tile."""
    if mode == ops.ROWS_PLAIN:
        return -(-M // 128)
    if mode == ops.ROWS_CONV2D:
        tw = th = 1
        while tw * 2 <= 16 and Wo % (tw * 2) == 0:
            tw *= 2
        while tw * th * 2 <= 128 and Ho % (th * 2) == 0:
            th *= 2
        return (Wo // tw) * (Ho // th) * (M // (Ho * Wo)) // (128 // (tw * th))
    HW, ts = Ho * Wo, 1
    while ts * 2 <= 128 and HW % (ts * 2) == 0:
        ts *= 2
    return (HW // ts) * (T // (128 // ts)) * (M // (HW * T))


def tc5_tile(K: int, N: int, m_tiles: int, sms: int, pair: int = -1):
    """(row tiles per CTA, tile width) that the engine picks (tc5_gemm in gemm_tc5.cu): tile pairs for K >= 1920 with at least
    four 128 x 128 tiles per SM, unless the pair-mode hook forces one or the other; then the width in {256, 192, 128, 64}
    ({128, 64} for pairs) with the least waves x (width + 48), ties to the wider tile."""
    nt = 2 if K >= 1920 and m_tiles * -(-N // 128) >= 4 * sms else 1
    if pair >= 0:
        nt = pair + 1
    units, best = -(-m_tiles // nt), None
    for bn in (128, 64) if nt == 2 else (256, 192, 128, 64):
        cost = -(-units * -(-N // bn) // sms) * (bn + 48)
        if best is None or cost < best[0]:
            best = (cost, bn)
    return nt, best[1]


def gemm_tile(gm: "ops.Gemm", sms: int):
    """tc5_tile of a baked GEMM (automatic pair mode)."""
    p = gm.p
    return tc5_tile(p.K, p.N, tc5_m_tiles(p.mode, p.M, p.Ho, p.Wo, p.T), sms)


# Tile targets (row tiles per CTA, tile width, N): every tile the engine has, and ragged last N tiles (320 = 192 + 128 and
# 128 + 128 + 64).  Single tiles run with the automatic choice (K < 1920 never pairs), pairs with the hook forcing them.
TILE_TARGETS = [(1, 256, 256), (1, 192, 192), (1, 128, 128), (1, 64, 64), (1, 192, 320), (2, 128, 128), (2, 64, 64),
                (2, 128, 320)]


def tile_geometry(mode: int, n: int):
    """(M, geom) of the n-th shape of a family per row mode: plain M = 128 n - 5 (a ragged last row tile); 2 n images of
    8 x 8 (two-image patches, n tiles); n clips of 16 frames of 64 pixels (two-frame patches, 8 n tiles)."""
    if mode == ops.ROWS_PLAIN:
        return 128 * n - 5, {}
    if mode == ops.ROWS_CONV2D:
        return 128 * n, dict(Ho=8, Wo=8, Hs=8, Ws=8)
    return 1024 * n, dict(Ho=64, Wo=1, T=16)


def tile_shape(mode: int, nt: int, bn: int, N: int, K: int, sms: int):
    """The smallest shape of the family that fills at least one wave of CTAs on `sms` SMs and for which the engine's cost
    model picks (nt, bn): (M, geom, pair mode to run it with)."""
    pair = 1 if nt == 2 else -1
    for n in range(1, 64 * sms):
        M, geom = tile_geometry(mode, n)
        mt = tc5_m_tiles(mode, M, geom.get("Ho", 1), geom.get("Wo", 1), geom.get("T", 1))
        if -(-mt // nt) * -(-N // bn) >= sms and tc5_tile(K, N, mt, sms, pair) == (nt, bn):
            return M, geom, pair
    raise AssertionError(f"no shape of mode {mode} selects {nt} x {bn} for N = {N} on {sms} SMs")


def tc5_launches(fn):
    """(row tiles per CTA, tile width, operand type) of each wgmma GEMM kernel fn() launches, read from the kernel names that
    torch.profiler records (gemm_tc5_kernel<BN, NT, Op>, demangled or not); None when the profiler delivers no kernel record
    (CUPTI drops them in some sessions of a long process)."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == DeviceType.CUDA]
    if not names:
        return None
    out = []
    for n in names:
        m = re.search(r"gemm_tc5_kernel<\s*(\d+)\s*,\s*(\d+)\s*,\s*([\w:]+)\s*>", n)
        if m:
            out.append((int(m[2]), int(m[1]), m[3]))
            continue
        m = re.search(r"gemm_tc5_kernelILi(\d+)ELi(\d+)E\d+(\w+?)EEv", n)
        if m:
            out.append((int(m[2]), int(m[1]), m[3]))
    assert out, f"no gemm_tc5_kernel among the recorded events {sorted(set(names))[:6]}"
    return out


def assert_launched(launched, want, what=""):
    """The launched kernels (tc5_launches) are [want]; without profiler events the launch is not cross-checked (printed)."""
    if launched is None:
        print(f"[tc5 launch] {what}: the profiler delivered no kernel record, launch of {want} not cross-checked")
        return
    assert launched == [want], (what, launched, want)


def run_pair_mode(pair: int, fn):
    """fn() with the engine's pair-mode hook set to `pair` (-1 automatic, 0 single tiles, 1 tile pairs), then automatic."""
    lib = _native.load()
    _native.check(lib.hi3d_gemm_tc5_set_pair_mode(pair), "hi3d_gemm_tc5_set_pair_mode")
    try:
        return fn()
    finally:
        lib.hi3d_gemm_tc5_set_pair_mode(-1)


@pytest.mark.parametrize("nt,bn,N", TILE_TARGETS + [(0, 0, 320), (0, 0, 64)])
def test_gemm_fp8_plain_tiles(nt, bn, N):
    """Each tile of the engine at a plain-rows shape derived from this device's SM count, the engine's launch checked against the
    restated cost model; nt = 0: few rows (300 and 77), whatever the engine picks."""
    sms = sm_count()
    K = 320
    if nt:
        M, _, pair = tile_shape(ops.ROWS_PLAIN, nt, bn, N, K, sms)
    else:
        M, pair = (300 if N == 320 else 77), -1
    print(f"[fp8 plain tiles] {sms} SMs: M = {M}, N = {N}, pair mode {pair} -> {tc5_tile(K, N, tc5_m_tiles(ops.ROWS_PLAIN, M), sms, pair)}")
    g = torch.Generator().manual_seed(M + N)
    a = _a8(M, K, g)
    W8, sc, Wd = _w8(N, K, g)
    bias = torch.randn(N, generator=g).to(DEV)
    out = torch.empty(M, N, dtype=torch.float16, device=DEV)
    gm = ops.Gemm([ops.SegSpec(a)], W8, out, M, bias=bias, w_scale=sc, engine="tc5")
    launched = run_pair_mode(pair, lambda: tc5_launches(gm))
    want = tc5_tile(K, N, tc5_m_tiles(ops.ROWS_PLAIN, M), sms, pair)
    assert_launched(launched, want + ("__nv_fp8_e4m3",), f"plain M={M} N={N}")
    if nt:
        assert want == (nt, bn)
    _check(out, a.float() @ Wd.t() + bias, a.float().abs() @ Wd.abs().t(), f"plain M={M} N={N} pair={pair}")


@pytest.mark.parametrize("epi", ["rowbias", "residual", "blend", "geglu", "geglu_e4m3", "residual_e4m3"])
def test_gemm_fp8_epilogues(epi):
    g = torch.Generator().manual_seed(7)
    M, K, N, HW = 1024, 640, 256, 64
    a = _a8(M, K, g)
    W8, sc, Wd = _w8(N, K, g)
    bias = torch.randn(N, generator=g).to(DEV)
    geglu = epi.startswith("geglu")
    n_out = N // 2 if geglu else N
    kw = dict(bias=bias, w_scale=sc, engine="tc5")
    rowbias = residual = blend_x = None
    if epi == "rowbias":
        rowbias = torch.randn(M // HW, N, generator=g).half().to(DEV)
        kw.update(rowbias=rowbias, rb_div=HW, rb_mod=M // HW)
    if epi.startswith("residual") or epi == "blend":
        residual = torch.randn(M, n_out, generator=g).half().to(DEV)
        kw.update(residual=residual)
    if epi == "blend":
        blend_x = torch.randn(M, n_out, generator=g).half().to(DEV)
        kw.update(blend_x=blend_x, alpha=0.3)
    if geglu:
        kw.update(act=ops.ACT_GEGLU)
    fp8_out = epi.endswith("e4m3")
    out = torch.empty(M, n_out, dtype=E4M3 if fp8_out else torch.float16, device=DEV)
    ops.Gemm([ops.SegSpec(a)], W8, out, M, **kw)()
    ref = _epilogue(a.float() @ Wd.t(), bias, rowbias, HW, ops.ACT_GEGLU if geglu else 0, residual, blend_x, 0.3)
    absprod = a.float().abs() @ Wd.abs().t()
    if geglu:       # value x gelu(gate): the value's error times |gelu(gate)| <= |gate| + 1, plus the gate's times |value|
        v = a.float() @ Wd.t() + bias
        absprod = absprod[:, 0::2] * (v[:, 1::2].abs() + 1) + absprod[:, 1::2] * (v[:, 0::2].abs() + 1)
    _check(out, ref, absprod, epi, fp8_out)


@pytest.mark.parametrize("two_sources", [False, True])
def test_gemm_fp8_conv3x3(two_sources):
    g = torch.Generator().manual_seed(11)
    n, h, w, C, Co = 4, 16, 16, 320, 320
    srcs = [_a8(n * h * w, C, g) for _ in range(2 if two_sources else 1)]
    Ci = C * len(srcs)
    wt = torch.randn(Co, Ci, 3, 3, generator=g) / (9 * Ci) ** 0.5
    W8, sc = pack.pack_e4m3(pack.pack_conv2d(wt))
    W8, sc = W8.to(DEV), sc.to(DEV)
    bias = torch.randn(Co, generator=g).to(DEV)
    out = torch.empty(n * h * w, Co, dtype=torch.float16, device=DEV)
    ops.Gemm(ops.conv_taps(srcs), W8, out, n * h * w, mode=ops.ROWS_CONV2D, geom=dict(Ho=h, Wo=w, Hs=h, Ws=w), bias=bias,
             w_scale=sc, engine="tc5")()
    wd = (W8.float() * sc[:, None]).view(Co, 3, 3, Ci).permute(0, 3, 1, 2)
    x = torch.cat([s.float() for s in srcs], 1).view(n, h, w, Ci).permute(0, 3, 1, 2)
    ref = F.conv2d(x, wd, bias, padding=1).permute(0, 2, 3, 1).reshape(n * h * w, Co)
    absprod = F.conv2d(x.abs(), wd.abs(), padding=1).permute(0, 2, 3, 1).reshape(n * h * w, Co)
    _check(out, ref, absprod, f"conv3x3 sources={len(srcs)}")


def test_gemm_fp8_temporal():
    g = torch.Generator().manual_seed(13)
    B, T, HW, C, Co = 2, 16, 64, 320, 640
    M = B * T * HW
    a = _a8(M, C, g)
    wt = torch.randn(Co, C, 3, 1, 1, generator=g) / (3 * C) ** 0.5
    W8, sc = pack.pack_e4m3(pack.pack_conv3d_t(wt))
    W8, sc = W8.to(DEV), sc.to(DEV)
    bias = torch.randn(Co, generator=g).to(DEV)
    out = torch.empty(M, Co, dtype=torch.float16, device=DEV)
    ops.Gemm(ops.temporal_taps(a), W8, out, M, mode=ops.ROWS_TEMPORAL, geom=dict(Ho=HW, Wo=1, T=T), bias=bias, w_scale=sc,
             engine="tc5")()
    wd = (W8.float() * sc[:, None]).view(Co, 3, C)
    x = F.pad(a.float().view(B, T, HW, C), (0, 0, 0, 0, 1, 1))
    ref = sum(x[:, d:d + T] @ wd[:, d].t() for d in range(3)).reshape(M, Co) + bias
    absprod = sum(x[:, d:d + T].abs() @ wd[:, d].abs().t() for d in range(3)).reshape(M, Co)
    _check(out, ref, absprod, "temporal")


def test_gemm_fp8_refuses_what_it_does_not_cover():
    g = torch.Generator().manual_seed(17)
    a = _a8(128, 64, g)
    W8, sc, _ = _w8(16, 64, g)                                # N < 32: the fp16 engine would hand this to mma.sync
    out = torch.empty(128, 16, dtype=torch.float16, device=DEV)
    with pytest.raises(_native.Hi3dError, match="not covered"):
        ops.Gemm([ops.SegSpec(a)], W8, out, 128, w_scale=sc)()


# ---- the UNet ---------------------------------------------------------------------------------------------------------------------
KW_S1 = dict(adm_in_channels=768, num_classes="sequential", use_checkpoint=True, in_channels=8, out_channels=4,
             model_channels=64, attention_resolutions=[4, 2, 1], num_res_blocks=2, channel_mult=[1, 2, 4, 4],
             num_head_channels=64, use_linear_in_transformer=True, transformer_depth=1, context_dim=1024,
             spatial_transformer_attn_type="softmax-xformers", extra_ff_mix_layer=True, use_spatial_context=True,
             merge_strategy="learned_with_images", video_kernel_size=[3, 1, 1])

FP8_LAYER = re.compile(r"\.(in_layers\.2|out_layers\.3|proj_in|attn1\.to_[qkv]|ff(_in)?\.net\.(0\.proj|2))$")


def _unet(seed=1):
    from hi3d_official_b200.unet import VideoUNet
    cfg = spec.UNetConfig.from_kwargs(**KW_S1)
    sd = spec.synth_state_dict(spec.unet_param_shapes(cfg), seed=seed)
    net = VideoUNet(**KW_S1)
    net.load_state_dict(sd, strict=True)
    return net.cuda().half(), {k: v.cuda() for k, v in sd.items()}


def _inputs(N, hw, T, seed=0, in_channels=8, adm=768):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, in_channels, hw, hw, generator=g).cuda()
    ctx = torch.randn(N // T, 1, 1024, generator=g).cuda()
    ctx[0] = 0
    y = torch.randn(N // T, adm, generator=g).cuda()
    return x, ctx, y, torch.full((N,), 0.7).cuda()


def _qw(w: torch.Tensor) -> torch.Tensor:
    """A state-dict weight as the fp8 plan multiplies it: rounded to fp16, then to e4m3 with one scale amax / 448 per output row
    (pack.pack_e4m3), dequantised."""
    w16 = w.half().float()
    amax = w16.abs().flatten(1).amax(1)
    sc = torch.where(amax > 0, amax / 448, torch.ones_like(amax)).view(-1, *([1] * (w.dim() - 1)))
    return (w16 / sc).clamp(-448, 448).to(E4M3).float() * sc


class _QuantisingF:
    """torch.nn.functional for the oracle, with the fp8 plan's rounding at the layers whose weights are in `weights`: the input is
    rounded to fp16 then to e4m3, the weight to fp16 then to e4m3 with its per-output-row scale (pack.pack_e4m3)."""

    def __init__(self, weights):
        self.ptrs = {w.data_ptr() for w in weights}

    def __getattr__(self, name):
        return getattr(F, name)

    def _q(self, x, w):
        if w.data_ptr() not in self.ptrs:
            return x, w
        return e4m3_ref(x.half()).float(), _qw(w)

    def linear(self, x, w, b=None):
        return F.linear(*self._q(x, w), b)

    def conv2d(self, x, w, b=None, **kw):
        return F.conv2d(*self._q(x, w), b, **kw)

    def conv3d(self, x, w, b=None, **kw):
        return F.conv3d(*self._q(x, w), b, **kw)


def _rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm())


@pytest.mark.parametrize("T,hw", [(4, 16), (16, 8), (16, 32)])
def test_fp8_unet_vs_quantising_oracle(T, hw, monkeypatch):
    net, sd = _unet()
    net.set_precision("fp8")
    N = 2 * T
    x, ctx, y, t = _inputs(N, hw, T)
    out = net(x, timesteps=t, context=ctx, y=y, num_video_frames=T)
    plan = net.get_plan(N, hw, hw, T)
    assert torch.isfinite(out).all()
    ref = O.unet_forward(sd, x, t, ctx, y, num_video_frames=T)
    monkeypatch.setattr(O, "F", _QuantisingF([sd[n + ".weight"] for n in plan.fp8_layers]))
    ref_emu = O.unet_forward(sd, x, t, ctx, y, num_video_frames=T)
    e_q, e_emu = _rel(out, ref), _rel(out, ref_emu)
    print(f"[fp8 unet mc=64 T={T} hw={hw}] e_q (vs fp32 oracle) {e_q:.4e}  e_emu (vs quantising oracle) {e_emu:.4e}")
    # The quantising oracle reproduces the plan's rounding only until an fp16-sized difference between the plan's and the
    # oracle's input of a quantiser crosses an e4m3 rounding boundary (one step is 6 to 12 %); such flips then cascade through
    # the later layers.  So it explains only part of the fp8 error: measured on an H100, e_emu / e_q = 0.87 .. 0.88 here.
    assert e_q < 0.12 and e_emu < 0.95 * e_q


# ---- layer by layer: every GEMM of the fp8 plan against the state dict, on the inputs the plan gave it ---------------------------
def _layer_reference(sd, g, srcs, residual, blend_x, rowbias, skip_ref):
    """fp32 reference of plan GEMM `g` (g.layers = the state-dict layers it computes) from the state dict alone, applied to the
    plan's own inputs of that GEMM (srcs: its distinct segment sources, e4m3 or fp16) and, for the epilogue, the plan's rowbias,
    residual and blend tensors -- except the residual of a channel-changing ResBlock's conv2, which is the reference 1x1 skip of
    the block input (`skip_ref`).  Returns (reference, sum |a w| per output)."""
    p, name = g.p, g.layers[0]
    x = torch.cat([t.float() for t in srcs], 1)
    w = torch.cat([sd[n + ".weight"] for n in g.layers], 0).float()
    w = _qw(w) if g.fp8 else w.half().float()
    b = torch.cat([sd[n + ".bias"] for n in g.layers], 0).float() if name + ".bias" in sd else None
    if w.dim() == 4 and w.shape[-1] == 3:                     # 3x3 conv
        xn = x.view(-1, p.Ho, p.Wo, x.shape[1]).permute(0, 3, 1, 2)
        y, a = (F.conv2d(v, u, padding=1).permute(0, 2, 3, 1).reshape(p.M, -1) for v, u in ((xn, w), (xn.abs(), w.abs())))
    elif w.dim() == 5:                                          # (3, 1, 1) temporal conv over [B, T, HW, C]
        HW = p.Ho * p.Wo
        x5 = x.view(-1, p.T, HW, x.shape[1]).permute(0, 3, 1, 2)[..., None]
        y, a = (F.conv3d(v, u, padding=(1, 0, 0))[..., 0].permute(0, 2, 3, 1).reshape(p.M, -1)
                for v, u in ((x5, w), (x5.abs(), w.abs())))
    else:                                                       # linear / 1x1 conv
        w = w.flatten(1)
        y, a = x @ w.t(), x.abs() @ w.abs().t()
    if b is not None:
        y = y + b
    if p.rowbias:
        y = y + rowbias.float()[torch.arange(p.M, device=DEV) // p.rb_div % p.rb_mod]
    if p.act == ops.ACT_GEGLU:                                  # reference row order [value ; gate]
        v, gt = y.chunk(2, 1)
        av, ag = a.chunk(2, 1)
        y, a = v * F.gelu(gt), av * (gt.abs() + 1) + ag * (v.abs() + 1)
    if name.endswith("out_layers.3") and skip_ref is not None:
        residual = skip_ref
    if residual is not None:
        y, a = y + residual.float(), a + 2 ** -10 * residual.float().abs()    # (+ the fp16 rounding of the plan's residual)
    if blend_x is not None:
        y = p.alpha * blend_x.float() + (1 - p.alpha) * y
    return y, a


def _teacher_forced_mismatches(net, sd, N, hw, T, inputs=_inputs, seen=None, after=None):
    """Runs the fp8 plan launch by launch; checks each GEMM that computes state-dict layers against _layer_reference with the
    GEMM tests' tolerance (_check).  Returns [(layer, message)] of the GEMMs outside it.  inputs(N, hw, T) -> (x, context, y,
    timesteps); seen: a list that gets (layer, GEMM, _check's ratio or None) of every checked GEMM; after(step): called after
    every other step."""
    x, ctx, y, t = inputs(N, hw, T)
    net(x, timesteps=t, context=ctx, y=y, num_video_frames=T)       # conditioning, input and timesteps of the plan
    plan = net.get_plan(N, hw, hw, T)
    bad, skip_ref, checked = [], None, 0
    for s in plan.steps:
        layers = getattr(s, "layers", None) if isinstance(s, ops.Gemm) else None
        if layers is None:
            s()
            if after is not None:
                after(s)
            continue
        segs, _, out, _, rowbias, residual, blend_x, _ = s._keep
        srcs = list({sg.src.data_ptr(): sg.src for sg in segs}.values())
        srcs = [t_.clone() for t_ in srcs]
        residual, blend_x = (None if t_ is None else t_.clone() for t_ in (residual, blend_x))
        s()
        ref, absprod = _layer_reference(sd, s, srcs, residual, blend_x, rowbias, skip_ref)
        checked += 1
        if layers[0].endswith("skip_connection"):
            skip_ref = ref
        elif layers[0].endswith("out_layers.3"):
            skip_ref = None
        ratio = None
        try:
            ratio = _check(out[:s.p.M], ref, absprod, layers[0], fp8_out=out.dtype == E4M3)
        except AssertionError as e:
            bad.append((layers[0], str(e).splitlines()[0]))
        if seen is not None:
            seen.append((layers[0], s, ratio))
    assert checked >= len(plan.fp8_layers) // 3
    return bad


def test_fp8_plan_layers_teacher_forced():
    """Every FP8 GEMM (and the fp16 1x1 skips split out of conv2) computes its state-dict layer: weight, scale, bias, epilogue."""
    net, sd = _unet()
    net.set_precision("fp8")
    bad = _teacher_forced_mismatches(net, sd, 32, 32, 16)
    assert not bad, bad


@pytest.mark.parametrize("fault", ["skip_bias_dropped", "conv2_with_fused_bias", "qkv_scale_off_by_one_step"])
def test_teacher_forced_check_catches_wiring_faults(fault):
    """The layer-by-layer check is sensitive: a wiring fault of the fp8 plan's new paths, planted in its packed weights, is
    reported at the layer it breaks."""
    net, sd = _unet()
    net.set_precision("fp8")
    Q, P = net._pack_fp8(), net._pack()
    blk = next(k[:-len("skip")] for k in Q if k.endswith("skip"))                    # a channel-changing ResBlock
    qkv = next(k for k in Q if k.endswith("qkv"))
    if fault == "skip_bias_dropped":
        Q[blk + "skip"] = (Q[blk + "skip"][0], torch.zeros_like(Q[blk + "skip"][1]))
        want = blk + "skip_connection"
    elif fault == "conv2_with_fused_bias":
        Q[blk + "conv2.bias"] = P[blk + "conv2"][1]
        want = blk + "out_layers.3"
    else:
        Q[qkv] = (Q[qkv][0], Q[qkv][1] * (1 + 2 ** -3))
        want = qkv[:-len("qkv")] + "attn1.to_q"
    bad = _teacher_forced_mismatches(net, sd, 32, 32, 16)
    assert want in [b[0] for b in bad], (want, bad)


def test_fp8_layer_set():
    """At 32^2 latents and 16 frames (as at the sampler's sizes) the e4m3 engine covers every layer of the FP8 set."""
    net, sd = _unet()
    net.set_precision("fp8")
    plan = net.get_plan(32, 32, 32, 16)
    expected = sorted(k[:-len(".weight")] for k in sd if k.endswith(".weight") and FP8_LAYER.search(k[:-len(".weight")]))
    assert len(plan.fp8_layers) == len(set(plan.fp8_layers))
    assert sorted(plan.fp8_layers) == expected
    net.set_precision("fp16")
    assert net.get_plan(32, 32, 32, 16).fp8_layers == []


@pytest.mark.parametrize("stage,hw", [(1, 64), (2, 128)])
def test_fp8_covers_every_layer_at_the_sampler_shapes(stage, hw):
    """The full-width UNets at the sampler's CFG batch (2 x 16 frames) and latent sizes run every layer of the FP8 set in FP8."""
    from hi3d_official_b200 import configs
    from hi3d_official_b200.unet import VideoUNet
    cfg = (configs.stage1_config() if stage == 1 else configs.stage2_config())["model"]["params"]["network_config"]["params"]
    net = VideoUNet(**cfg).cuda().half()
    spec.synth_fill_(net, seed=0, fast=True)
    net.set_precision("fp8")
    plan = net.get_plan(32, hw, hw, 16)
    names = [k[:-len(".weight")] for k in net.state_dict() if k.endswith(".weight")]
    assert sorted(plan.fp8_layers) == sorted(n for n in names if FP8_LAYER.search(n))


def test_fp8_sampler_step_repeatable_and_batch_invariant():
    from test_batch_gpu import _fused_step, _stage1_model
    torch.manual_seed(0)
    model = _stage1_model()
    model.model.diffusion_model.set_precision("fp8")
    B, T, h = 2, 16, 16
    g = torch.Generator().manual_seed(31)
    x = (torch.randn(B * T, 4, h, h, generator=g) * 8).to(DEV)
    c = dict(crossattn=torch.randn(B, 1, 1024, generator=g).to(DEV), vector=torch.randn(B, 768, generator=g).to(DEV),
             concat=(torch.randn(B * T, 4, h, h, generator=g) * 0.18).half().to(DEV))
    uc = dict(crossattn=torch.zeros_like(c["crossattn"]), vector=c["vector"].clone(), concat=torch.zeros_like(c["concat"]))
    sigma = torch.full((B * T,), 8.0, device=DEV)
    sigma_next = torch.full((B * T,), 6.5, device=DEV)
    xb, db = _fused_step(model, x, c, uc, sigma, sigma_next)
    xb2, db2 = _fused_step(model, x, c, uc, sigma, sigma_next)
    assert torch.isfinite(xb).all()
    assert torch.equal(xb, xb2) and torch.equal(db, db2), "two fp8 runs of the same batched step differ"
    model.sampler._fused.clear()
    s = slice(0, T)
    cb = {k: (v[s] if k == "concat" else v[0:1]).contiguous() for k, v in c.items()}
    ucb = {k: (v[s] if k == "concat" else v[0:1]).contiguous() for k, v in uc.items()}
    x1, d1 = _fused_step(model, x[s].contiguous(), cb, ucb, sigma[s].contiguous(), sigma_next[s].contiguous())
    assert torch.equal(xb[s], x1) and torch.equal(db[s], d1), "fp8: object 0 alone differs from object 0 of a batch of two"


def _run(script, *args):
    r = subprocess.run([sys.executable, os.path.join(ROOT, script), *args], capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-1500:] + r.stderr[-3000:]
    return r.stdout


def test_pipelines_run_fp8(tmp_path):
    out = str(tmp_path / "out")
    assert "first.mp4" in _run("pipeline_i2v_eval_v01.py", "--tiny", "--synthetic", "--precision", "fp8", "--output_dir", out,
                               "--seed", "1")
    first = torch.load(os.path.join(out, "first_step", "first.pt"))
    assert first.shape == (16, 3, 128, 128) and torch.isfinite(first.float()).all()
    assert "second.mp4" in _run("pipeline_i2v_eval_v02.py", "--tiny", "--synthetic", "--precision", "fp8", "--output_dir", out,
                                "--seed", "1")
    second = torch.load(os.path.join(out, "second_step_video", "second.pt"))
    assert second.shape == (16, 3, 256, 256) and torch.isfinite(second.float()).all()
