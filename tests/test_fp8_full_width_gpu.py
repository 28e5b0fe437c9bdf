"""FP8 at the UNet's full width: the e4m3 wgmma GEMM at the shapes of the full-width plans (tile pairs in conv and temporal
modes, a 9-tap x 2-source concat at K = 23040), tile coverage derived from this device's SM count, the accumulation error of
Hopper's FP8 MMA at long K (GEMM and attention), and the full-width stage-1 / stage-2 plans layer by layer and as a whole against
fp32 references.

Tolerances are test_fp8_gpu._check's (2e-3 |ref| + 2^-10 sum_k |a_k w_k| + 1e-3 mean |ref|, one e4m3 step for e4m3 outputs) and
test_fp8_attention_gpu.reference_and_bound's for the e4m3 attention core."""
import functools
import gc
import re

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from hi3d_official_b200 import configs, ops, pack, spec  # noqa: E402
from oracle import hi3d_oracle as O  # noqa: E402
from test_fp8_attention_gpu import _assert_within, attn_fp8, reference_and_bound  # noqa: E402
from test_fp8_gpu import (DEV, E4M3, TILE_TARGETS, _a8, _check, _epilogue, _inputs, _rel, _teacher_forced_mismatches,  # noqa: E402
                          _w8, assert_launched, gemm_tile, run_pair_mode, sm_count, tc5_launches, tc5_m_tiles, tc5_tile, tile_shape)

F16 = torch.float16
FP8_KERNEL = "__nv_fp8_e4m3"


# ---- 1. the e4m3 GEMM at the full-width plans' shapes --------------------------------------------------------------------------
def _conv_case(g, n, hw, cs, Co):
    """3x3 conv over the channel concat of e4m3 sources with cs channels (9 taps x len(cs) segments), bias + per-image rowbias
    as the ResBlock's conv1."""
    srcs = [_a8(n * hw * hw, c, g) for c in cs]
    Ci = sum(cs)
    wt = torch.randn(Co, Ci, 3, 3, generator=g) / (9 * Ci) ** 0.5
    W8, sc = (t.to(DEV) for t in pack.pack_e4m3(pack.pack_conv2d(wt)))
    bias = torch.randn(Co, generator=g).to(DEV)
    emb = torch.randn(n, Co, generator=g).half().to(DEV)
    M = n * hw * hw
    kw = dict(mode=ops.ROWS_CONV2D, geom=dict(Ho=hw, Wo=hw, Hs=hw, Ws=hw), bias=bias, rowbias=emb, rb_div=hw * hw, rb_mod=n)
    wd = (W8.float() * sc[:, None]).view(Co, 3, 3, Ci).permute(0, 3, 1, 2)
    x = torch.cat([s.float() for s in srcs], 1).view(n, hw, hw, Ci).permute(0, 3, 1, 2)
    acc, absprod = (F.conv2d(v, u, padding=1).permute(0, 2, 3, 1).reshape(M, Co) for v, u in ((x, wd), (x.abs(), wd.abs())))
    ref = _epilogue(acc, bias, emb, hw * hw, 0, None, None, 0.0)
    return ops.conv_taps(srcs), W8, sc, M, kw, ref, absprod


def _temporal_case(g, B, T, HW, C):
    """(3, 1, 1) temporal conv over clips of T frames, residual + blend as the temporal ResBlock's conv2."""
    M = B * T * HW
    a = _a8(M, C, g)
    wt = torch.randn(C, C, 3, 1, 1, generator=g) / (3 * C) ** 0.5
    W8, sc = (t.to(DEV) for t in pack.pack_e4m3(pack.pack_conv3d_t(wt)))
    bias = torch.randn(C, generator=g).to(DEV)
    res, blend = (torch.randn(M, C, generator=g).half().to(DEV) for _ in range(2))
    kw = dict(mode=ops.ROWS_TEMPORAL, geom=dict(Ho=HW, Wo=1, T=T), bias=bias, residual=res, blend_x=blend, alpha=0.4)
    wd = (W8.float() * sc[:, None]).view(C, 3, C)
    x = F.pad(a.float().view(B, T, HW, C), (0, 0, 0, 0, 1, 1))
    acc = sum(x[:, d:d + T] @ wd[:, d].t() for d in range(3)).reshape(M, C)
    absprod = sum(x[:, d:d + T].abs() @ wd[:, d].abs().t() for d in range(3)).reshape(M, C)
    return ops.temporal_taps(a), W8, sc, M, kw, _epilogue(acc, bias, None, 1, 0, res, blend, 0.4), absprod


def _plain_case(g, M, K, N, geglu=False):
    """The feed-forward's output projection (+ residual), or its GEGLU input projection (W rows interleaved value / gate)."""
    a = _a8(M, K, g)
    W8, sc, Wd = _w8(N, K, g)
    bias = torch.randn(N, generator=g).to(DEV)
    acc, absprod = a.float() @ Wd.t(), a.float().abs() @ Wd.abs().t()
    if geglu:
        v = acc + bias          # value x gelu(gate): the value's error times |gelu(gate)| <= |gate| + 1, plus the gate's times |value|
        absprod = absprod[:, 0::2] * (v[:, 1::2].abs() + 1) + absprod[:, 1::2] * (v[:, 0::2].abs() + 1)
        return [ops.SegSpec(a)], W8, sc, M, dict(bias=bias, act=ops.ACT_GEGLU), _epilogue(acc, bias, None, 1, ops.ACT_GEGLU,
                                                                                          None, None, 0.0), absprod
    res = torch.randn(M, N, generator=g).half().to(DEV)
    return [ops.SegSpec(a)], W8, sc, M, dict(bias=bias, residual=res), _epilogue(acc, bias, None, 1, 0, res, None, 0.0), absprod


CASES = {
    "conv3x3_c320_32x64x64": lambda g: _conv_case(g, 32, 64, [320], 320),                    # K = 2880
    "conv1_concat_1280+1280_32x16x16": lambda g: _conv_case(g, 32, 16, [1280, 1280], 1280),  # K = 23040, 18 segments, 2 maps
    "conv1_concat_1280+1280_32x8x8": lambda g: _conv_case(g, 32, 8, [1280, 1280], 1280),     # two-image patches
    "temporal_c640_T16": lambda g: _temporal_case(g, 2, 16, 1024, 640),                       # K = 1920
    "temporal_c1280_T16": lambda g: _temporal_case(g, 2, 16, 256, 1280),                      # K = 3840
    "ff2_k2560": lambda g: _plain_case(g, 32768, 2560, 640),
    "ff2_k5120": lambda g: _plain_case(g, 8192, 5120, 1280),
    "geglu_c1280": lambda g: _plain_case(g, 8192, 1280, 10240, geglu=True),
}


def _nan_out(rows, cols, dtype):
    """An output buffer full of NaN (0x7F in e4m3)."""
    if dtype == E4M3:
        return torch.full((rows, cols), 0x7F, dtype=torch.uint8, device=DEV).view(E4M3)
    return torch.full((rows, cols), float("nan"), dtype=F16, device=DEV)


def _untouched(t: torch.Tensor) -> bool:
    return bool((t.view(torch.uint8) == 0x7F).all()) if t.dtype == E4M3 else bool(torch.isnan(t).all())


@pytest.mark.parametrize("case", list(CASES))
def test_gemm_fp8_full_width_shapes(case):
    """Each case with the pair mode automatic, single tiles forced and pairs forced, into fp16 and e4m3 outputs with 37 extra rows
    and 24 extra columns of NaN: the kernel the engine launches is the one the restated cost model names, every result is
    within _check, and nothing outside [M, N] is written."""
    g = torch.Generator().manual_seed(len(case))
    segs, W8, sc, M, kw, ref, absprod = CASES[case](g)
    sms, K, N = sm_count(), W8.shape[1], W8.shape[0]
    n_out = ref.shape[1]
    p = kw.get("geom", {})
    m_tiles = tc5_m_tiles(kw.get("mode", ops.ROWS_PLAIN), M, p.get("Ho", 1), p.get("Wo", 1), p.get("T", 1))
    assert len(segs) <= 24 and len({s.src.data_ptr() for s in segs}) <= 4
    worst = {}
    for dtype in (F16, E4M3):
        for pair in (-1, 0, 1):
            out = _nan_out(M + 37, n_out + 24, dtype)
            gm = ops.Gemm(segs, W8, out, M, w_scale=sc, engine="tc5", **kw)
            launched = run_pair_mode(pair, lambda: tc5_launches(gm))
            tile = tc5_tile(K, N, m_tiles, sms, pair)
            assert_launched(launched, tile + (FP8_KERNEL,), f"{case} pair mode {pair}")
            what = f"{case} K={K} {'e4m3' if dtype == E4M3 else 'fp16'} out, pair mode {pair} ({tile[0]} x {tile[1]})"
            worst[(dtype, pair, tile)] = _check(out[:M, :n_out], ref, absprod, what, fp8_out=dtype == E4M3)
            assert _untouched(out[M:]) and _untouched(out[:M, n_out:]), f"{what}: wrote outside [M, N]"
    print(f"[fp8 full-width GEMM] {case}: M={M} K={K} N={N}, {len(segs)} segments, {sms} SMs; worst err/tol (fp16) or e4m3 steps: "
          + ", ".join(f"{'e4m3' if d == E4M3 else 'fp16'} pair {p_} {t[0]}x{t[1]}: {r:.3f}" for (d, p_, t), r in worst.items()))


# ---- 2. tile coverage from this device's SM count ------------------------------------------------------------------------------
@pytest.mark.parametrize("nt,bn,N", TILE_TARGETS)
@pytest.mark.parametrize("mode", [ops.ROWS_CONV2D, ops.ROWS_TEMPORAL], ids=["conv2d", "temporal"])
def test_gemm_fp8_tile_coverage(mode, nt, bn, N):
    """Each tile of the engine in conv2d (8 x 8 images, two-image patches) and temporal (16 frames of 64 pixels, two-frame
    patches) mode, at the shape tile_shape derives from this device's SM count (plain rows: test_fp8_gpu.test_gemm_fp8_plain_tiles)."""
    sms = sm_count()
    conv = mode == ops.ROWS_CONV2D
    C = 64 if conv else 128
    K = 9 * C if conv else 3 * C
    M, geom, pair = tile_shape(mode, nt, bn, N, K, sms)
    print(f"[fp8 tile coverage] {sms} SMs, {'conv2d' if conv else 'temporal'}: M = {M}, N = {N}, pair mode {pair} -> {nt} x {bn}")
    g = torch.Generator().manual_seed(M + N)
    a = _a8(M, C, g)
    bias = torch.randn(N, generator=g).to(DEV)
    if conv:
        hw = geom["Ho"]
        wt = torch.randn(N, C, 3, 3, generator=g) / K ** 0.5
        W8, sc = (t.to(DEV) for t in pack.pack_e4m3(pack.pack_conv2d(wt)))
        segs = ops.conv_taps([a])
        wd = (W8.float() * sc[:, None]).view(N, 3, 3, C).permute(0, 3, 1, 2)
        x = a.float().view(-1, hw, hw, C).permute(0, 3, 1, 2)
        acc, absprod = (F.conv2d(v, u, padding=1).permute(0, 2, 3, 1).reshape(M, N) for v, u in ((x, wd), (x.abs(), wd.abs())))
    else:
        HW, T = geom["Ho"], geom["T"]
        wt = torch.randn(N, C, 3, 1, 1, generator=g) / K ** 0.5
        W8, sc = (t.to(DEV) for t in pack.pack_e4m3(pack.pack_conv3d_t(wt)))
        segs = ops.temporal_taps(a)
        wd = (W8.float() * sc[:, None]).view(N, 3, C)
        x = F.pad(a.float().view(-1, T, HW, C), (0, 0, 0, 0, 1, 1))
        acc = sum(x[:, d:d + T] @ wd[:, d].t() for d in range(3)).reshape(M, N)
        absprod = sum(x[:, d:d + T].abs() @ wd[:, d].abs().t() for d in range(3)).reshape(M, N)
    out = torch.empty(M, N, dtype=F16, device=DEV)
    gm = ops.Gemm(segs, W8, out, M, mode=mode, geom=geom, bias=bias, w_scale=sc, engine="tc5")
    launched = run_pair_mode(pair, lambda: tc5_launches(gm))
    assert_launched(launched, (nt, bn, FP8_KERNEL), f"mode {mode} M={M} N={N}")
    _check(out, acc + bias, absprod, f"{'conv2d' if conv else 'temporal'} M={M} N={N} {nt} x {bn}")


# ---- 3. accumulation error at long K -------------------------------------------------------------------------------------------
def _accumulation(out, ref, absprod):
    """(max err / sum |a w|, max err / |ref|) of an fp16 output against a float64 reference."""
    err = (out.double() - ref).abs()
    live = absprod > 0                                # not the all-zero weight row of _w8
    return float((err / absprod)[live].max()), float((err / ref.abs())[live].max())


@pytest.mark.parametrize("K", [2880, 11520, 23040])
def test_accumulation_error_long_k(K):
    """Hopper's FP8 wgmma adds products into its accumulator with reduced precision relative to the accumulator's magnitude; the
    engine restarts the chain every 128 K elements and adds it into fp32 registers.  Random e4m3 operands like the layers' (N(0, 1)
    activations, weights of std K^-1/2 with per-row scales) must meet _check; structured ones -- a dominant product of 448 first
    or last, then K - 1 positive products whose sum is 2^-5 .. 2^2 times it, one ratio per column -- are the worst case for the
    truncation: measured on an H100, 1 to 5.4 x 2^-10 of sum |a w| with the 128-element chains, 46 to 549 x 2^-10 with one chain
    over the whole K.  They must stay below 8 x 2^-10.  Both are printed as fractions of sum |a w| (and of |ref|)."""
    g = torch.Generator().manual_seed(K)
    M, N = 2048, 256
    a = _a8(M, K, g)
    W8, sc, Wd = _w8(N, K, g)
    out = torch.empty(M, N, dtype=F16, device=DEV)
    ops.Gemm([ops.SegSpec(a)], W8, out, M, w_scale=sc, engine="tc5")()
    ref, absprod = a.double() @ Wd.double().t(), a.double().abs() @ Wd.double().abs().t()
    ratio = _check(out, ref.float(), absprod.float(), f"random e4m3 K={K}")
    e_abs, e_rel = _accumulation(out, ref, absprod)
    lines = [f"random: err/sum|aw| {e_abs:.3e} ({e_abs * 1024:.3f} x 2^-10), err/|ref| {e_rel:.3e}, err/tol {ratio:.3f}"]
    Ms, Ns, worst = 256, 64, 0.0
    j = torch.arange(Ns) % 8 - 5
    for pos, where in ((0, "first"), (K - 1, "last")):
        a_s = (torch.rand(Ms, K, generator=g) * 1.5 + 0.5).to(E4M3).float()
        a_s[:, pos] = 448
        w = (448 / K * 2.0 ** j.float())[:, None].expand(Ns, K).clone()
        w[:, pos] = 1
        W8s, scs = (t.to(DEV) for t in pack.pack_e4m3(w.half()))
        a8 = a_s.to(E4M3).to(DEV)
        o = torch.empty(Ms, Ns, dtype=F16, device=DEV)
        ops.Gemm([ops.SegSpec(a8)], W8s, o, Ms, w_scale=scs, engine="tc5")()
        torch.cuda.synchronize()
        wd = W8s.double() * scs.double()[:, None]
        r = a8.double() @ wd.t()                      # every product is positive: sum |a w| = ref
        e_abs, _ = _accumulation(o, r, r)
        lines.append(f"dominant {where}: err/sum|aw| {e_abs:.3e} ({e_abs * 1024:.3f} x 2^-10)")
        worst = max(worst, e_abs)
    print(f"[fp8 accumulation K={K}] " + "; ".join(lines))
    assert worst < 8 * 2 ** -10


@pytest.mark.parametrize("L", [4096, 16384])
def test_attention_fp8_spread_over_long_l(L):
    """Attention spread over all L keys (scores within a few units) on values of mean 1: P V sums L products of one sign, the
    worst case for the reduced-precision accumulation of P V (before each 128-key tile got its own accumulator, the outputs came
    out up to 8 % small at L = 4096).  Every output within reference_and_bound."""
    n_img, heads = 2, 2
    C = heads * 64
    g = torch.Generator(device=DEV).manual_seed(L)
    qk = torch.randn(n_img * L, 2 * C, generator=g, device=DEV) * 0.25
    v = 1 + 0.5 * torch.randn(n_img * L, C, generator=g, device=DEV)
    qkv8 = torch.cat([qk, v], 1).to(E4M3)
    out = attn_fp8(qkv8, n_img, L, heads)
    rows = torch.arange(0, L, L // 256, device=DEV)
    worst = 0.0
    for img, h in ((0, 0), (n_img - 1, heads - 1)):
        ref, bound = reference_and_bound(qkv8, n_img, L, heads, 0.125, img, h, rows)
        worst = max(worst, _assert_within(out[img * L + rows, h * 64:(h + 1) * 64], ref, bound, f"L={L} image {img} head {h}"))
    print(f"[fp8 attention spread, L={L}] max |err| / bound {worst:.3f}")


# ---- 4-6. the full-width plans -----------------------------------------------------------------------------------------------
_MODEL = {}


def _full_width(stage: int):
    """(VideoUNet, fp32 state dict on the GPU, inputs(N, hw, T) for its channel counts) of the full-width stage-`stage` UNet,
    synthetic weights (seed 1); one model at a time."""
    if stage not in _MODEL:
        _release()
        from hi3d_official_b200.unet import VideoUNet
        cfg = (configs.stage1_config() if stage == 1 else configs.stage2_config())["model"]["params"]["network_config"]["params"]
        net = VideoUNet(**cfg).cuda().half()
        spec.synth_fill_(net, seed=1, fast=True)
        sd = {k: v.float() for k, v in net.state_dict().items()}
        _MODEL[stage] = (net, sd, functools.partial(_inputs, in_channels=cfg["in_channels"], adm=cfg["adm_in_channels"]))
    return _MODEL[stage]


def _release():
    _MODEL.clear()
    gc.collect()
    torch.cuda.empty_cache()


@pytest.fixture(scope="module", autouse=True)
def _one_model_at_a_time():
    yield
    _release()


def _kind(layer: str) -> str:
    base = next(k for pat, k in ((r"skip_connection$", "1x1 skip (fp16)"), (r"(in|out)_layers\.\d$", "conv"),
                                 (r"proj_in$", "proj_in"), (r"attn1\.to_q$", "q|k|v"), (r"net\.0\.proj$", "GEGLU"),
                                 (r"net\.2$", "ff2")) if re.search(pat, layer))
    return ("temporal " if ".time_stack." in layer else "spatial ") + base


def _attention_checker(ratios: list):
    """after(step) for _teacher_forced_mismatches: every e4m3 attention step against reference_and_bound on every
    (L / 256)-th query row of its first and last (image, head)."""
    def after(s):
        if not hasattr(s, "io"):
            return
        qkv8, att, n_img, L, heads = s.io
        rows = torch.arange(0, L, max(1, L // 256), device=DEV)
        for img, h in ((0, 0), (n_img - 1, heads - 1)):
            ref, bound = reference_and_bound(qkv8.t, n_img, L, heads, 0.125, img, h, rows)
            ratios.append(_assert_within(att.t[img * L + rows, h * 64:(h + 1) * 64], ref, bound, f"{s.block} image {img} head {h}"))
    return after


def _teacher_forced_full_width(stage: int, hw: int, precision: str):
    """The full-width plan at the sampler's CFG batch (2 x 16 frames) launch by launch: every GEMM against its state-dict layer,
    and with fp8_attn every e4m3 attention step against its bound."""
    net, sd, inputs = _full_width(stage)
    net.set_precision(precision)
    sms = sm_count()
    seen, attn = [], []
    after = _attention_checker(attn) if precision == "fp8_attn" else None
    try:
        bad = _teacher_forced_mismatches(net, sd, 32, hw, 16, inputs=inputs, seen=seen, after=after)
        n_attention = len(net.get_plan(32, hw, hw, 16).fp8_attention)
    finally:
        net.set_precision("fp16")                                      # drops the plan and its buffers
    kinds = {}
    for layer, gm, ratio in seen:
        k = kinds.setdefault(_kind(layer), [0, 0, 0.0, 0, gm.out.dtype == E4M3])
        k[0] += 1
        k[1] += gemm_tile(gm, sms)[0] == 2
        k[2] = max(k[2], ratio or 0.0)
        k[3] = max(k[3], gm.p.K)
    n_pairs = sum(k[1] for k in kinds.values())
    print(f"\n[fp8 full width stage {stage}, {hw}x{hw}, {precision}] {sms} SMs: {len(seen)} GEMMs checked, {n_pairs} on tile pairs")
    for name, (n, pairs, worst, kmax, e4m3_out) in sorted(kinds.items()):
        print(f"  {name:24s} {n:3d} GEMMs ({pairs:3d} on pairs), K up to {kmax:5d}: worst "
              + (f"e4m3 steps {worst:.0f}" if e4m3_out else f"err/tol {worst:.3f}"))
    if attn:
        print(f"  e4m3 attention           {len(attn) // 2:3d} steps: worst err/bound {max(attn):.3f}")
    assert not bad, bad
    assert n_pairs > 0
    assert kinds["spatial conv"][3] == 23040
    if precision == "fp8_attn":
        assert len(attn) == 2 * n_attention > 0


@pytest.mark.parametrize("precision", ["fp8", "fp8_attn"])
def test_stage1_full_width_teacher_forced(precision):
    _teacher_forced_full_width(1, 64, precision)


def test_stage1_full_width_check_catches_a_scale_fault_on_a_pair_concat_conv():
    """A weight scale one e4m3 step off on a K = 23040 concat conv1 that runs on tile pairs is reported at that layer."""
    net, sd, inputs = _full_width(1)
    sms = sm_count()
    net.set_precision("fp8")
    plan = net.get_plan(32, 64, 64, 16)
    target = next(s for s in plan.steps if isinstance(s, ops.Gemm) and s.fp8 and s.layers and s.p.K == 23040
                  and re.search(r"^output_blocks\.\d+\.0\.in_layers\.2$", s.layers[0]) and gemm_tile(s, sms)[0] == 2)
    want = target.layers[0]
    key = want[:-len("in_layers.2")] + "conv1"
    del plan, target
    Q = net._pack_fp8()
    orig = Q[key]
    Q[key] = (orig[0], orig[1] * (1 + 2 ** -3))
    net.set_precision("fp16")                                          # the next fp8 plan bakes the planted scale
    net.set_precision("fp8")
    try:
        bad = _teacher_forced_mismatches(net, sd, 32, 64, 16, inputs=inputs)
    finally:
        Q[key] = orig
        net.set_precision("fp16")
    print(f"[planted scale fault at {want}] reported: {bad}")
    assert want in [b[0] for b in bad], (want, bad)


def test_stage1_full_width_forward_vs_fp32_oracle():
    """The whole stage-1 forward at full width (CFG batch 2 x 16 frames, 64^2 latents) in fp8 and fp8_attn against the fp32
    oracle on the same weights: relative L2 below 0.12, the bar of the model_channels = 64 UNet."""
    net, sd, inputs = _full_width(1)
    T, hw = 16, 64
    x, ctx, y, t = inputs(2 * T, hw, T)
    with torch.no_grad():
        ref = O.unet_forward(sd, x, t, ctx, y, num_video_frames=T)
    errs = {}
    try:
        for precision in ("fp16", "fp8", "fp8_attn"):
            net.set_precision(precision)
            out = net(x, timesteps=t, context=ctx, y=y, num_video_frames=T)
            assert torch.isfinite(out).all()
            errs[precision] = _rel(out, ref)
    finally:
        net.set_precision("fp16")
    print(f"[full width stage 1, {hw}x{hw}] rel L2 vs fp32 oracle: " + "  ".join(f"{k} {v:.4e}" for k, v in errs.items()))
    assert errs["fp8"] < 0.12 and errs["fp8_attn"] < 0.12


@pytest.mark.slow
@pytest.mark.parametrize("precision", ["fp8", "fp8_attn"])
def test_stage2_full_width_teacher_forced(precision):
    """Stage 2: 17 input channels, adm 512, 128^2 latents (L = 16384 at the top level)."""
    _teacher_forced_full_width(2, 128, precision)
