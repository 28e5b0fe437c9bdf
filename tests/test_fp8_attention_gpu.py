"""FP8 spatial attention (VideoUNet.set_precision("fp8_attn")): the V transpose bit for bit against a restatement of its documented
layout, the e4m3 kernel's wiring (one-hot keys), its arithmetic where P is exact, random e4m3 inputs at the UNet's shapes against
fp32 softmax attention with a bound derived from the kernel's rounding, tails, reproducibility, and the fp8_attn plan.

Error bound (reference_and_bound), per output element, with p_k = exp(scale (s_k - max s)) of the exact scores:
  [ sum_k max(2^-4 p'_k, 2^-18) |v_k|      P rounded to e4m3 after its 2^8 scaling (half a step, or half the smallest subnormal)
  + sum_k p_k eps_k (|v_k| + |ref|)        S error of Hopper's reduced-precision FP8 accumulation, |dS_k| <= 2^-10 sum_d |q_d k_d|,
                                           eps_k = exp(scale |dS_k|) - 1 (a shift common to all keys cancels in O / l)
  + 2^-10 sum_k p'_k |v_k| ] / sum_k p_k   P V accumulation
  + 2^-11 |ref|                            fp16 output
with p'_k = p_k (1 + eps_k)."""
import math
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

from hi3d_official_b200 import ops, spec  # noqa: E402
from oracle import hi3d_oracle as O  # noqa: E402

DEV = "cuda"
E4M3 = torch.float8_e4m3fn
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
UNET_SHAPES = [(32, 16384, 5), (32, 4096, 10), (32, 1024, 20), (32, 256, 20)]   # stage-2 spatial attention (n_img, L, heads)


def pi(k: torch.Tensor) -> torch.Tensor:
    """Key held by column k of a 32-block of vt (include/hi3d_b200.h)."""
    return (k & 16) + 8 * ((k >> 1) & 1) + 2 * ((k >> 2) & 3) + (k & 1)


def vt_reference(qkv8: torch.Tensor, n_img: int, L: int, heads: int) -> torch.Tensor:
    """vt as documented: e4m3 [n_img, heads, 64, Lp], V^T per (image, head), keys permuted by pi within 32-blocks, zero past L."""
    C = heads * 64
    Lp = (L + 127) // 128 * 128
    v = qkv8.view(torch.uint8)[:n_img * L, 2 * C:3 * C].reshape(n_img, L, heads, 64).permute(0, 2, 3, 1)
    pad = torch.zeros(n_img, heads, 64, Lp, dtype=torch.uint8, device=qkv8.device)
    pad[..., :L] = v
    col = torch.arange(Lp, device=qkv8.device)
    return pad[..., (col & ~31) + pi(col & 31)].contiguous()


def _vt(qkv8, n_img, L, heads):
    vt = torch.empty(ops.attention_vt_bytes(n_img, L, heads), dtype=E4M3, device=DEV)
    ops.attention_vt_e4m3(qkv8, n_img, L, heads, vt)
    return vt


def attn_fp8(qkv8, n_img, L, heads, scale=0.125, out=None):
    """The e4m3 path as the plan runs it: transpose, then the kernel."""
    vt = _vt(qkv8, n_img, L, heads)
    if out is None:
        out = torch.empty(n_img * L, heads * 64, dtype=torch.float16, device=DEV)
    ops.attention_d64_fp8(qkv8, vt, n_img, L, heads, out, scale)
    return out


def _e4m3_randn(rows, cols, g, std=1.0):
    return (torch.randn(rows, cols, generator=g, device=DEV) * std).to(E4M3)


def reference_and_bound(qkv8, n_img, L, heads, scale, img, h, rows):
    """fp32/fp64 softmax attention of query rows `rows` of (image img, head h) on the e4m3 values, and the error bound of the
    module docstring.  Returns (ref, bound), both [len(rows), 64]."""
    C = heads * 64
    x = qkv8[img * L:(img + 1) * L].double()
    q, k, v = x[rows, h * 64:(h + 1) * 64], x[:, C + h * 64:C + (h + 1) * 64], x[:, 2 * C + h * 64:2 * C + (h + 1) * 64]
    s = q @ k.t()
    p = torch.exp(scale * (s - s.amax(1, keepdim=True)))
    l = p.sum(1, keepdim=True)
    ref = (p @ v) / l
    ds = 2.0 ** -10 * (q.abs() @ k.abs().t())
    eps = torch.expm1(scale * ds)
    p1 = p * (1 + eps)
    err = torch.maximum(2.0 ** -4 * p1, torch.full_like(p1, 2.0 ** -18)) @ v.abs()
    err += (p * eps) @ v.abs() + (p * eps).sum(1, keepdim=True) * ref.abs()      # sum p eps |v - ref|, by the triangle inequality
    err += 2.0 ** -10 * (p1 @ v.abs())
    return ref, err / l + 2.0 ** -11 * ref.abs()


def _assert_within(out_rows, ref, bound, what):
    d = (out_rows.double() - ref).abs()
    bad = d > bound
    assert not bool(bad.any()), (f"{what}: {int(bad.sum())} of {bad.numel()} outside the bound; worst excess "
                                 f"{float((d - bound).max()):.3e}, max |err| {float(d.max()):.3e}")
    return float((d / bound.clamp_min(1e-30)).max())


# ---- 1. transpose --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_img,L,heads", [(3, 1, 2), (3, 77, 2), (2, 128, 5), (3, 1000, 3), (2, 16384, 5)])
def test_vt_matches_documented_layout(n_img, L, heads):
    g = torch.Generator(device=DEV).manual_seed(L)
    qkv8 = torch.randint(0, 256, (n_img * L, 3 * heads * 64), generator=g, device=DEV, dtype=torch.uint8)
    qkv8[qkv8 == 0x7F] = 0x7E
    qkv8[qkv8 == 0xFF] = 0xFE
    qkv8 = qkv8.view(E4M3)
    n = ops.attention_vt_bytes(n_img, L, heads)
    assert n == n_img * heads * 64 * ((L + 127) // 128 * 128)
    vt = torch.full((n,), 0x7F, dtype=torch.uint8, device=DEV).view(E4M3)        # NaN everywhere, pads included
    ops.attention_vt_e4m3(qkv8, n_img, L, heads, vt)
    want = vt_reference(qkv8, n_img, L, heads)
    assert torch.equal(vt.view(torch.uint8).view(want.shape), want)


# ---- 2. one-hot wiring ---------------------------------------------------------------------------------------------------------
_E4M3_CODES = torch.tensor([b for b in range(256) if b not in (0x7F, 0xFF)], dtype=torch.uint8)


def test_one_hot_keys_select_their_v_row():
    """Every query row has one key scoring >= 40 / scale above all others, that key sits at every position of a 32-block and of a
    128-key tile across the rows, and V holds distinct e4m3 values per (key mod 128, d): out must be that key's V row exactly."""
    n_img, L, heads, scale = 2, 300, 2, 0.125
    C = heads * 64
    pairs = torch.combinations(torch.arange(64), 2)                     # 2016 codes: key k has 24 at two channels
    assert L <= len(pairs)
    qkv = torch.zeros(n_img * L, 3 * C, dtype=torch.float32)
    tgt = torch.zeros(n_img, heads, L, dtype=torch.long)
    for i in range(n_img):
        for h in range(heads):
            key_code = pairs[torch.randperm(len(pairs), generator=torch.Generator().manual_seed(7 * i + h))[:L]]
            t = (torch.arange(L) * 7 + 3 + 5 * h + 11 * i) % L          # a bijection: every key is some row's target
            tgt[i, h] = t
            r = torch.arange(L)
            for c in range(2):
                qkv[i * L + r, h * 64 + key_code[t, c]] = 24.0
                qkv[i * L + r, C + h * 64 + key_code[r, c]] = 24.0
            d = torch.arange(64)
            code = (r[:, None] % 128 + 3 * d[None] + 5 * (r[:, None] // 128) + 11 * h + 13 * i) % len(_E4M3_CODES)
            qkv[i * L:(i + 1) * L, 2 * C + h * 64:2 * C + (h + 1) * 64] = _E4M3_CODES[code].view(E4M3).float()
    # the margin: target score 2 * 24^2, any other key at most 24^2
    assert 24.0 ** 2 >= 40 / scale
    qkv8 = qkv.to(E4M3).to(DEV)
    assert torch.equal(qkv8.float().cpu(), qkv)
    out = attn_fp8(qkv8, n_img, L, heads, scale).float().cpu()
    for i in range(n_img):
        for h in range(heads):
            want = qkv[i * L + tgt[i, h], 2 * C + h * 64:2 * C + (h + 1) * 64]
            got = out[i * L:(i + 1) * L, h * 64:(h + 1) * 64]
            bad = (got != want).any(1)
            assert not bool(bad.any()), f"image {i} head {h}: rows {bad.nonzero().flatten()[:8].tolist()} take the wrong V row"


# ---- 3. exact P ----------------------------------------------------------------------------------------------------------------
def test_exact_p_matches_oracle_to_accumulation_error():
    """Integer scores within 17 of the row maximum and scale = ln 2: every P * 256 is an exact power of two in e4m3."""
    n_img, L, heads, scale = 2, 1000, 3, math.log(2.0)
    C = heads * 64
    g = torch.Generator().manual_seed(3)
    q = torch.zeros(n_img * L, C)
    for h in range(heads):
        idx = torch.rand(n_img * L, 64, generator=g).argsort(1)[:, :8] + h * 64
        q.scatter_(1, idx, 1.0)                                          # 8 ones per row and head
    k = torch.randint(-1, 2, (n_img * L, C), generator=g).float()        # scores in [-8, 8]
    v = torch.randn(n_img * L, C, generator=g).to(E4M3).float()
    qkv8 = torch.cat([q, k, v], 1).to(E4M3).to(DEV)
    out = attn_fp8(qkv8, n_img, L, heads, scale)
    for i in range(n_img):
        for h in range(heads):
            x = qkv8[i * L:(i + 1) * L].double()
            s = x[:, h * 64:(h + 1) * 64] @ x[:, C + h * 64:C + (h + 1) * 64].t()
            assert float((s.amax(1, keepdim=True) - s).max()) <= 17
            p = torch.exp2(s - s.amax(1, keepdim=True))
            vv = x[:, 2 * C + h * 64:2 * C + (h + 1) * 64]
            l = p.sum(1, keepdim=True)
            ref = p @ vv / l
            bound = 2.0 ** -10 * (p @ vv.abs()) / l + 2.0 ** -11 * ref.abs()
            _assert_within(out[i * L:(i + 1) * L, h * 64:(h + 1) * 64], ref, bound, f"exact P image {i} head {h}")


# ---- 4. random e4m3 at the UNet shapes -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_img,L,heads", UNET_SHAPES)
def test_random_e4m3_at_unet_shapes(n_img, L, heads):
    g = torch.Generator(device=DEV).manual_seed(L + heads)
    C = heads * 64
    qkv8 = _e4m3_randn(n_img * L, 3 * C, g)
    out = attn_fp8(qkv8, n_img, L, heads)
    rows = torch.randperm(L, generator=torch.Generator().manual_seed(1))[:512].to(DEV)
    worst = 0.0
    for img, h in ((0, 0), (n_img - 1, heads - 1), (n_img // 2, heads // 2)):
        ref, bound = reference_and_bound(qkv8, n_img, L, heads, 0.125, img, h, rows)
        worst = max(worst, _assert_within(out[img * L + rows, h * 64:(h + 1) * 64], ref, bound, f"image {img} head {h}"))
    out16 = torch.empty_like(out)
    ops.attention_d64(qkv8.half(), n_img, L, heads, out16, engine="tc5")
    rel = float((out.float() - out16.float()).norm() / out16.float().norm())
    print(f"[fp8 attention {n_img}x{L}x{heads}] max |err| / bound {worst:.3f}; rel L2 vs the fp16 kernel on the same values {rel:.4e}")


# ---- 5. tails and guards -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("L", [1, 77, 200, 4097])
def test_tails_and_rows_past_the_output(L):
    n_img, heads = 3, 2
    C = heads * 64
    g = torch.Generator(device=DEV).manual_seed(L)
    qkv8 = _e4m3_randn(n_img * L, 3 * C, g)
    out = torch.full((n_img * L + 100, C), 7.0, dtype=torch.float16, device=DEV)
    attn_fp8(qkv8, n_img, L, heads, out=out)
    assert bool((out[n_img * L:] == 7.0).all()), "rows past n_img * L were written"
    rows = torch.arange(L, device=DEV) if L <= 512 else torch.cat([torch.arange(256), torch.arange(L - 256, L)]).to(DEV)
    for img in range(n_img):
        for h in range(heads):
            ref, bound = reference_and_bound(qkv8, n_img, L, heads, 0.125, img, h, rows)
            _assert_within(out[img * L + rows, h * 64:(h + 1) * 64], ref, bound, f"L={L} image {img} head {h}")


# ---- 6. reproducibility --------------------------------------------------------------------------------------------------------
def test_repeatable_and_image_independent():
    n_img, L, heads = 4, 1024, 5
    g = torch.Generator(device=DEV).manual_seed(6)
    qkv8 = _e4m3_randn(n_img * L, 3 * heads * 64, g)
    a, b = attn_fp8(qkv8, n_img, L, heads), attn_fp8(qkv8, n_img, L, heads)
    assert torch.equal(a, b)
    for i in range(n_img):
        one = attn_fp8(qkv8[i * L:(i + 1) * L].contiguous(), 1, L, heads)
        assert torch.equal(one, a[i * L:(i + 1) * L]), f"image {i} alone differs from image {i} of the batch"


def test_fp8_attn_sampler_step_repeatable_and_batch_invariant():
    from test_batch_gpu import _fused_step, _stage1_model
    torch.manual_seed(0)
    model = _stage1_model()
    net = model.model.diffusion_model
    net.set_precision("fp8_attn")
    B, T, h = 2, 16, 16
    g = torch.Generator().manual_seed(31)
    x = (torch.randn(B * T, 4, h, h, generator=g) * 8).to(DEV)
    c = dict(crossattn=torch.randn(B, 1, 1024, generator=g).to(DEV), vector=torch.randn(B, 768, generator=g).to(DEV),
             concat=(torch.randn(B * T, 4, h, h, generator=g) * 0.18).half().to(DEV))
    uc = dict(crossattn=torch.zeros_like(c["crossattn"]), vector=c["vector"].clone(), concat=torch.zeros_like(c["concat"]))
    sigma = torch.full((B * T,), 8.0, device=DEV)
    sigma_next = torch.full((B * T,), 6.5, device=DEV)
    xb, db = _fused_step(model, x, c, uc, sigma, sigma_next)
    assert all(p.fp8_attention for p in net._plans.values())
    xb2, db2 = _fused_step(model, x, c, uc, sigma, sigma_next)
    assert torch.isfinite(xb).all()
    assert torch.equal(xb, xb2) and torch.equal(db, db2), "two fp8_attn runs of the same batched step differ"
    model.sampler._fused.clear()
    s = slice(0, T)
    cb = {k: (v[s] if k == "concat" else v[0:1]).contiguous() for k, v in c.items()}
    ucb = {k: (v[s] if k == "concat" else v[0:1]).contiguous() for k, v in uc.items()}
    x1, d1 = _fused_step(model, x[s].contiguous(), cb, ucb, sigma[s].contiguous(), sigma_next[s].contiguous())
    assert torch.equal(xb[s], x1) and torch.equal(db[s], d1), "fp8_attn: object 0 alone differs from object 0 of a batch of two"


# ---- 7. plan -------------------------------------------------------------------------------------------------------------------
def _unet(seed=1):
    from test_fp8_gpu import _unet as unet
    return unet(seed)


def _spatial_blocks(net):
    return sorted(L.name + f"transformer_blocks.{d}." for blk in net.plan_desc.input_blocks + [net.plan_desc.middle] +
                  net.plan_desc.output_blocks for L in blk if L.kind == "attn" for d in range(net.cfg.transformer_depth))


def _check_plans(net, N, hw, T):
    net.set_precision("fp8")
    p8 = net.get_plan(N, hw, hw, T)
    layers8, n_attn8 = list(p8.fp8_layers), sum(getattr(s, "kind", "") == "spatial_attention" for s in p8.steps)
    assert p8.fp8_attention == [] and "vt" not in p8.arena.bufs and "qkv8" not in p8.arena.bufs
    del p8
    net.set_precision("fp8_attn")
    pa = net.get_plan(N, hw, hw, T)
    assert sorted(pa.fp8_attention) == _spatial_blocks(net) and len(set(pa.fp8_attention)) == len(pa.fp8_attention)
    assert pa.fp8_layers == layers8
    assert sum(getattr(s, "kind", "") == "spatial_attention" for s in pa.steps) == n_attn8 + len(pa.fp8_attention)
    assert sum(hasattr(s, "io") for s in pa.steps) == len(pa.fp8_attention)


def test_fp8_attn_plan_mc64():
    net, _ = _unet()
    _check_plans(net, 32, 32, 16)


@pytest.mark.parametrize("stage,hw", [(1, 64), (2, 128)])
def test_fp8_attn_plan_full_width(stage, hw):
    from hi3d_official_b200 import configs
    from hi3d_official_b200.unet import VideoUNet
    cfg = (configs.stage1_config() if stage == 1 else configs.stage2_config())["model"]["params"]["network_config"]["params"]
    net = VideoUNet(**cfg).cuda().half()
    spec.synth_fill_(net, seed=0, fast=True)
    _check_plans(net, 32, hw, 16)


# ---- 8. teacher-forced ---------------------------------------------------------------------------------------------------------
def test_fp8_attn_plan_teacher_forced():
    """The fp8_attn plan launch by launch: each spatial q|k|v is the fp8 GEMM's fp16 value rounded to e4m3, and each e4m3 attention
    step meets the kernel's bound on the plan's own q|k|v."""
    from test_fp8_gpu import _inputs, e4m3_ref
    net, _ = _unet()
    net.set_precision("fp8_attn")
    N, hw, T = 32, 32, 16
    x, ctx, y, t = _inputs(N, hw, T)
    net(x, timesteps=t, context=ctx, y=y, num_video_frames=T)
    plan = net.get_plan(N, hw, hw, T)
    n_qkv = n_attn = 0
    for s in plan.steps:
        s()
        if isinstance(s, ops.Gemm) and s.out.dtype == E4M3 and s.layers and s.layers[0].endswith("attn1.to_q"):
            segs, W, out, *_, ws = s._keep
            out16 = torch.empty(out.shape, dtype=torch.float16, device=DEV)
            ops.Gemm(segs, W, out16, s.p.M, w_scale=ws)()
            assert torch.equal(out[:s.p.M].view(torch.uint8), e4m3_ref(out16[:s.p.M]).view(torch.uint8)), s.layers[0]
            n_qkv += 1
        elif hasattr(s, "io"):
            qkv8, att, n_img, L, heads = s.io
            rows = torch.arange(0, L, max(1, L // 256), device=DEV)
            for img, h in ((0, 0), (n_img - 1, heads - 1)):
                ref, bound = reference_and_bound(qkv8.t, n_img, L, heads, 0.125, img, h, rows)
                _assert_within(att.t[img * L + rows, h * 64:(h + 1) * 64], ref, bound, f"{s.block} image {img} head {h}")
            n_attn += 1
    assert n_qkv == n_attn == len(plan.fp8_attention) > 0


# ---- 9. UNet -------------------------------------------------------------------------------------------------------------------
def test_fp8_attn_unet_vs_fp32_oracle():
    from test_fp8_gpu import _inputs, _rel
    net, sd = _unet()
    T, hw = 16, 32
    N = 2 * T
    x, ctx, y, t = _inputs(N, hw, T)
    ref = O.unet_forward(sd, x, t, ctx, y, num_video_frames=T)
    errs = {}
    for prec in ("fp8", "fp8_attn"):
        net.set_precision(prec)
        out = net(x, timesteps=t, context=ctx, y=y, num_video_frames=T)
        assert torch.isfinite(out).all()
        errs[prec] = _rel(out, ref)
    print(f"[fp8_attn unet mc=64 T={T} hw={hw}] rel L2 vs fp32 oracle: fp8 {errs['fp8']:.4e}  fp8_attn {errs['fp8_attn']:.4e}")
    assert errs["fp8_attn"] < 0.12


# ---- 10. end to end ------------------------------------------------------------------------------------------------------------
def _run(script, *args):
    r = subprocess.run([sys.executable, os.path.join(ROOT, script), *args], capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-1500:] + r.stderr[-3000:]
    return r.stdout


def test_pipelines_run_fp8_attn(tmp_path):
    out = str(tmp_path / "out")
    assert "first.mp4" in _run("pipeline_i2v_eval_v01.py", "--tiny", "--synthetic", "--precision", "fp8_attn", "--output_dir", out,
                               "--seed", "1")
    first = torch.load(os.path.join(out, "first_step", "first.pt"))
    assert first.shape == (16, 3, 128, 128) and torch.isfinite(first.float()).all()
    assert "second.mp4" in _run("pipeline_i2v_eval_v02.py", "--tiny", "--synthetic", "--precision", "fp8_attn", "--output_dir",
                                out, "--seed", "1")
    second = torch.load(os.path.join(out, "second_step_video", "second.pt"))
    assert second.shape == (16, 3, 256, 256) and torch.isfinite(second.float()).all()
