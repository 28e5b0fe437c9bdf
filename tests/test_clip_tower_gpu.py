"""CLIP image towers on the H100: the head-dim-80 attention kernel, the GELU / QuickGELU GEMM epilogues and the patch rows
against fp32 PyTorch, then the full-width OpenCLIP ViT-H/14 and OpenAI ViT-L/14 towers (and the aesthetic score) against the
fp32 oracle of tests/clip_oracle.py, the native stage-1 conditioner, and the stage-1 script starting from an image."""
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

import clip_oracle as CO  # noqa: E402
from hi3d_official_b200 import ops  # noqa: E402
from test_kernels_gpu import DEV, H, close, rnd  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def ref_attn80(qkv, n_img, L, heads, scale):
    C = heads * 80
    q, k, v = (t.view(n_img, L, heads, 80).transpose(1, 2).float() for t in qkv.view(n_img * L, 3, C).unbind(1))
    return (torch.softmax(q @ k.transpose(-1, -2) * scale, -1) @ v).transpose(1, 2).reshape(n_img * L, C)


@pytest.mark.parametrize("n_img", [1, 3])
@pytest.mark.parametrize("L", [1, 65, 128, 257, 1000])
def test_attention_d80(n_img, L):
    heads, scale = 2, 80 ** -0.5
    qkv = rnd(n_img * L, 3 * heads * 80, seed=L * 10 + n_img).to(H)
    out = torch.full((n_img * L, heads * 80), float("nan"), dtype=H, device=DEV)
    ops.attention_d80(qkv, n_img, L, heads, out, scale)
    close(out, ref_attn80(qkv, n_img, L, heads, scale), atol=2e-3, name=f"d80 L={L}")


def test_attention_d80_moving_max():
    """Scores that grow along the keys: the running maximum moves in every key tile, so the rescaling of O and l is
    exercised; a large scale also makes the softmax peaked (the fp16 P error scales with max |v|)."""
    n_img, L, heads, scale = 2, 257, 3, 3.0
    qkv = rnd(n_img * L, 3 * heads * 80, seed=7)
    C = heads * 80
    ramp = torch.linspace(-2, 2, L, device=DEV).repeat(n_img)[:, None]
    qkv[:, C:2 * C] += ramp                                   # k grows with the key index
    qkv[:, :C] = qkv[:, :C].abs() * 0.5 + 0.5                 # q > 0: q . k grows as well
    qkv = qkv.to(H)
    out = torch.zeros(n_img * L, C, dtype=H, device=DEV)
    ops.attention_d80(qkv, n_img, L, heads, out, scale)
    close(out, ref_attn80(qkv, n_img, L, heads, scale), atol=2e-3 * scale, name="d80 moving max")


@pytest.mark.parametrize("engine", ["tc5", "mma"])
@pytest.mark.parametrize("act", ["gelu", "quickgelu"])
@pytest.mark.parametrize("n,N,K", [(1, 256, 128), (3, 512, 256), (2, 64, 192)])
def test_gemm_clip_activations(engine, act, n, N, K):
    M = 257 * n
    a, w, b = rnd(M, K, seed=1).to(H), rnd(N, K, scale=K ** -0.5, seed=2).to(H), rnd(N, scale=0.5, seed=3)
    res = rnd(M, N, seed=4).to(H)
    out = torch.zeros(M, N, dtype=H, device=DEV)
    code = ops.ACT_GELU if act == "gelu" else ops.ACT_QUICKGELU
    ops.Gemm([ops.SegSpec(a)], w, out, M, bias=b, act=code, residual=res, engine=engine)()
    y = a.float() @ w.float().t() + b
    y = F.gelu(y) if act == "gelu" else y * torch.sigmoid(1.702 * y)
    close(out, y.half().float() + res.float(), name=f"{engine} {act}")


def test_gemm_clip_activations_engines_agree():
    M, N, K = 257 * 2, 384, 320
    a, w = rnd(M, K, seed=5).to(H), rnd(N, K, scale=K ** -0.5, seed=6).to(H)
    for act in (ops.ACT_GELU, ops.ACT_QUICKGELU):
        o1, o2 = (torch.zeros(M, N, dtype=H, device=DEV) for _ in range(2))
        ops.Gemm([ops.SegSpec(a)], w, o1, M, act=act, engine="tc5")()
        ops.Gemm([ops.SegSpec(a)], w, o2, M, act=act, engine="mma")()
        close(o1, o2, atol=4e-3, name=f"tc5 vs mma act {act}")


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("normalize", [True, False])
def test_clip_patchify(dtype, normalize):
    n, patch, kpad = 2, 14, 640
    img = rnd(n, 3, 224, 224, seed=9).to(dtype)
    out = torch.full((n * 257, kpad), float("nan"), dtype=H, device=DEV)
    ops.clip_patchify(img, patch, out, normalize=normalize)
    x = img.float()
    if normalize:
        x = (x - torch.tensor(CO.CLIP_MEAN, device=DEV).view(1, 3, 1, 1)) / torch.tensor(CO.CLIP_STD, device=DEV).view(1, 3, 1, 1)
    p = x.reshape(n, 3, 16, patch, 16, patch).permute(0, 2, 4, 1, 3, 5).reshape(n, 256, 3 * patch * patch)
    ref = torch.zeros(n, 257, kpad, device=DEV)
    ref[:, 1:, :588] = p
    close(out.view(n, 257, kpad), ref.half().float(), atol=1e-6, rtol=1e-3, name="patchify")


# ---- full-width towers against the fp32 oracle (SURVEY §8c: our fp16 error <= 2x the oracle's own error under autocast) ----
TOWERS = {"vit_h14": dict(width=1280, layers=32, head_width=80, out_dim=1024, quick_gelu=False),
          "vit_l14": dict(width=1024, layers=24, head_width=64, out_dim=768, quick_gelu=True)}


def _images(n, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(n, 3, 224, 224, generator=g).to(DEV)


def _tower_errors(cfg, seed, n=4):
    from hi3d_official_b200.clip_vision import ClipVisionTower
    sd = CO.random_visual_sd(cfg["width"], cfg["layers"], cfg["head_width"], cfg["out_dim"], seed=seed, device=DEV)
    img = _images(n, seed + 1)
    xn = CO.normalize(img)
    ref = CO.vision_forward(sd, xn, cfg["head_width"], cfg["quick_gelu"])
    with torch.autocast("cuda", dtype=torch.float16):
        amp = CO.vision_forward(sd, xn, cfg["head_width"], cfg["quick_gelu"]).float()
    got = ClipVisionTower(sd, cfg["head_width"], cfg["quick_gelu"], device=DEV)(img)
    return sd, xn, ref, amp, got


@pytest.mark.parametrize("name", list(TOWERS))
def test_tower_full_width(name):
    _, _, ref, amp, got = _tower_errors(TOWERS[name], seed=11)
    e, e_amp = CO.relerr(got, ref), CO.relerr(amp, ref)
    print(f"{name}: rel-L2 error native {e:.3e}, oracle under autocast {e_amp:.3e}, ratio {e / e_amp:.2f}")
    assert e <= 2 * e_amp, f"{name}: native error {e:.3e} > 2 x autocast error {e_amp:.3e}"


def test_aesthetic_score_full_width():
    """The score enters `vector` as timestep_embedding(100 * score): its error is the one that matters."""
    from hi3d_official_b200.clip_vision import AestheticScorer, fold_linear_chain
    cfg = TOWERS["vit_l14"]
    sd, xn, ref_f, amp_f, _ = _tower_errors(cfg, seed=21, n=8)
    mlp = {k: v.to(DEV) for k, v in CO.random_aesthetic_mlp(seed=22).items()}
    score = lambda f: CO.aesthetic_mlp(mlp, f / f.norm(dim=-1, keepdim=True))   # noqa: E731
    ref, amp = score(ref_f), score(amp_f)
    w, b = fold_linear_chain(mlp)
    got = AestheticScorer(sd, w, b, device=DEV)(xn)
    e, e_amp = float((got - ref).abs().max()), float((amp - ref).abs().max())
    print(f"aesthetic score: max abs error native {e:.3e}, oracle under autocast {e_amp:.3e} (x100 in the embedding: "
          f"{100 * e:.3e}), score range {float(ref.min()):.3f} .. {float(ref.max()):.3f}")
    assert e <= 2 * e_amp + 1e-5, f"aesthetic score: native error {e:.3e} > 2 x autocast error {e_amp:.3e}"


# ---- the stage-1 conditioner and script with native towers (reduced-width tower weights) ----------------------------------
def _small_towers(seed):
    vh = CO.random_visual_sd(320, 2, 80, 1024, seed=seed)           # ViT-H style: 4 heads of 80, GELU, -> crossattn 1024
    vl = CO.random_visual_sd(128, 2, 64, 768, seed=seed + 1)        # ViT-L style: 2 heads of 64, QuickGELU, -> 768 features
    return vh, vl, CO.random_aesthetic_mlp(seed=seed + 2)


def test_stage1_conditioning_native_vs_oracle():
    import pipeline_i2v_eval_v01 as P1
    from hi3d_official_b200 import conditioner as cond
    model = P1.load_model("none.yaml", "none.pt", 1, tiny=True)
    emb = model.conditioner.embedders
    i_clip = next(i for i, e in enumerate(emb) if isinstance(e, cond.FrozenOpenCLIPImagePredictionEmbedder))
    i_aes = next(i for i, e in enumerate(emb) if isinstance(e, cond.AesEmbedder))
    vh, vl, mlp = _small_towers(31)
    sd = {f"conditioner.embedders.{i_clip}.open_clip.model.visual.{k}": v for k, v in vh.items()}
    sd.update({f"conditioner.embedders.{i_aes}.aesthetic_model.visual.{k}": v for k, v in vl.items()})
    sd.update({f"conditioner.embedders.{i_aes}.aesthetic_mlp.{k}": v for k, v in mlp.items()})
    assert sorted(model.conditioner.load_tower_weights(sd)) == ["aes", "clip"]
    T = model.num_samples
    g = torch.Generator().manual_seed(32)
    img = (torch.rand(3, 128, 128, generator=g) * 2 - 1).to(DEV)
    frames = img[:, None].repeat(1, T, 1, 1)
    # oracle tower outputs on the very inputs the conditioner's towers see
    x_clip = frames[None][:, :, 0].half().float()
    clip_ref = CO.openclip_embed({k: v.to(DEV) for k, v in vh.items()}, x_clip)
    x_aes = emb[i_aes].preprocess(frames[None])
    aes_ref = CO.aesthetic_score({k: v.to(DEV) for k, v in vl.items()}, {k: v.to(DEV) for k, v in mlp.items()}, x_aes)
    torch.manual_seed(5)
    c, uc = P1.cond_from_towers(model, frames, None, 10, 1)
    torch.manual_seed(5)
    c_ref, uc_ref = P1.cond_from_towers(model, frames, {"clip": clip_ref, "aes": aes_ref}, 10, 1)
    e_clip = CO.relerr(c["crossattn"].float(), c_ref["crossattn"].float())
    d_score = float((c["vector"][:, 0] - c_ref["vector"][:, 0]).abs().max())
    print(f"stage-1 conditioning: crossattn rel-L2 {e_clip:.2e}; aesthetic score {float(aes_ref):.4f}, abs error {d_score:.2e}")
    assert e_clip < 1e-2
    assert d_score < 2e-3
    torch.testing.assert_close(c["vector"][:, 256:], c_ref["vector"][:, 256:])          # elevation / cond_aug embeddings
    torch.testing.assert_close(c["vector"][:, 1:256], cond.timestep_embedding(c["vector"][:, 0] * 100, 255), atol=2e-3, rtol=0)
    # the cond-frame latent does not involve the towers; the VAE's GroupNorm statistics are summed with atomics, so two runs
    # may differ in the last fp16 bit
    torch.testing.assert_close(c["concat"].float(), c_ref["concat"].float(), atol=1e-2, rtol=1e-2)
    assert torch.count_nonzero(uc["crossattn"]) == 0 and torch.count_nonzero(uc["concat"]) == 0
    torch.testing.assert_close(uc["vector"], c["vector"])


def test_stage1_script_from_image_with_native_towers(tmp_path):
    import cv2
    import numpy as np
    from test_clip_tower_cpu import _Archive
    vh, vl, mlp = _small_towers(41)
    os.makedirs(tmp_path / "ckpts" / "metric_models")
    bin_sd = {"visual." + k: v for k, v in vh.items()}
    bin_sd["text_projection"] = torch.zeros(8, 8)                    # text-tower keys are ignored
    torch.save(bin_sd, tmp_path / "ckpts" / "open_clip_pytorch_model.bin")
    torch.jit.trace(_Archive({"visual." + k: v.half() for k, v in vl.items()}), torch.ones(2)).save(
        str(tmp_path / "ckpts" / "ViT-L-14.pt"))
    torch.save(mlp, tmp_path / "ckpts" / "metric_models" / "sac+logos+ava1-l14-linearMSE.pth")
    img = (np.random.default_rng(0).random((160, 200, 3)) * 255).astype(np.uint8)
    cv2.imwrite(str(tmp_path / "in.png"), img)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "pipeline_i2v_eval_v01.py"), "--tiny", "--seed", "0",
                        "--image_path", "in.png", "--output_dir", "out"], capture_output=True, text=True, timeout=900,
                       cwd=str(tmp_path))
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    assert os.path.getsize(tmp_path / "out" / "first_step" / "first.mp4") > 0
    frames = torch.load(tmp_path / "out" / "first_step" / "first.pt")
    assert frames.shape[0] == 16 and bool(torch.isfinite(frames.float()).all())
