"""CLIP image towers, host side: the fp32 oracle against `transformers`' CLIPVisionModelWithProjection, the kornia resize
restatement, the three checkpoint readers and the aesthetic-MLP folding, and the conditioner's behaviour without weights."""
import os

import pytest
import torch
import torch.nn as nn

import clip_oracle as CO
from hi3d_official_b200 import clip_vision as CV
from hi3d_official_b200 import conditioner as cond


# ---- oracle vs transformers -----------------------------------------------------------------------------------------------
def _hf_from_visual(sd, head_width, act, out_dim):
    transformers = pytest.importorskip("transformers")
    width, _, patch, _ = sd["conv1.weight"].shape
    layers = len({k.split(".")[2] for k in sd if k.startswith("transformer.resblocks.")})
    grid = int(round((sd["positional_embedding"].shape[0] - 1) ** 0.5))
    cfg = transformers.CLIPVisionConfig(hidden_size=width, intermediate_size=sd["transformer.resblocks.0.mlp.c_fc.weight"].shape[0],
                                        num_hidden_layers=layers, num_attention_heads=width // head_width,
                                        image_size=grid * patch, patch_size=patch, hidden_act=act, projection_dim=out_dim,
                                        layer_norm_eps=1e-5)
    m = transformers.CLIPVisionModelWithProjection(cfg).eval()
    hs = {"vision_model.embeddings.class_embedding": sd["class_embedding"],
          "vision_model.embeddings.patch_embedding.weight": sd["conv1.weight"],
          "vision_model.embeddings.position_embedding.weight": sd["positional_embedding"],
          "vision_model.pre_layrnorm.weight": sd["ln_pre.weight"], "vision_model.pre_layrnorm.bias": sd["ln_pre.bias"],
          "vision_model.post_layernorm.weight": sd["ln_post.weight"], "vision_model.post_layernorm.bias": sd["ln_post.bias"],
          "visual_projection.weight": sd["proj"].t()}
    for i in range(layers):
        p, q = f"transformer.resblocks.{i}.", f"vision_model.encoder.layers.{i}."
        for n, w, b in zip(("q_proj", "k_proj", "v_proj"), sd[p + "attn.in_proj_weight"].chunk(3), sd[p + "attn.in_proj_bias"].chunk(3)):
            hs[q + f"self_attn.{n}.weight"], hs[q + f"self_attn.{n}.bias"] = w, b
        hs.update({q + "self_attn.out_proj.weight": sd[p + "attn.out_proj.weight"], q + "self_attn.out_proj.bias": sd[p + "attn.out_proj.bias"],
                   q + "layer_norm1.weight": sd[p + "ln_1.weight"], q + "layer_norm1.bias": sd[p + "ln_1.bias"],
                   q + "layer_norm2.weight": sd[p + "ln_2.weight"], q + "layer_norm2.bias": sd[p + "ln_2.bias"],
                   q + "mlp.fc1.weight": sd[p + "mlp.c_fc.weight"], q + "mlp.fc1.bias": sd[p + "mlp.c_fc.bias"],
                   q + "mlp.fc2.weight": sd[p + "mlp.c_proj.weight"], q + "mlp.fc2.bias": sd[p + "mlp.c_proj.bias"]})
    missing, unexpected = m.load_state_dict(hs, strict=False)
    assert not unexpected and all("position_ids" in k for k in missing), (missing, unexpected)
    return m


@pytest.mark.parametrize("head_width,act,quick", [(80, "gelu", False), (64, "quick_gelu", True)],
                         ids=["vit_h_style", "vit_l_style"])
def test_oracle_matches_transformers(head_width, act, quick):
    sd = CO.random_visual_sd(head_width * 4, 2, head_width, 96, patch=14, grid=4, seed=3)
    m = _hf_from_visual(sd, head_width, act, 96)
    x = torch.randn(2, 3, 56, 56, generator=torch.Generator().manual_seed(4))
    with torch.no_grad():
        ref = m(pixel_values=x).image_embeds
    got = CO.vision_forward(sd, x, head_width, quick)
    torch.testing.assert_close(got, ref, rtol=1e-4, atol=1e-4)


# ---- kornia resize ----------------------------------------------------------------------------------------------------------
def test_resize_blur_taps_downscale():
    """512 -> 224: sigma = (512/224 - 1)/2 = 0.643, kernel 3, taps [0.187, 0.626, 0.187]."""
    sig = (512 / 224 - 1) / 2
    assert abs(sig - 0.643) < 1e-3
    taps = CO.gaussian_kernel1d(3, sig)
    torch.testing.assert_close(taps, torch.tensor([0.187, 0.626, 0.187]), atol=1e-3, rtol=0)
    x = torch.randn(1, 3, 512, 512, generator=torch.Generator().manual_seed(0))
    k = taps[:, None] * taps[None, :]
    xp = torch.nn.functional.pad(x, (1, 1, 1, 1), mode="reflect")
    blurred = torch.nn.functional.conv2d(xp, k.expand(3, 1, 3, 3), groups=3)
    ref = torch.nn.functional.interpolate(blurred, size=(224, 224), mode="bicubic", align_corners=True)
    torch.testing.assert_close(CO.kornia_resize(x), ref, atol=1e-5, rtol=1e-5)
    torch.testing.assert_close(CV.kornia_resize(x), ref, atol=1e-5, rtol=1e-5)


def test_resize_upscale_is_plain_bicubic():
    x = torch.randn(2, 3, 128, 160, generator=torch.Generator().manual_seed(1))
    ref = torch.nn.functional.interpolate(x, size=(224, 224), mode="bicubic", align_corners=True)
    torch.testing.assert_close(CV.kornia_resize(x), ref)
    torch.testing.assert_close(CO.kornia_resize(x), ref)
    assert CV.kornia_resize(torch.ones(1, 3, 224, 224)) is not None


def test_openclip_preprocess_range():
    x = torch.rand(1, 3, 320, 320) * 2 - 1
    y = CV.openclip_preprocess(x)
    torch.testing.assert_close(y, (CO.kornia_resize(x) + 1) / 2, atol=1e-5, rtol=1e-5)


# ---- checkpoint readers ----------------------------------------------------------------------------------------------------
def _small_visual(seed=0):
    return CO.random_visual_sd(128, 1, 64, 64, patch=14, grid=2, seed=seed)


def test_load_open_clip_bin(tmp_path):
    vis = _small_visual()
    sd = {"visual." + k: v for k, v in vis.items()}
    sd.update({"transformer.resblocks.0.attn.in_proj_weight": torch.zeros(3), "token_embedding.weight": torch.zeros(4, 2),
               "text_projection": torch.zeros(2, 2), "logit_scale": torch.tensor(1.0)})
    for i, wrap in enumerate((lambda d: d, lambda d: {"state_dict": {"module." + k: v for k, v in d.items()}})):
        p = tmp_path / f"open_clip_{i}.bin"
        torch.save(wrap(sd), p)
        got = CV.load_open_clip(str(p))
        assert set(got) == set(vis)
        for k in vis:
            assert torch.equal(got[k], vis[k])


def _module_tree(sd):
    root = nn.Module()
    for k, v in sd.items():
        *path, leaf = k.split(".")
        m = root
        for name in path:
            if not hasattr(m, name):
                m.add_module(name, nn.Module())
            m = getattr(m, name)
        m.register_parameter(leaf, nn.Parameter(v.clone(), requires_grad=False))
    return root


class _Archive(nn.Module):
    def __init__(self, sd):
        super().__init__()
        tree = _module_tree(sd)
        for name, child in tree.named_children():
            self.add_module(name, child)
        self.logit_scale = nn.Parameter(torch.tensor(4.6), requires_grad=False)

    def forward(self, x):
        return x * self.logit_scale


def test_load_openai_torchscript(tmp_path):
    vis = {k: v.half() for k, v in _small_visual(1).items()}
    sd = {"visual." + k: v for k, v in vis.items()}
    sd["transformer.resblocks.0.attn.in_proj_weight"] = torch.zeros(6, 2)
    traced = torch.jit.trace(_Archive(sd), torch.ones(2))
    p = tmp_path / "ViT-L-14.pt"
    traced.save(str(p))
    got = CV.load_openai_clip(str(p))
    assert set(got) == set(vis)
    for k in vis:
        assert torch.equal(got[k], vis[k])
    p2 = tmp_path / "plain.pt"                               # a plain state dict is read with torch.load
    torch.save(sd, p2)
    assert set(CV.load_openai_clip(str(p2))) == set(vis)


def test_aesthetic_mlp_fold(tmp_path):
    mlp = CO.random_aesthetic_mlp(seed=5)
    p = tmp_path / "sac+logos+ava1-l14-linearMSE.pth"
    torch.save(mlp, p)
    w, b = CV.load_aesthetic_mlp(str(p))
    assert w.shape == (768,) and w.dtype == torch.float32 and b.dim() == 0
    x = torch.randn(16, 768, generator=torch.Generator().manual_seed(6))
    x = x / x.norm(dim=-1, keepdim=True)
    ref = CO.aesthetic_mlp(mlp, x.double()).float()[:, 0]
    torch.testing.assert_close(x @ w + b, ref, atol=1e-5, rtol=1e-5)


# ---- conditioner without weights ------------------------------------------------------------------------------------------
def test_towers_without_weights_behave_as_before(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)                              # no ckpts/ here
    emb = cond.FrozenOpenCLIPImageEmbedder(version=str(tmp_path / "missing.bin"), freeze=True)
    assert emb.native() is None and len(list(emb.parameters())) == 0
    with pytest.raises(NotImplementedError):
        emb(torch.zeros(1, 3, 8, 8))
    emb.set_fn(lambda x: torch.ones(x.shape[0], 1024))
    assert emb(torch.zeros(2, 3, 8, 8)).shape == (2, 1024)
    aes = cond.AesEmbedder()
    assert aes.scorer.native() is None and len(list(aes.parameters())) == 0
    with pytest.raises(NotImplementedError):
        aes(torch.zeros(1, 3, 3, 16, 16))
    aes.scorer.set_fn(lambda x: torch.full((x.shape[0], 1), 0.5))
    assert aes(torch.zeros(1, 3, 3, 16, 16)).shape == (1, 256)


def test_towers_weights_from_checkpoint_keys(tmp_path, monkeypatch):
    """load_tower_weights routes the reference's module paths; pre-computed batch entries still take precedence."""
    monkeypatch.chdir(tmp_path)
    c = cond.GeneralConditioner([
        {"target": "sgm.modules.encoders.modules.FrozenOpenCLIPImagePredictionEmbedder", "input_key": "cond_frames_without_noise",
         "params": {"n_cond_frames": 1, "n_copies": 1, "open_clip_embedding_config": {
             "target": "sgm.modules.encoders.modules.FrozenOpenCLIPImageEmbedder", "params": {"version": "none.bin"}}}},
        {"target": "vtdm.encoders.AesEmbedder", "input_key": "video"}])
    assert c.missing_towers() == ["clip", "aes"]
    vis = _small_visual(2)
    sd = {f"conditioner.embedders.0.open_clip.model.visual.{k}": v for k, v in vis.items()}
    sd.update({f"conditioner.embedders.1.aesthetic_model.visual.{k}": v for k, v in vis.items()})
    assert c.load_tower_weights(sd) == ["clip", "aes"]
    assert c.missing_towers() == ["aes"]                    # the aesthetic MLP is still missing
    sd = {f"conditioner.embedders.1.aesthetic_mlp.{k}": v for k, v in CO.random_aesthetic_mlp(seed=1).items()}
    assert c.load_tower_weights(sd) == ["aes"]
    assert c.missing_towers() == []
    pre = torch.full((1, 1024), 0.25)
    out = c({"cond_frames_without_noise": torch.zeros(1, 3, 8, 8), "cond_frames_without_noise:clip": pre,
             "video": torch.zeros(1, 3, 3, 8, 8), "video:aes": torch.tensor([[0.5]])})
    assert torch.equal(out["crossattn"], pre[:, None])
    assert float(out["vector"][0, 0]) == 0.5


def test_tower_files_in_working_directory(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    os.makedirs("ckpts/metric_models")
    vis = _small_visual(3)
    torch.save({"visual." + k: v for k, v in vis.items()}, "ckpts/open_clip_pytorch_model.bin")
    torch.jit.trace(_Archive({"visual." + k: v for k, v in vis.items()}), torch.ones(2)).save("ckpts/ViT-L-14.pt")
    torch.save(CO.random_aesthetic_mlp(dim=64, seed=2), "ckpts/metric_models/sac+logos+ava1-l14-linearMSE.pth")
    emb = cond.FrozenOpenCLIPImageEmbedder(version="ckpts/open_clip_pytorch_model.bin")
    aes = cond.AesEmbedder()
    assert emb.native() is not None and aes.scorer.native() is not None
