"""MiDaS DPT-Hybrid depth tower, host side: the fp32 oracle against `transformers`' DPTForDepthEstimation (hybrid), the loader of
the reference's checkpoint file, checkpoint-key routing in the conditioner, and the depth tower's behaviour without weights."""
import os

import pytest
import torch

import midas_oracle as MO
from hi3d_official_b200 import conditioner as cond
from hi3d_official_b200 import midas


# ---- oracle vs transformers -----------------------------------------------------------------------------------------------
def _hf_key(k):
    """The reference's key -> transformers' DPT hybrid key (None: not in transformers' model)."""
    r = [(MO.BB + "stem.conv.", "dpt.embeddings.backbone.bit.embedder.convolution."),
         (MO.BB + "stem.norm.", "dpt.embeddings.backbone.bit.embedder.norm."),
         (MO.BB + "stages.", "dpt.embeddings.backbone.bit.encoder.stages."),
         (MO.VIT + "patch_embed.proj.", "dpt.embeddings.projection."),
         (MO.VIT + "cls_token", "dpt.embeddings.cls_token"), (MO.VIT + "pos_embed", "dpt.embeddings.position_embeddings"),
         (MO.VIT + "norm.", "dpt.layernorm."),
         ("pretrained.act_postprocess3.0.project.", "neck.reassemble_stage.readout_projects.2."),
         ("pretrained.act_postprocess4.0.project.", "neck.reassemble_stage.readout_projects.3."),
         ("pretrained.act_postprocess3.3.", "neck.reassemble_stage.layers.2.projection."),
         ("pretrained.act_postprocess4.3.", "neck.reassemble_stage.layers.3.projection."),
         ("pretrained.act_postprocess4.4.", "neck.reassemble_stage.layers.3.resize."),
         ("scratch.output_conv.", "head.head.")]
    if k.startswith(MO.VIT + "head."):
        return None
    for a, b in r:
        if k.startswith(a):
            return (b + k[len(a):]).replace(".blocks.", ".layers.")
    if k.startswith(MO.VIT + "blocks."):
        i, rest = k[len(MO.VIT + "blocks."):].split(".", 1)
        rest = {"norm1.weight": "layernorm_before.weight", "norm1.bias": "layernorm_before.bias",
                "norm2.weight": "layernorm_after.weight", "norm2.bias": "layernorm_after.bias",
                "attn.proj.weight": "attention.output.dense.weight", "attn.proj.bias": "attention.output.dense.bias",
                "mlp.fc1.weight": "intermediate.dense.weight", "mlp.fc1.bias": "intermediate.dense.bias",
                "mlp.fc2.weight": "output.dense.weight", "mlp.fc2.bias": "output.dense.bias"}.get(rest, rest)
        return f"dpt.encoder.layer.{i}.{rest}"
    if k.startswith("scratch.layer"):
        i = int(k[len("scratch.layer")])
        return f"neck.convs.{i - 1}.weight"
    if k.startswith("scratch.refinenet"):
        i, rest = k[len("scratch.refinenet"):].split(".", 1)
        rest = rest.replace("resConfUnit1.", "residual_layer1.").replace("resConfUnit2.", "residual_layer2.")
        rest = rest.replace("conv1.", "convolution1.").replace("conv2.", "convolution2.").replace("out_conv.", "projection.")
        return f"neck.fusion_stage.layers.{4 - int(i)}.{rest}"
    raise KeyError(k)


def _hf_model(sd):
    transformers = pytest.importorskip("transformers")
    cfg = transformers.DPTConfig(
        is_hybrid=True, image_size=384, hidden_size=768, num_hidden_layers=12, num_attention_heads=12, intermediate_size=3072,
        layer_norm_eps=1e-6, readout_type="project", backbone_out_indices=[2, 5, 8, 11], neck_hidden_sizes=[256, 512, 768, 768],
        reassemble_factors=[1, 1, 1, 0.5], fusion_hidden_size=256, neck_ignore_stages=[0, 1], head_in_index=-1,
        use_batch_norm_in_fusion_residual=False,
        backbone_config=dict(model_type="bit", global_padding="same", layer_type="bottleneck", depths=[3, 4, 9],
                             hidden_sizes=[256, 512, 1024], embedding_dynamic_padding=True,
                             out_features=["stage1", "stage2", "stage3"]))
    m = transformers.DPTForDepthEstimation(cfg).eval()
    hs = {}
    for k, v in sd.items():
        hk = _hf_key(k)
        if hk is None:
            continue
        if ".attn.qkv." in hk:
            base, leaf = hk.rsplit(".attn.qkv.", 1)
            for name, t in zip(("query", "key", "value"), v.chunk(3)):
                hs[f"{base}.attention.attention.{name}.{leaf}"] = t
        else:
            hs[hk] = v
    missing, unexpected = m.load_state_dict(hs, strict=False)
    assert not unexpected and not missing, (missing, unexpected)
    return m


@pytest.mark.parametrize("dtype,tol", [(torch.float64, 1e-10), (torch.float32, 1e-4)], ids=["fp64", "fp32"])
def test_oracle_matches_transformers(dtype, tol):
    """Full-size random weights at 384^2.  In fp64 the two agree to 1e-13, so the fp32 difference (~3e-5 over 16 bottlenecks,
    12 blocks and the unnormalised fusion path) is round-off."""
    sd = {k: v.to(dtype) for k, v in MO.random_dpt_hybrid_sd(seed=1, **MO.FULL).items()}
    m = _hf_model(sd).to(dtype)
    x = (torch.rand(2, 3, 384, 384, generator=torch.Generator().manual_seed(2)) * 2 - 1).to(dtype)
    with torch.no_grad():
        ref = m(pixel_values=x).predicted_depth
        got = MO.dpt_forward(sd, x)
    assert ref.shape == got.shape == (2, 384, 384)
    e = MO.relerr(got, ref)
    print(f"oracle vs transformers ({dtype}): rel-L2 {e:.2e}; depth range {float(ref.min()):.3f} .. {float(ref.max()):.3f}, "
          f"{float((ref == 0).float().mean()):.1%} zeros")
    assert e < tol
    # random weights give a varied map: not a constant, and not mostly zeroed by the final ReLU
    assert float(ref.std()) > 0.1 * float(ref.abs().mean()) and float((ref == 0).float().mean()) < 0.1


def test_oracle_pos_embed_resize():
    """vit.py:104-121 at a non-384 size: the 24 x 24 grid is resized bilinearly, the class row is kept."""
    pos = torch.randn(1, 1 + 24 * 24, 8, generator=torch.Generator().manual_seed(3))
    got = MO.resize_pos_embed(pos, 6, 4)
    assert got.shape == (1, 25, 8)
    torch.testing.assert_close(got[:, 0], pos[:, 0])
    grid = pos[0, 1:].reshape(24, 24, 8).permute(2, 0, 1)[None]
    ref = torch.nn.functional.interpolate(grid, size=(6, 4), mode="bilinear", align_corners=False)
    torch.testing.assert_close(got[0, 1:], ref[0].permute(1, 2, 0).reshape(24, 8))
    torch.testing.assert_close(MO.resize_pos_embed(pos, 24, 24), pos)
    torch.testing.assert_close(midas.resize_pos_embed(pos[0], 6, 4), got[0])


# ---- the checkpoint loader ---------------------------------------------------------------------------------------------------
def test_load_plain_and_wrapped(tmp_path):
    sd = MO.random_dpt_hybrid_sd(seed=4, **MO.SMALL)
    live = {k for k in sd if k not in midas.dead_keys(sd)}
    assert not any(k.startswith(("pretrained.model.norm.", "pretrained.model.head.", "scratch.refinenet4.resConfUnit1."))
                   for k in live)
    for i, wrap in enumerate((lambda d: d, lambda d: {"model": d, "optimizer": {"state": {}}})):
        p = tmp_path / f"dpt_hybrid_{i}.pt"
        torch.save(wrap(sd), p)
        got = midas.load_dpt_hybrid(str(p))
        assert set(got) == live
        for k in live:
            assert torch.equal(got[k], sd[k])


def test_load_rejects_missing_and_unknown(tmp_path):
    sd = MO.random_dpt_hybrid_sd(seed=5, **MO.SMALL)
    for drop in ("scratch.output_conv.4.bias", MO.BB + "stages.1.blocks.0.downsample.norm.weight",
                 "pretrained.model.blocks.11.mlp.fc2.weight", "pretrained.act_postprocess4.4.weight"):
        bad = {k: v for k, v in sd.items() if k != drop}
        torch.save(bad, tmp_path / "bad.pt")
        with pytest.raises(KeyError, match="missing"):
            midas.load_dpt_hybrid(str(tmp_path / "bad.pt"))
    torch.save(dict(sd, **{"pretrained.model.dist_token": torch.zeros(1, 1, 128)}), tmp_path / "extra.pt")
    with pytest.raises(KeyError, match="unexpected"):
        midas.load_dpt_hybrid(str(tmp_path / "extra.pt"))
    torch.save({k: v for k, v in sd.items() if not k.startswith(("pretrained.model.norm.", "pretrained.model.head."))},
               tmp_path / "no_dead.pt")
    assert set(midas.load_dpt_hybrid(str(tmp_path / "no_dead.pt"))) == {k for k in sd if k not in midas.dead_keys(sd)}


def test_tower_rejects_bad_state_dict_and_input():
    sd = MO.random_dpt_hybrid_sd(seed=6, **MO.SMALL)
    with pytest.raises(KeyError):
        midas.DPTHybridTower({k: v for k, v in sd.items() if k != "scratch.layer3_rn.weight"}, device="cpu")
    tower = midas.DPTHybridTower(sd, device="cpu")                    # packing only; nothing runs on the CPU
    assert (tower.width, tower.heads, tower.features) == (128, 2, 128)
    assert [len(s) for s in tower.stages] == [1, 1, 1]
    for shape in ((2, 3, 96, 100), (2, 1, 96, 96), (3, 96, 96)):
        with pytest.raises(ValueError):
            tower(torch.zeros(shape))


# ---- the conditioner ---------------------------------------------------------------------------------------------------------
def test_depth_without_weights_behaves_as_before(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)                              # no ckpts/ here
    emb = cond.DepthEmbedder()
    assert emb.model.native() is None and len(list(emb.parameters())) == 0
    with pytest.raises(NotImplementedError):
        emb(torch.zeros(16, 3, 256, 256))
    seen = []
    emb.model.set_fn(lambda x: seen.append(tuple(x.shape)) or x[:, 0] * 0 + torch.linspace(0, 1, x.shape[-1]))
    y = emb(torch.zeros(16, 3, 256, 256))
    assert seen == [(16, 3, 96, 96)] and y.shape == (16, 9, 32, 32)
    c = cond.GeneralConditioner([{"target": "vtdm.encoders.DepthEmbedder", "input_key": "cond_frames"}])
    assert c.missing_towers() == ["depth"]


def test_depth_weights_from_checkpoint_keys(tmp_path, monkeypatch):
    """load_tower_weights routes conditioner.embedders.N.model.model.*; a batch `cond_frames:depth` still comes first."""
    monkeypatch.chdir(tmp_path)
    c = cond.GeneralConditioner([{"target": "vtdm.encoders.DepthEmbedder", "input_key": "cond_frames"}])
    sd = MO.random_dpt_hybrid_sd(seed=7, **MO.SMALL)
    full = {f"conditioner.embedders.0.model.model.{k}": v for k, v in sd.items()}
    full["model.diffusion_model.x"] = torch.zeros(1)
    assert c.load_tower_weights(full) == ["depth"]
    assert c.missing_towers() == []
    assert set(c.embedders[0].model._sd) == {k for k in sd if k not in midas.dead_keys(sd)}
    pre = torch.rand(16, 24, 24)
    x = torch.zeros(16, 3, 64, 64)
    out = c({"cond_frames": x, "cond_frames:depth": pre})
    torch.testing.assert_close(out["concat"], cond.depth_to_concat(pre, 64, 64, 3))
    bad = {k: v for k, v in full.items() if not k.endswith("output_conv.4.bias")}
    with pytest.raises(KeyError):
        cond.GeneralConditioner([{"target": "vtdm.encoders.DepthEmbedder", "input_key": "cond_frames"}]).load_tower_weights(bad)


def test_depth_file_in_working_directory(tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    os.makedirs("ckpts")
    torch.save({"model": MO.random_dpt_hybrid_sd(seed=8, **MO.SMALL), "optimizer": {}}, "ckpts/dpt_hybrid_384.pt")
    emb = cond.DepthEmbedder()
    assert emb.model.native() is not None and len(list(emb.parameters())) == 0
