"""Config / plugin glue: the reference's drop-in seam is `target:` strings resolved by
`sgm.util.instantiate_from_config` / `get_obj_from_str` (sgm/util.py:168-185).  The same functions here resolve
the *unmodified* strings of configs/inference-v0{1,2}.yaml to the H100 classes of this package."""
from __future__ import annotations

import importlib
from typing import Any, Dict

import torch

# reference target string -> (module in this package, attribute)
TARGET_ALIASES: Dict[str, str] = {
    "sgm.modules.diffusionmodules.video_model.VideoUNet": "hi3d_official_b200.unet.VideoUNet",
    "sgm.modules.diffusionmodules.wrappers.OpenAIWrapper": "hi3d_official_b200.sampling.OpenAIWrapper",
    "sgm.modules.diffusionmodules.wrappers.IdentityWrapper": "hi3d_official_b200.sampling.IdentityWrapper",
    "sgm.modules.diffusionmodules.denoiser.Denoiser": "hi3d_official_b200.sampling.Denoiser",
    "sgm.modules.diffusionmodules.denoiser_scaling.VScalingWithEDMcNoise":
        "hi3d_official_b200.sampling.VScalingWithEDMcNoise",
    "sgm.modules.diffusionmodules.denoiser_scaling.EDMScaling": "hi3d_official_b200.sampling.EDMScaling",
    "sgm.modules.diffusionmodules.denoiser_scaling.EpsScaling": "hi3d_official_b200.sampling.EpsScaling",
    "sgm.modules.diffusionmodules.denoiser_scaling.VScaling": "hi3d_official_b200.sampling.VScaling",
    "sgm.modules.diffusionmodules.discretizer.EDMDiscretization": "hi3d_official_b200.sampling.EDMDiscretization",
    "sgm.modules.diffusionmodules.guiders.LinearPredictionGuider": "hi3d_official_b200.sampling.LinearPredictionGuider",
    "sgm.modules.diffusionmodules.guiders.VanillaCFG": "hi3d_official_b200.sampling.VanillaCFG",
    "sgm.modules.diffusionmodules.guiders.IdentityGuider": "hi3d_official_b200.sampling.IdentityGuider",
    "sgm.modules.diffusionmodules.sampling.EulerEDMSampler": "hi3d_official_b200.sampling.EulerEDMSampler",
    "sgm.modules.diffusionmodules.sampling.HeunEDMSampler": "hi3d_official_b200.sampling.HeunEDMSampler",
    "sgm.modules.diffusionmodules.sampling.DPMPP2MSampler": "hi3d_official_b200.sampling.DPMPP2MSampler",
    "sgm.models.autoencoder.AutoencoderKL": "hi3d_official_b200.vae.AutoencoderKL",
    "sgm.models.autoencoder.AutoencoderKLModeOnly": "hi3d_official_b200.vae.AutoencoderKLModeOnly",
    # north_star's name for the first stage with the temporal decoder (SURVEY F3: no such class in the reference; its parts are
    # AutoencodingEngineLegacy + temporal_ae.VideoDecoder)
    "sgm.models.autoencoder.AutoencoderKLTemporal": "hi3d_official_b200.vae.AutoencoderKLTemporal",
    "sgm.modules.autoencoding.temporal_ae.VideoDecoder": "hi3d_official_b200.vae.VideoDecoder",
    "sgm.modules.diffusionmodules.model.Encoder": "hi3d_official_b200.vae.Encoder",
    "sgm.modules.diffusionmodules.model.Decoder": "hi3d_official_b200.vae.Decoder",
    "sgm.modules.GeneralConditioner": "hi3d_official_b200.conditioner.GeneralConditioner",
    "sgm.modules.encoders.modules.GeneralConditioner": "hi3d_official_b200.conditioner.GeneralConditioner",
    "sgm.modules.encoders.modules.ConcatTimestepEmbedderND": "hi3d_official_b200.conditioner.ConcatTimestepEmbedderND",
    "sgm.modules.encoders.modules.VideoPredictionEmbedderWithEncoder":
        "hi3d_official_b200.conditioner.VideoPredictionEmbedderWithEncoder",
    "sgm.modules.encoders.modules.FrozenOpenCLIPImagePredictionEmbedder":
        "hi3d_official_b200.conditioner.FrozenOpenCLIPImagePredictionEmbedder",
    "sgm.modules.encoders.modules.FrozenOpenCLIPImageEmbedder": "hi3d_official_b200.conditioner.FrozenOpenCLIPImageEmbedder",
    "vtdm.encoders.DepthEmbedder": "hi3d_official_b200.conditioner.DepthEmbedder",
    "vtdm.encoders.AesEmbedder": "hi3d_official_b200.conditioner.AesEmbedder",
    "vtdm.vtdm_gen_v01.VideoLDM": "hi3d_official_b200.engine.VideoLDM",
    "vtdm.vtdm_gen_stage2_degradeImage.VideoLDM": "hi3d_official_b200.engine.VideoLDMStage2",
    "sgm.models.diffusion.DiffusionEngine": "hi3d_official_b200.engine.DiffusionEngine",
    "torch.nn.Identity": "torch.nn.Identity",
}


def get_obj_from_str(string: str, reload: bool = False, invalidate_cache: bool = True):
    """sgm/util.py:178-185 with the alias table applied first."""
    string = TARGET_ALIASES.get(string, string)
    module, cls = string.rsplit(".", 1)
    if invalidate_cache:
        importlib.invalidate_caches()
    mod = importlib.import_module(module)
    if reload:
        mod = importlib.reload(mod)
    return getattr(mod, cls)


def instantiate_from_config(config: Dict[str, Any]):
    """sgm/util.py:168-175."""
    if "target" not in config:
        if config in ("__is_first_stage__", "__is_unconditional__"):
            return None
        raise KeyError("Expected key `target` to instantiate.")
    return get_obj_from_str(config["target"])(**(config.get("params", dict()) or dict()))


def default(val, d):
    if val is not None:
        return val
    return d() if callable(d) and not isinstance(d, (torch.nn.Module, type)) else d


def append_dims(x: torch.Tensor, target_dims: int) -> torch.Tensor:
    """sgm/util.py:192-199."""
    dims_to_append = target_dims - x.ndim
    if dims_to_append < 0:
        raise ValueError(f"input has {x.ndim} dims but target_dims is {target_dims}, which is less")
    return x[(...,) + (None,) * dims_to_append]


def append_zero(x: torch.Tensor) -> torch.Tensor:
    return torch.cat([x, x.new_zeros([1])])


def disabled_train(self, mode=True):
    """sgm/util.py: overwrite model.train so the first stage stays in eval mode."""
    return self


def load_yaml(path: str) -> dict:
    """OmegaConf.load stand-in (plain dict; the inference configs use no interpolation)."""
    import yaml
    with open(path, "r") as f:
        return yaml.safe_load(f)
