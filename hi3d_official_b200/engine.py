"""Model-engine layer: `DiffusionEngine` (sgm/models/diffusion.py:19-150) and the two `VideoLDM`s of
vtdm/vtdm_gen_v01.py / vtdm/vtdm_gen_stage2_degradeImage.py, restricted to what the inference entry points
(pipeline_i2v_eval_v0{1,2}.py) touch: construction from the unmodified YAML, checkpoint loading with the
reference's key prefixes, `encode_first_stage` / `decode_first_stage`, `.denoiser/.model/.sampler/.conditioner`
attributes, and the two hot loops (`sample_stage1`, `sample_stage2`) restated on top of the fused sampler.

Out of scope (SURVEY.md section 2): training (`shared_step`, optimisers, EMA, logging) and the MiDaS depth tower.  The CLIP
image towers run natively (clip_vision.py); `init_from_ckpt` hands their `conditioner.embedders.N.*` tensors to the
conditioner.  `PassThroughConditioner` keeps the seam: it returns conditioning dictionaries that the caller supplies
pre-computed (synthetic in the benches).
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Union

import torch
import torch.nn as nn

from .sampling import OPENAIUNETWRAPPER, FusedDenoiser
from .util import default, disabled_train, get_obj_from_str, instantiate_from_config, load_yaml


from .conditioner import GeneralConditioner

# Round-1 name of the conditioner seam; the real GeneralConditioner (conditioner.py) still passes ready-made batch["c"] /
# batch["uc"] dictionaries through, which is what the benches and tests feed.
PassThroughConditioner = GeneralConditioner


class DiffusionEngine(nn.Module):
    def __init__(self, network_config, denoiser_config, first_stage_config, conditioner_config=None,
                 sampler_config=None, optimizer_config=None, scheduler_config=None, loss_fn_config=None,
                 network_wrapper: Union[None, str] = None, ckpt_path: Union[None, str] = None, use_ema: bool = False,
                 ema_decay_rate: float = 0.9999, scale_factor: float = 1.0, disable_first_stage_autocast=False,
                 input_key: str = "jpg", log_keys=None, no_cond_log: bool = False, compile_model: bool = False,
                 en_and_decode_n_samples_a_time: Optional[int] = None):
        super().__init__()
        if use_ema:
            raise NotImplementedError("EMA weights are training-only (out of scope)")
        self.log_keys, self.input_key = log_keys, input_key
        model = instantiate_from_config(network_config)
        self.model = get_obj_from_str(default(network_wrapper, OPENAIUNETWRAPPER))(model, compile_model=compile_model)
        self.denoiser = instantiate_from_config(denoiser_config)
        self.sampler = instantiate_from_config(sampler_config) if sampler_config is not None else None
        self.conditioner = instantiate_from_config(conditioner_config) if conditioner_config is not None \
            else PassThroughConditioner()
        self._init_first_stage(first_stage_config)
        self.loss_fn = None                     # loss_fn_config is training-only
        self.scale_factor = scale_factor
        self.disable_first_stage_autocast = disable_first_stage_autocast
        self.en_and_decode_n_samples_a_time = en_and_decode_n_samples_a_time
        if ckpt_path is not None:
            self.init_from_ckpt(ckpt_path)

    def _init_first_stage(self, config):
        model = instantiate_from_config(config).eval()
        model.train = disabled_train.__get__(model)
        for p in model.parameters():
            p.requires_grad = False
        self.first_stage_model = model

    @property
    def device(self):
        return self.model.diffusion_model.device

    # -- checkpoints: prefixes model.diffusion_model.* | first_stage_model.* | conditioner.* (SURVEY App. B) ---------
    @staticmethod
    def _read_ckpt(path: str) -> Dict[str, torch.Tensor]:
        if path.endswith("ckpt"):
            sd = torch.load(path, map_location="cpu")
            return sd.get("state_dict", sd)
        if path.endswith("pt"):            # DeepSpeed: {'module': {'module.<key>': tensor}} (vtdm_gen_v01.py:38-42)
            raw = torch.load(path, map_location="cpu")
            return {k[len("module."):]: v for k, v in raw["module"].items()}
        if path.endswith("safetensors"):
            from safetensors.torch import load_file
            return load_file(path)
        raise NotImplementedError(path)

    def init_from_ckpt(self, path: str) -> None:
        sd = self._read_ckpt(path)
        missing, unexpected = self.load_state_dict(sd, strict=False)
        towers = self.conditioner.load_tower_weights(sd) if hasattr(self.conditioner, "load_tower_weights") else []
        if towers:
            print(f"native conditioner towers from {path}: {towers}")
        unexpected = [k for k in unexpected if not k.startswith(("conditioner.", "loss_fn.", "model_ema."))]
        print(f"Restored from {path} with {len(missing)} missing and {len(unexpected)} unexpected keys")
        if missing:
            print(f"Missing Keys: {missing}")
        if unexpected:
            print(f"Unexpected Keys: {unexpected}")

    # -- first stage (diffusion.py:117-150) -----------------------------------------------------------------------------
    @torch.no_grad()
    def decode_first_stage(self, z: torch.Tensor) -> torch.Tensor:
        from .vae import VideoDecoder
        n_samples = default(self.en_and_decode_n_samples_a_time, z.shape[0])
        outs = []
        for i in range(0, z.shape[0], n_samples):
            zi = z[i:i + n_samples]
            # diffusion.py:126-129: a temporal decoder is told how many frames the chunk holds
            kw = {"timesteps": len(zi)} if isinstance(self.first_stage_model.decoder, VideoDecoder) else {}
            outs.append(self.first_stage_model.decode(zi, scale=1.0 / self.scale_factor, **kw))
        return torch.cat(outs, 0) if len(outs) > 1 else outs[0]

    @torch.no_grad()
    def encode_first_stage(self, x: torch.Tensor, noise: Optional[torch.Tensor] = None) -> torch.Tensor:
        n_samples = default(self.en_and_decode_n_samples_a_time, x.shape[0])
        outs = [self.first_stage_model.encode(x[i:i + n_samples], scale=self.scale_factor,
                                              noise=None if noise is None else noise[i:i + n_samples])
                for i in range(0, x.shape[0], n_samples)]
        return torch.cat(outs, 0) if len(outs) > 1 else outs[0]

    # -- the pipelines' denoiser closure as a fusable binding ---------------------------------------------------------------
    def bind_denoiser(self, shard=None, **additional_model_inputs) -> FusedDenoiser:
        return FusedDenoiser(self.denoiser, self.model, shard=shard, **additional_model_inputs)


class VideoLDM(DiffusionEngine):
    """vtdm/vtdm_gen_v01.py:24-76."""

    def __init__(self, num_samples, trained_param_keys=("",), *args, **kwargs):
        self.trained_param_keys = trained_param_keys
        super().__init__(*args, **kwargs)
        self.num_samples = num_samples

    @torch.no_grad()
    def add_custom_cond(self, batch, infer=False):
        """vtdm_gen_v01.py:59-76 (inference branch): cond_aug = 0.02, cond_frames = image + 0.02 * randn."""
        if not infer:
            raise NotImplementedError("training-time cond_aug sampling is out of scope")
        batch["num_video_frames"] = self.num_samples
        image = batch["video"][:, :, 0]
        batch["cond_frames_without_noise"] = image.half()
        n = batch["video"].shape[0]
        cond_aug = torch.full((n,), 0.02, device=image.device).half()
        batch["cond_aug"] = cond_aug
        batch["cond_frames"] = (image + cond_aug.view(-1, 1, 1, 1) * torch.randn_like(image)).half()
        if "image_only_indicator" not in batch:
            batch["image_only_indicator"] = torch.zeros((n, self.num_samples), device=image.device).half()
        return batch

    # ---- hot loop of pipeline_i2v_eval_v01.py:62-98 (after conditioning) ------------------------------------------------------
    @torch.no_grad()
    def sample_stage1(self, c: Dict, uc: Dict, randn: torch.Tensor, decode: bool = True, shard=None):
        """shard = (rank, world): `randn` and c/uc['concat'] hold only this rank's frames (frame-sharded video); the
        returned latents / decoded frames are this rank's frames too."""
        T = self.num_samples
        den = self.bind_denoiser(shard=shard, image_only_indicator=None, num_video_frames=T)
        samples = self.sampler(den, randn, cond=c, uc=uc)
        if not decode:
            return samples
        return self.decode_first_stage(samples.half())


class VideoLDMStage2(VideoLDM):
    """vtdm/vtdm_gen_stage2_degradeImage.py VideoLDM (inference surface only)."""

    @torch.no_grad()
    def add_custom_cond(self, batch, infer=False):
        """vtdm_gen_stage2_degradeImage.py:63-86 (inference): cond frames are all T frames of the low-res video."""
        if not infer:
            raise NotImplementedError("training-time degradation pipeline is out of scope")
        batch["num_video_frames"] = self.num_samples
        video = batch["video"]                                   # (b, c, t, h, w)
        frames = video.permute(0, 2, 1, 3, 4).reshape(-1, *video.shape[1:2], *video.shape[3:])
        batch["cond_frames_without_noise"] = video[:, :, 0].half()
        n = video.shape[0]
        cond_aug = torch.full((n,), 0.02, device=video.device).half()
        batch["cond_aug"] = cond_aug
        batch["cond_frames"] = (frames + 0.02 * torch.randn_like(frames)).half()
        if "image_only_indicator" not in batch:
            batch["image_only_indicator"] = torch.zeros((n, self.num_samples), device=video.device).half()
        return batch

    # ---- hot loop of pipeline_i2v_eval_v02.py:86-137 ---------------------------------------------------------------------------
    @torch.no_grad()
    def sample_stage2(self, c: Dict, uc: Dict, init_latents: torch.Tensor, z: torch.Tensor, decode: bool = True,
                      alpha_pow: float = 40.0, shard=None):
        """init_latents ~ N(0,1) (T,4,h,w) fp32; z = encode_first_stage(low-res frames) (T,4,h,w).
        shard = (rank, world): all per-frame tensors hold only this rank's frames."""
        from . import ops
        smp = self.sampler
        T = self.num_samples
        sigmas = smp.discretization(smp.num_steps, device="cpu").to(init_latents.device)
        num_sigmas = len(sigmas)
        sig_host = sigmas.tolist()
        s_in = init_latents.new_ones([init_latents.shape[0]])
        latents = (init_latents * math.sqrt(1.0 + sig_host[0] ** 2.0)).contiguous()
        init_latents = init_latents.float().contiguous()
        z = z.float().contiguous()
        den = self.bind_denoiser(shard=shard, image_only_indicator=None, num_video_frames=T)
        for i in smp.get_sigma_gen(num_sigmas):
            alpha = math.pow(0.5 * (1 + math.cos(i * 1.0 / smp.num_steps)), alpha_pow)
            ops.renoise_blend(latents, init_latents, z, alpha, sig_host[i])           # v02:131-132
            latents = smp.step_call(den, latents, i, s_in, sigmas, num_sigmas, c, uc)   # v02:134-135
        if not decode:
            return latents
        return self.decode_first_stage(latents.half())


def create_model(config_path: str, **overrides):
    """vtdm/model.py:24-28 -- the unmodified reference YAML resolves to the H100 classes through util.TARGET_ALIASES."""
    config = load_yaml(config_path)
    cfg = config["model"]
    params = dict(cfg.get("params", {}))
    params.update(overrides)
    model = get_obj_from_str(cfg["target"])(**params)
    print(f"Loaded model config from [{config_path}]")
    return model
