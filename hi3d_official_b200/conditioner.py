"""Conditioner side of the pipelines (SURVEY §8f N2): `GeneralConditioner` and the embedders of configs/inference-v0{1,2}.yaml
that do not need third-party model weights, with the reference's names, ctor kwargs and call semantics:

  GeneralConditioner                    sgm/modules/encoders/modules.py:71-184
  ConcatTimestepEmbedderND              :913-929      (sinusoidal embedding per scalar: hi3d_timestep_embedding kernel)
  VideoPredictionEmbedderWithEncoder    :951-1025     (cond-frame latents through THIS package's AutoencoderKL encoder)
  FrozenOpenCLIPImagePredictionEmbedder :1028-1046    (frame / copy bookkeeping around an image tower)
  DepthEmbedder                         vtdm/encoders.py:15-53   (resize, per-image min-max, 3x3 pixel-unshuffle to 9 channels)
  AesEmbedder                           vtdm/encoders.py:56-90   ([score | timestep_embedding(100 score, 255)])

The three towers -- OpenCLIP ViT-H/14 (image embedding), OpenAI CLIP ViT-L/14 + the aesthetic MLP (score) and MiDaS DPT-Hybrid
(depth) -- run natively on this package's kernels (clip_vision.py, midas.py) once their weights are loaded: from the reference's
files (the OpenCLIP embedder's `version` path; ckpts/ViT-L-14.pt, ckpts/metric_models/sac+logos+ava1-l14-linearMSE.pth and
ckpts/dpt_hybrid_384.pt relative to the working directory, as vtdm/encoders.py:18,60-64 hard-codes them), or from the
`conditioner.embedders.N.*` tensors of a full checkpoint (GeneralConditioner.load_tower_weights, called by
DiffusionEngine.init_from_ckpt), which win.  Every tower sits behind an `ExternalTower`: a callable installed with
`.set_fn(...)` comes first, then the native tower, and a pre-computed tensor passed in the batch under `<input_key>:<tower>`
(e.g. batch["cond_frames_without_noise:clip"] = (B, 1024)) takes precedence over both.  Without weights, calling a tower
raises.  Everything AROUND the towers is the reference's arithmetic, so the unmodified conditioner_config instantiates and
produces the reference's `c` / `uc` dictionaries (crossattn (B,1,1024), vector (B,768|512), concat (B*T, 4|13, h, w)).

Compatibility: a batch that already holds ready-made dictionaries (`batch["c"]`, optional `batch["uc"]`) is passed through --
the benches and tests feed synthetic conditioning that way.
"""
from __future__ import annotations

import math
import os
from contextlib import nullcontext
from typing import Callable, Dict, List, Optional, Sequence, Union

import torch
import torch.nn as nn

from .util import disabled_train, instantiate_from_config


class AbstractEmbModel(nn.Module):
    """sgm/modules/encoders/modules.py:33-68 (is_trainable / ucg_rate / input_key properties as plain attributes)."""

    def __init__(self):
        super().__init__()
        self.is_trainable = False
        self.ucg_rate = 0.0
        self.input_key: Optional[str] = None
        self.legacy_ucg_val = None


class ExternalTower(AbstractEmbModel):
    """Stand-in for a third-party network (OpenCLIP image tower, MiDaS, CLIP-L + aesthetic MLP).  Accepts the reference
    ctor kwargs and ignores them; `set_fn` installs the real model (any callable tensor -> tensor)."""

    def __init__(self, *args, **kwargs):
        super().__init__()
        self.kwargs = kwargs
        self.fn: Optional[Callable] = None

    def set_fn(self, fn: Callable):
        self.fn = fn
        return self

    def native(self) -> Optional[Callable]:
        """The tower on this package's kernels, when its weights are loaded (subclasses)."""
        return None

    def forward(self, x):
        if self.fn is None and self.native() is not None:
            return self.native()(x)
        if self.fn is None:
            raise NotImplementedError(
                f"{type(self).__name__}: this third-party tower (ctor kwargs {self.kwargs}) is outside the H100 hot path and its "
                f"checkpoint is not bundled; install it with .set_fn(callable) or pass its output in the batch "
                f"(see hi3d_official_b200/conditioner.py)")
        return self.fn(x)


class FrozenOpenCLIPImageEmbedder(ExternalTower):
    """sgm/modules/encoders/modules.py:570-728 (OpenCLIP ViT-H-14 image tower -> (N, 1024)): images in [-1, 1] -> kornia bicubic
    antialiased resize to 224^2 -> [0, 1] -> CLIP normalisation -> ViT.  Native once weights are loaded: at construction from
    the `version` file when it exists, or later with load_visual()."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.arch = kwargs.get("arch", "ViT-H-14")
        self._visual_sd: Optional[Dict[str, torch.Tensor]] = None     # `visual.*` tensors (no prefix), packed on first use
        self._tower = None
        version = kwargs.get("version")
        if isinstance(version, str) and os.path.isfile(version):
            from . import clip_vision
            self.load_visual(clip_vision.load_open_clip(version))

    def load_visual(self, sd: Dict[str, torch.Tensor]):
        self._visual_sd, self._tower = dict(sd), None
        return self

    def native(self) -> Optional[Callable]:
        return None if self._visual_sd is None else self._run_native

    def _run_native(self, x: torch.Tensor) -> torch.Tensor:
        from . import clip_vision
        if self._tower is None or self._tower.device != x.device:
            self._tower = clip_vision.ClipVisionTower(self._visual_sd, clip_vision.head_width_of(self.arch), quick_gelu=False,
                                                      device=x.device)
        return self._tower(clip_vision.openclip_preprocess(x)).to(x.dtype if x.is_floating_point() else torch.float32)


class MiDaSInference(ExternalTower):
    """annotator/midas/api.py:146-165 (DPT-hybrid -> (N, h, w) inverse depth).  Native (midas.py) once weights are loaded: at
    construction from ckpts/dpt_hybrid_384.pt under the working directory when it exists (the path vtdm/encoders.py:18
    hard-codes), or later with load_weights()."""
    PATH = os.path.join("ckpts", "dpt_hybrid_384.pt")

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self._sd: Optional[Dict[str, torch.Tensor]] = None       # the reference's DPTDepthModel tensors, packed on first use
        self._tower = None
        if os.path.isfile(self.PATH):
            from . import midas
            self.load_weights(midas.load_dpt_hybrid(self.PATH))

    def load_weights(self, sd: Dict[str, torch.Tensor]):
        """`sd`: the DPTDepthModel state dict (reference keys); raises KeyError when a tensor is missing."""
        from . import midas
        self._sd, self._tower = midas.live_state_dict(dict(sd)), None
        return self

    def native(self) -> Optional[Callable]:
        return None if self._sd is None else self._run_native

    def _run_native(self, x: torch.Tensor) -> torch.Tensor:
        from . import midas
        if self._tower is None or self._tower.device != x.device:
            self._tower = midas.DPTHybridTower(self._sd, device=x.device)
        return self._tower(x)


class AestheticScore(ExternalTower):
    """vtdm/encoders.py:57-88: CLIP ViT-L image features -> normalised -> aesthetic MLP -> (N, 1) score.  Native once weights
    are loaded: at construction from the reference's files under the working directory when both exist, or later with
    load_weights()."""
    CLIP_PATH = os.path.join("ckpts", "ViT-L-14.pt")
    MLP_PATH = os.path.join("ckpts", "metric_models", "sac+logos+ava1-l14-linearMSE.pth")

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self._parts = [None, None, None]     # `visual.*` tensors (no prefix), folded MLP weight (768,) and bias ()
        self._scorer = None
        if os.path.isfile(self.CLIP_PATH) and os.path.isfile(self.MLP_PATH):
            from . import clip_vision
            self.load_weights(clip_vision.load_openai_clip(self.CLIP_PATH), *clip_vision.load_aesthetic_mlp(self.MLP_PATH))

    def load_weights(self, visual_sd: Optional[Dict[str, torch.Tensor]] = None, mlp_w: Optional[torch.Tensor] = None,
                     mlp_b: Optional[torch.Tensor] = None):
        """The CLIP tower and the folded MLP may come separately; the scorer is native once both are there."""
        for i, t in enumerate((visual_sd, mlp_w, mlp_b)):
            if t is not None:
                self._parts[i] = dict(t) if isinstance(t, dict) else t
        self._scorer = None
        return self

    def native(self) -> Optional[Callable]:
        return self._run_native if all(t is not None for t in self._parts) else None

    def _run_native(self, x: torch.Tensor) -> torch.Tensor:
        from . import clip_vision
        if self._scorer is None or self._scorer.tower.device != x.device:
            self._scorer = clip_vision.AestheticScorer(*self._parts, device=x.device)
        return self._scorer(x)


def timestep_embedding(t: torch.Tensor, dim: int, max_period: float = 10000.0) -> torch.Tensor:
    """sgm/modules/diffusionmodules/util.py:207-231 through the CUDA kernel (fp16 out, widened to fp32); CPU tensors take
    the closed form (host-only unit tests)."""
    t = t.reshape(-1).float()
    if t.is_cuda:
        from . import ops
        out = torch.empty(t.numel(), dim, dtype=torch.float16, device=t.device)
        ops.timestep_embedding(t.contiguous(), dim, out, max_period)
        return out.float()
    half = dim // 2
    freqs = torch.exp(-math.log(max_period) * torch.arange(half, dtype=torch.float32) / half)
    args = t[:, None] * freqs[None]
    emb = torch.cat([torch.cos(args), torch.sin(args)], -1)
    if dim % 2:
        emb = torch.cat([emb, torch.zeros_like(emb[:, :1])], -1)
    return emb


class ConcatTimestepEmbedderND(AbstractEmbModel):
    """embeds each dimension independently and concatenates them (modules.py:913-929)."""

    def __init__(self, outdim: int):
        super().__init__()
        self.outdim = outdim

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if x.ndim == 1:
            x = x[:, None]
        assert x.ndim == 2
        b, dims = x.shape
        emb = timestep_embedding(x.reshape(b * dims), self.outdim)           # "(b d) d2"
        return emb.reshape(b, dims * self.outdim)                             # "b (d d2)"


class VideoPredictionEmbedderWithEncoder(AbstractEmbModel):
    """modules.py:951-1025: cond frames -> first-stage latents (mode of the posterior for AutoencoderKLModeOnly) * scale_factor,
    "(b t) c h w -> b () (t c) h w", repeated n_copies times along the batch."""

    def __init__(self, n_cond_frames: int, n_copies: int, encoder_config: dict, sigma_sampler_config: Optional[dict] = None,
                 sigma_cond_config: Optional[dict] = None, is_ae: bool = False, scale_factor: float = 1.0,
                 disable_encoder_autocast: bool = False, en_and_decode_n_samples_a_time: Optional[int] = None):
        super().__init__()
        if sigma_sampler_config is not None or sigma_cond_config is not None:
            raise NotImplementedError("sigma_sampler / sigma_cond (training-time noise augmentation) are out of scope")
        self.n_cond_frames, self.n_copies = n_cond_frames, n_copies
        self.encoder = instantiate_from_config(encoder_config)
        self.is_ae, self.scale_factor = is_ae, scale_factor
        self.disable_encoder_autocast = disable_encoder_autocast
        self.en_and_decode_n_samples_a_time = en_and_decode_n_samples_a_time

    def forward(self, vid: torch.Tensor) -> torch.Tensor:
        n_samples = self.en_and_decode_n_samples_a_time or vid.shape[0]
        outs = []
        for i in range(0, vid.shape[0], n_samples):
            chunk = vid[i:i + n_samples]
            outs.append(self.encoder.encode(chunk) if self.is_ae else self.encoder(chunk))
        z = torch.cat(outs, 0) if len(outs) > 1 else outs[0]
        z = z * self.scale_factor
        bt, c, h, w = z.shape
        b = bt // self.n_cond_frames
        z = z.reshape(b, self.n_cond_frames * c, h, w)                        # "(b t) c h w -> b (t c) h w"
        return z.repeat_interleave(self.n_copies, dim=0)                      # "b 1 c h w -> (b t) c h w"


class FrozenOpenCLIPImagePredictionEmbedder(AbstractEmbModel):
    """modules.py:1028-1046: image tower on the cond frames, "(b t) d -> b t d", each sample repeated n_copies times."""

    def __init__(self, open_clip_embedding_config: Dict, n_cond_frames: int, n_copies: int):
        super().__init__()
        self.n_cond_frames, self.n_copies = n_cond_frames, n_copies
        self.open_clip = instantiate_from_config(open_clip_embedding_config)

    def arrange(self, emb: torch.Tensor) -> torch.Tensor:
        emb = emb.reshape(-1, self.n_cond_frames, emb.shape[-1])
        return emb.repeat_interleave(self.n_copies, dim=0)

    def forward(self, vid: torch.Tensor) -> torch.Tensor:
        return self.arrange(self.open_clip(vid))


def depth_to_concat(y: torch.Tensor, H: int, W: int, shuffle_size: int = 3) -> torch.Tensor:
    """vtdm/encoders.py:44-50: depth maps (n, h', w') -> bilinear to (H/8*s, W/8*s), per-image min-max to [0, 1],
    "b c (h h0) (w w0) -> b (c h0 w0) h w": (n, s*s, H/8, W/8)."""
    y = y[:, None].float()
    y = torch.nn.functional.interpolate(y, [H // 8 * shuffle_size, W // 8 * shuffle_size], mode="bilinear")
    y = y - y.amin(dim=(1, 2, 3), keepdim=True)
    y = y / y.amax(dim=(1, 2, 3), keepdim=True).clamp_min(1e-6)
    n, c, hh, ww = y.shape
    s = shuffle_size
    return y.reshape(n, c, hh // s, s, ww // s, s).permute(0, 1, 3, 5, 2, 4).reshape(n, c * s * s, hh // s, ww // s)


class DepthEmbedder(AbstractEmbModel):
    """vtdm/encoders.py:15-53 around the MiDaS DPT-Hybrid depth tower (`self.model`)."""

    def __init__(self, freeze: bool = True, use_3d: bool = False, shuffle_size: int = 3, scale_factor: float = 2.6666):
        super().__init__()
        self.model = MiDaSInference(model_type="dpt_hybrid")
        self.use_3d, self.shuffle_size, self.scale_factor = use_3d, shuffle_size, scale_factor

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if x.ndim == 4:
            x = x.reshape(-1, 16, *x.shape[1:]).permute(0, 2, 1, 3, 4)        # "(b t) c h w -> b c t h w", t = 16
        B, C, T, H, W = x.shape
        sH, sW = int(H / self.scale_factor / 32) * 32, int(W / self.scale_factor / 32) * 32
        y = x.permute(0, 2, 1, 3, 4).reshape(B * T, C, H, W)
        y = torch.nn.functional.interpolate(y.float(), [sH, sW], mode="bilinear")
        y = depth_to_concat(self.model(y), H, W, self.shuffle_size)
        if self.use_3d:
            y = y.reshape(B, T, *y.shape[1:]).permute(0, 2, 1, 3, 4)
        return y


class AesEmbedder(AbstractEmbModel):
    """vtdm/encoders.py:56-90: middle frame -> 224 x 384 bilinear -> centre 224 crop -> CLIP normalisation -> external
    aesthetic scorer -> [score | timestep_embedding(100 * score, 255)] (256-d vector conditioning)."""
    MEAN = (0.48145466, 0.4578275, 0.40821073)
    STD = (0.26862954, 0.26130258, 0.27577711)

    def __init__(self, freeze: bool = True):
        super().__init__()
        self.scorer = AestheticScore()

    def preprocess(self, x: torch.Tensor) -> torch.Tensor:
        B, C, T, H, W = x.shape
        y = torch.nn.functional.interpolate(x[:, :, T // 2].float(), [224, 384], mode="bilinear")[:, :, :, 80:304]
        y = (y + 1) * 0.5
        m = torch.tensor(self.MEAN, device=y.device).view(1, 3, 1, 1)
        s = torch.tensor(self.STD, device=y.device).view(1, 3, 1, 1)
        return (y - m) / s

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        aesthetic = self.scorer(self.preprocess(x)).reshape(-1, 1).float()
        return torch.cat([aesthetic, timestep_embedding(aesthetic[:, 0] * 100, 255)], 1)


class GeneralConditioner(nn.Module):
    OUTPUT_DIM2KEYS = {2: "vector", 3: "crossattn", 4: "concat", 5: "concat"}
    KEY2CATDIM = {"vector": 1, "crossattn": 2, "concat": 1}
    TOWER_OF = {"FrozenOpenCLIPImagePredictionEmbedder": "clip", "DepthEmbedder": "depth", "AesEmbedder": "aes"}

    def __init__(self, emb_models: Optional[Sequence] = None):
        super().__init__()
        embedders = []
        for n, embconfig in enumerate(emb_models or []):
            embedder = instantiate_from_config(embconfig)
            assert isinstance(embedder, AbstractEmbModel), \
                f"embedder model {embedder.__class__.__name__} has to inherit from AbstractEmbModel"
            embedder.is_trainable = embconfig.get("is_trainable", False)
            embedder.ucg_rate = embconfig.get("ucg_rate", 0.0)
            if embedder.is_trainable:
                raise NotImplementedError("trainable embedders are training-only (out of scope)")
            embedder.train = disabled_train.__get__(embedder)
            for p in embedder.parameters():
                p.requires_grad = False
            embedder.eval()
            if "input_key" in embconfig:
                embedder.input_key = embconfig["input_key"]
            elif "input_keys" in embconfig:
                embedder.input_keys = embconfig["input_keys"]
            else:
                raise KeyError(f"need either 'input_key' or 'input_keys' for embedder {embedder.__class__.__name__}")
            embedder.legacy_ucg_val = embconfig.get("legacy_ucg_value", None)
            if embedder.legacy_ucg_val is not None:
                raise NotImplementedError("legacy_ucg_value (training-time classifier-free dropout) is out of scope")
            embedders.append(embedder)
        self.embedders = nn.ModuleList(embedders)
        self.emb_model_configs = list(emb_models or [])

    # -- native tower weights from a full checkpoint (DiffusionEngine.init_from_ckpt) ---------------------------------------------
    def load_tower_weights(self, sd: Dict[str, torch.Tensor], prefix: str = "conditioner.") -> List[str]:
        """Routes `<prefix>embedders.N.open_clip.model.visual.*`, `...N.aesthetic_model.visual.*`, `...N.aesthetic_mlp.*` and
        `...N.model.model.*` (DepthEmbedder -> MiDaSInference -> DPTDepthModel) to the native towers (the reference's module paths).
        Returns the names of the towers that received weights."""
        from . import clip_vision
        loaded = []
        for i, e in enumerate(self.embedders):
            p = f"{prefix}embedders.{i}."
            if isinstance(e, FrozenOpenCLIPImagePredictionEmbedder) and isinstance(e.open_clip, FrozenOpenCLIPImageEmbedder):
                vis = {k[len(p + "open_clip.model.visual."):]: v for k, v in sd.items() if k.startswith(p + "open_clip.model.visual.")}
                if vis:
                    e.open_clip.load_visual(vis)
                    loaded.append("clip")
            elif isinstance(e, AesEmbedder):
                vis = {k[len(p + "aesthetic_model.visual."):]: v for k, v in sd.items() if k.startswith(p + "aesthetic_model.visual.")}
                mlp = {k[len(p + "aesthetic_mlp."):]: v for k, v in sd.items() if k.startswith(p + "aesthetic_mlp.")}
                if vis or mlp:
                    e.scorer.load_weights(vis or None, *(clip_vision.fold_linear_chain(mlp) if mlp else (None, None)))
                    loaded.append("aes")
            elif isinstance(e, DepthEmbedder) and isinstance(e.model, MiDaSInference):
                dpt = {k[len(p + "model.model."):]: v for k, v in sd.items() if k.startswith(p + "model.model.")}
                if dpt:
                    e.model.load_weights(dpt)
                    loaded.append("depth")
        return loaded

    def missing_towers(self) -> List[str]:
        """Towers of this conditioner that can neither run natively nor through an installed callable ('clip', 'depth',
        'aes'): their outputs must come in the batch."""
        out = []
        for e in self.embedders:
            tower = self.TOWER_OF.get(type(e).__name__)
            ext = {"clip": lambda m: m.open_clip, "depth": lambda m: m.model, "aes": lambda m: m.scorer}.get(tower)
            if ext is None:
                continue
            t = ext(e)
            if isinstance(t, ExternalTower) and t.fn is None and t.native() is None:
                out.append(tower)
        return out

    # -- one embedder, honouring pre-computed tower outputs in the batch -------------------------------------------------------
    def _embed(self, embedder: AbstractEmbModel, batch: Dict):
        if getattr(embedder, "input_key", None) is not None:
            tower = self.TOWER_OF.get(type(embedder).__name__)
            pre = batch.get(f"{embedder.input_key}:{tower}") if tower else None
            if pre is not None:
                if tower == "clip":
                    return embedder.arrange(pre)
                if tower == "depth":
                    x = batch[embedder.input_key]
                    return depth_to_concat(pre, x.shape[-2], x.shape[-1], embedder.shuffle_size)
                pre = pre.reshape(-1, 1).float()
                return torch.cat([pre, timestep_embedding(pre[:, 0] * 100, 255)], 1)
            return embedder(batch[embedder.input_key])
        return embedder(*[batch[k] for k in embedder.input_keys])

    def forward(self, batch: Dict, force_zero_embeddings: Optional[List] = None) -> Dict:
        if "c" in batch:                                  # ready-made conditioning (benches / tests)
            return batch["c"]
        output: Dict[str, torch.Tensor] = {}
        force_zero_embeddings = force_zero_embeddings or []
        for embedder in self.embedders:
            with (nullcontext() if embedder.is_trainable else torch.no_grad()):
                emb_out = self._embed(embedder, batch)
            assert isinstance(emb_out, (torch.Tensor, list, tuple)), \
                f"encoder outputs must be tensors or a sequence, but got {type(emb_out)}"
            if not isinstance(emb_out, (list, tuple)):
                emb_out = [emb_out]
            for emb in emb_out:
                out_key = self.OUTPUT_DIM2KEYS[emb.dim()]
                if embedder.ucg_rate > 0.0 and embedder.legacy_ucg_val is None:
                    keep = torch.bernoulli((1.0 - embedder.ucg_rate) * torch.ones(emb.shape[0], device=emb.device))
                    emb = keep.view(-1, *([1] * (emb.dim() - 1))) * emb
                if getattr(embedder, "input_key", None) in force_zero_embeddings:
                    emb = torch.zeros_like(emb)
                if out_key in output:
                    output[out_key] = torch.cat((output[out_key], emb.to(output[out_key].dtype)), self.KEY2CATDIM[out_key])
                else:
                    output[out_key] = emb
        return output

    def get_unconditional_conditioning(self, batch_c: Dict, batch_uc: Optional[Dict] = None,
                                       force_uc_zero_embeddings: Optional[List[str]] = None,
                                       force_cond_zero_embeddings: Optional[List[str]] = None):
        src = batch_c if batch_uc is None else batch_uc
        if "c" in batch_c:
            c = batch_c["c"]
            if "uc" in src:
                return c, src["uc"]
            # reference semantics of force_uc_zero_embeddings=['cond_frames', 'cond_frames_without_noise']
            # (pipeline_i2v_eval_v01.py:75-78): the CLIP token and the concat latent are zeroed, `vector` is kept
            return c, {k: (torch.zeros_like(v) if k in ("crossattn", "concat") else v.clone()) for k, v in c.items()}
        rates = [e.ucg_rate for e in self.embedders]
        for e in self.embedders:
            e.ucg_rate = 0.0
        c = self(batch_c, force_cond_zero_embeddings)
        uc = self(src, force_uc_zero_embeddings or [])
        for e, r in zip(self.embedders, rates):
            e.ucg_rate = r
        return c, uc
