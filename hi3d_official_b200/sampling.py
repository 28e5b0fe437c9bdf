"""Sampler-side operator surface of the reference, same names and call signatures:

  EDMDiscretization            sgm/modules/diffusionmodules/discretizer.py:17-39
  VScalingWithEDMcNoise (+EDM/Eps/V scalings)   denoiser_scaling.py:11-59
  Denoiser                     denoiser.py:12-39
  IdentityWrapper / OpenAIWrapper   wrappers.py:8-34
  IdentityGuider / VanillaCFG / LinearPredictionGuider   guiders.py:24-99
  BaseDiffusionSampler / EDMSampler / EulerEDMSampler (+ Hi3D's step_call)   sampling.py:21-147,228-232
  HeunEDMSampler / DPMPP2MSampler   sampling.py:235-254,304-379
  AncestralSampler / EulerAncestralSampler / DPMPP2SAncestralSampler / LinearMultistepSampler   sampling.py:150-226,254-302

Two execution paths with identical results:
  * generic: `denoiser` is any Python callable (x, sigma, cond) -> denoised, exactly like the reference; the
    few elementwise ops on the (16, 4, h, w) fp32 sampler state are torch glue around whatever the callable does;
  * fused (the product path): when the callable is a `FusedDenoiser` binding (Denoiser + OpenAIWrapper(VideoUNet)),
    one Euler step is  hi3d_sampler_pre -> VideoUNet launch plan -> hi3d_sampler_post  with no host sync,
    no torch math and the step-invariant conditioning computed once per video.  Every sampler and guider takes it: each
    network evaluation is a CUDA-graph replay, and a stochastic step's noise is drawn into a static buffer before the replay.
"""
from __future__ import annotations

import os
from typing import Dict, List, Optional, Tuple, Union

import torch
import torch.nn as nn

from . import _native, ops
from .unet import CIN_PAD, VideoUNet
from .util import append_dims, append_zero, default, instantiate_from_config

OPENAIUNETWRAPPER = "sgm.modules.diffusionmodules.wrappers.OpenAIWrapper"


# ------------------------------------------------------------------------------------------------------------
# discretisation / scalings
# ------------------------------------------------------------------------------------------------------------
class Discretization:
    def __call__(self, n, do_append_zero=True, device="cpu", flip=False):
        sigmas = self.get_sigmas(n, device=device)
        sigmas = append_zero(sigmas) if do_append_zero else sigmas
        return sigmas if not flip else torch.flip(sigmas, (0,))

    def get_sigmas(self, n, device):
        raise NotImplementedError


class EDMDiscretization(Discretization):
    def __init__(self, sigma_min=0.002, sigma_max=80.0, rho=7.0):
        self.sigma_min, self.sigma_max, self.rho = sigma_min, sigma_max, rho

    def get_sigmas(self, n, device="cpu"):
        ramp = torch.linspace(0, 1, n, device=device)
        min_inv_rho = self.sigma_min ** (1 / self.rho)
        max_inv_rho = self.sigma_max ** (1 / self.rho)
        return (max_inv_rho + ramp * (min_inv_rho - max_inv_rho)) ** self.rho


class EDMScaling:
    def __init__(self, sigma_data: float = 0.5):
        self.sigma_data = sigma_data

    def __call__(self, sigma):
        c_skip = self.sigma_data ** 2 / (sigma ** 2 + self.sigma_data ** 2)
        c_out = sigma * self.sigma_data / (sigma ** 2 + self.sigma_data ** 2) ** 0.5
        c_in = 1 / (sigma ** 2 + self.sigma_data ** 2) ** 0.5
        return c_skip, c_out, c_in, 0.25 * sigma.log()


class EpsScaling:
    def __call__(self, sigma):
        return torch.ones_like(sigma), -sigma, 1 / (sigma ** 2 + 1.0) ** 0.5, sigma.clone()


class VScaling:
    def __call__(self, sigma):
        return 1.0 / (sigma ** 2 + 1.0), -sigma / (sigma ** 2 + 1.0) ** 0.5, 1.0 / (sigma ** 2 + 1.0) ** 0.5, sigma.clone()


class VScalingWithEDMcNoise:
    def __call__(self, sigma):
        c_skip = 1.0 / (sigma ** 2 + 1.0)
        c_out = -sigma / (sigma ** 2 + 1.0) ** 0.5
        c_in = 1.0 / (sigma ** 2 + 1.0) ** 0.5
        c_noise = 0.25 * sigma.log()
        return c_skip, c_out, c_in, c_noise


# ------------------------------------------------------------------------------------------------------------
# denoiser + wrappers
# ------------------------------------------------------------------------------------------------------------
class Denoiser(nn.Module):
    def __init__(self, scaling_config: Dict):
        super().__init__()
        self.scaling = instantiate_from_config(scaling_config)

    def possibly_quantize_sigma(self, sigma):
        return sigma

    def possibly_quantize_c_noise(self, c_noise):
        return c_noise

    def forward(self, network: nn.Module, input: torch.Tensor, sigma: torch.Tensor, cond: Dict,
                **additional_model_inputs) -> torch.Tensor:
        sigma = self.possibly_quantize_sigma(sigma)
        sigma_shape = sigma.shape
        sigma = append_dims(sigma, input.ndim)
        c_skip, c_out, c_in, c_noise = self.scaling(sigma)
        c_noise = self.possibly_quantize_c_noise(c_noise.reshape(sigma_shape))
        return network(input * c_in, c_noise, cond, **additional_model_inputs) * c_out + input * c_skip


class IdentityWrapper(nn.Module):
    def __init__(self, diffusion_model, compile_model: bool = False):
        super().__init__()
        if compile_model:
            raise NotImplementedError("torch.compile is not part of the H100 path (explicit kernels + CUDA graphs)")
        self.diffusion_model = diffusion_model

    def forward(self, *args, **kwargs):
        return self.diffusion_model(*args, **kwargs)


class OpenAIWrapper(IdentityWrapper):
    def forward(self, x: torch.Tensor, t: torch.Tensor, c: dict, **kwargs) -> torch.Tensor:
        x = torch.cat((x, c.get("concat", torch.Tensor([]).type_as(x)).to(x.dtype)), dim=1)
        return self.diffusion_model(x, timesteps=t, context=c.get("crossattn", None), y=c.get("vector", None), **kwargs)


# ------------------------------------------------------------------------------------------------------------
# guiders
# ------------------------------------------------------------------------------------------------------------
class IdentityGuider:
    def __call__(self, x, sigma):
        return x

    def prepare_inputs(self, x, s, c, uc):
        return x, s, {k: c[k] for k in c}


class VanillaCFG:
    def __init__(self, scale: float):
        self.scale = scale

    def __call__(self, x, sigma):
        x_u, x_c = x.chunk(2)
        return x_u + self.scale * (x_c - x_u)

    def prepare_inputs(self, x, s, c, uc):
        c_out = dict()
        for k in c:
            if k in ["vector", "crossattn", "concat"]:
                c_out[k] = torch.cat((uc[k], c[k]), 0)
            else:
                assert c[k] == uc[k]
                c_out[k] = c[k]
        return torch.cat([x] * 2), torch.cat([s] * 2), c_out


class LinearPredictionGuider:
    def __init__(self, max_scale: float, num_frames: int, min_scale: float = 1.0,
                 additional_cond_keys: Optional[Union[List[str], str]] = None):
        self.min_scale, self.max_scale, self.num_frames = min_scale, max_scale, num_frames
        self.scale = torch.linspace(min_scale, max_scale, num_frames).unsqueeze(0)
        additional_cond_keys = default(additional_cond_keys, [])
        if isinstance(additional_cond_keys, str):
            additional_cond_keys = [additional_cond_keys]
        self.additional_cond_keys = additional_cond_keys

    def __call__(self, x: torch.Tensor, sigma: torch.Tensor) -> torch.Tensor:
        x_u, x_c = x.chunk(2)
        T = self.num_frames
        x_u = x_u.reshape(-1, T, *x_u.shape[1:])
        x_c = x_c.reshape(-1, T, *x_c.shape[1:])
        scale = append_dims(self.scale.expand(x_u.shape[0], T), x_u.ndim).to(x_u.device)
        out = x_u + scale * (x_c - x_u)
        return out.reshape(-1, *out.shape[2:])

    def prepare_inputs(self, x, s, c, uc) -> Tuple[torch.Tensor, torch.Tensor, dict]:
        c_out = dict()
        for k in c:
            if k in ["vector", "crossattn", "concat"] + self.additional_cond_keys:
                c_out[k] = torch.cat((uc[k], c[k]), 0)
            else:
                assert c[k] == uc[k]
                c_out[k] = c[k]
        return torch.cat([x] * 2), torch.cat([s] * 2), c_out


# ------------------------------------------------------------------------------------------------------------
# fused binding
# ------------------------------------------------------------------------------------------------------------
class FusedDenoiser:
    """The pipelines' closure `lambda input, sigma, c: model.denoiser(model.model, input, sigma, c, **kw)`
    (pipeline_i2v_eval_v01.py:85-88) as an inspectable object, so the sampler can run the fused H100 step.
    Calling it behaves exactly like the closure (generic path)."""

    def __init__(self, denoiser: Denoiser, network: nn.Module, shard: Optional[Tuple[int, int]] = None,
                 **additional_model_inputs):
        self.denoiser, self.network, self.kwargs = denoiser, network, additional_model_inputs
        # shard = (rank, world): the caller passes only this rank's frames of x / cond['concat'] (frame sharding over
        # GPUs, SURVEY 8e); num_video_frames stays the GLOBAL frame count
        self.shard = None if shard is None or shard[1] == 1 else (int(shard[0]), int(shard[1]))

    def __call__(self, input, sigma, c):
        if self.shard is not None:
            raise NotImplementedError("a frame-sharded FusedDenoiser can only be evaluated by the fused Euler step "
                                      "(the generic closure has no cross-rank exchanges)")
        return self.denoiser(self.network, input, sigma, c, **self.kwargs)

    def fusable(self) -> bool:
        return (isinstance(self.denoiser.scaling, VScalingWithEDMcNoise) and isinstance(self.network, OpenAIWrapper)
                and isinstance(self.network.diffusion_model, VideoUNet) and "num_video_frames" in self.kwargs)


class _FusedState:
    """Per-(shape, guider) fused network evaluation bound to one VideoUNet launch plan.  `scale` is the guider's CFG scale per
    frame ([T] for LinearPredictionGuider, [1] for VanillaCFG) or None for IdentityGuider, whose plan holds F rows (the
    conditional half only) instead of 2F."""

    def __init__(self, unet: VideoUNet, F_: int, H: int, W: int, T: int, scale: Optional[torch.Tensor], shard=None):
        self.guided = scale is not None
        self.plan = unet.get_plan((2 if self.guided else 1) * F_, H, W, T, shard=shard)
        dev = unet.device
        self.scale = None if scale is None else scale.reshape(-1).to(device=dev, dtype=torch.float32).contiguous()
        self.key = None
        self.cc = self.cuc = None
        # CUDA-graph replay of every kind of evaluation (pre -> ~750 launches -> post), one graph per kind, all reading and
        # writing the static buffers below.  Frame-sharded plans are captured too when their exchanges are peer-memory
        # kernels (every rank replays the same graph, the flag barriers inside it keep the ranks in step); with NCCL
        # exchanges the evaluations stay eager.
        self.use_graph = os.environ.get("HI3D_CUDA_GRAPH", "1") != "0" and (shard is None or self.plan.exchange_mode == "peer")
        self._graphs: Dict[tuple, Tuple[torch.cuda.CUDAGraph, int]] = {}
        self._gx, self._gxo, self._gden, self._gxh, self._geps = (torch.zeros(F_, 4, H, W, dtype=torch.float32, device=dev)
                                                                  for _ in range(5))
        self._gs, self._gst, self._gsf, self._gsu, self._gsn = (torch.ones(F_, dtype=torch.float32, device=dev)
                                                                for _ in range(5))

    def set_conditioning(self, c: dict, uc: dict):
        if self.guided:
            ctx = torch.cat((uc["crossattn"], c["crossattn"]), 0)
            y = torch.cat((uc["vector"], c["vector"]), 0)
        else:                                   # IdentityGuider.prepare_inputs: the conditional rows alone
            ctx, y = c["crossattn"], c["vector"]
        self.plan.prepare_conditioning(ctx, y)
        cc, cuc = c.get("concat", None), uc.get("concat", None)
        if cc is None:
            if self.cc is not None:
                self._graphs.clear()
            self.cc = self.cuc = None
            return
        dt = cc.dtype if cc.dtype in (torch.float16, torch.float32) else torch.float32
        if self.cc is None or self.cc.shape != cc.shape or self.cc.dtype != dt:
            # persistent copies: their addresses are baked into the captured graphs
            self.cc, self.cuc = torch.empty_like(cc, dtype=dt).contiguous(), torch.empty_like(cc, dtype=dt).contiguous()
            self._graphs.clear()
        self.cc.copy_(cc)
        if cuc is None or not self.guided:
            self.cuc.zero_()
        else:
            self.cuc.copy_(cuc)

    @staticmethod
    def cond_key(c: dict, uc: dict):
        return tuple((k, d[k].data_ptr(), d[k]._version, tuple(d[k].shape)) for d in (c, uc) for k in sorted(d)
                     if torch.is_tensor(d[k]))

    def noise_buffer(self) -> Optional[torch.Tensor]:
        """Where a sampler draws the step's noise before a replay (the graphs read it from there), or None when eager."""
        return self._geps if self.use_graph else None

    def _launch(self, x, sigma, sigma_to, x_out, den, churn=None, noise=None):
        """pre -> launch plan -> post.  churn = (sigma_from, eps, s_noise, x_hat): the network sees the churned x_hat at sigma
        and the update starts from it.  noise = (eps, s_noise, sigma_up, sigma_next): the ancestral noise of the update.
        The CFG-guided Euler evaluation keeps hi3d_sampler_pre / hi3d_sampler_post."""
        plan = self.plan
        F_, Cx, H, W = x.shape
        xin = plan.xin.t.view(-1, H, W, CIN_PAD)
        if self.guided and churn is None:
            ops.sampler_pre(x, sigma, self.cuc, self.cc, xin, c_noise_out=plan.t_in)
        else:
            ops.sampler_pre_ex(x, sigma, self.cuc, self.cc, xin, self.guided, c_noise_out=plan.t_in, churn=churn)
        plan.run()
        xp = x if churn is None else churn[3]
        if self.guided and noise is None:
            ops.sampler_post(plan.net_out.t, xp, sigma, sigma_to, self.scale, x_out, den)
        else:
            ops.sampler_post_ancestral(plan.net_out.t, xp, sigma, sigma_to, self.scale, x_out, den, noise)

    def run(self, x: torch.Tensor, sigma: torch.Tensor, sigma_to: torch.Tensor, want_denoised: bool = False,
            churn: Optional[tuple] = None, noise: Optional[tuple] = None):
        """One network evaluation and its update x + (x - D)/sigma * (sigma_to - sigma): returns (x_out, D or None, x_hat or
        None).  churn = (sigma_from, eps, s_noise) and noise = (eps, s_noise, sigma_up, sigma_next) as in `_launch`.  With
        graphs on, the inputs are copied into the static buffers (eps is drawn there directly when it is `noise_buffer()`)
        and the graph of this kind of call is replayed; it is captured on first use."""
        if self.use_graph and x.shape == self._gx.shape:
            key = (want_denoised, None if churn is None else float(churn[2]), None if noise is None else float(noise[1]))
            self._gx.copy_(x)
            self._gs.copy_(sigma)
            self._gst.copy_(sigma_to)
            eps = churn[1] if churn is not None else noise[0] if noise is not None else None
            if eps is not None and eps.data_ptr() != self._geps.data_ptr():
                self._geps.copy_(eps)
            g_churn = g_noise = None
            if churn is not None:
                self._gsf.copy_(churn[0])
                g_churn = (self._gsf, self._geps, float(churn[2]), self._gxh)
            if noise is not None:
                self._gsu.copy_(noise[2])
                self._gsn.copy_(noise[3])
                g_noise = (self._geps, float(noise[1]), self._gsu, self._gsn)
            args = (self._gx, self._gs, self._gst, self._gxo, self._gden if want_denoised else None, g_churn, g_noise)
            if key not in self._graphs:
                self._launch(*args)                  # eager warm-up (lazy one-time init)
                torch.cuda.synchronize()
                g = torch.cuda.CUDAGraph()
                n0 = _native.launch_count()
                with torch.cuda.graph(g):
                    self._launch(*args)
                n = _native.launch_count() - n0
                _native.note_graph_replay(-n)        # capture-time calls did not execute
                self._graphs[key] = (g, n)
            g, n = self._graphs[key]
            g.replay()
            _native.note_graph_replay(n)
            return (self._gxo.clone(), self._gden.clone() if want_denoised else None,
                    self._gxh.clone() if churn is not None else None)
        x = x.contiguous()
        x_out = torch.empty_like(x)
        den = torch.empty_like(x) if want_denoised else None
        x_hat = None
        if churn is not None:
            x_hat = torch.empty_like(x)
            churn = (churn[0].contiguous(), churn[1].contiguous(), churn[2], x_hat)
        if noise is not None:
            noise = (noise[0].contiguous(), noise[1], noise[2].contiguous(), noise[3].contiguous())
        self._launch(x, sigma.contiguous(), sigma_to.contiguous(), x_out, den, churn, noise)
        return x_out, den, x_hat

    def denoise(self, x: torch.Tensor, sigma: torch.Tensor, churn: Optional[tuple] = None):
        """Guided denoised latents D(x, sigma) on the fused path: the network evaluation of ANY sampler (Heun's second
        evaluation, DPM-Solver++), without the update.  With churn = (sigma_from, eps, s_noise) returns (D, x_hat)."""
        _, den, x_hat = self.run(x, sigma, sigma, True, churn)
        return den if churn is None else (den, x_hat)

    def step(self, x: torch.Tensor, sigma: torch.Tensor, next_sigma: torch.Tensor, want_denoised: bool = False):
        x_out, den, _ = self.run(x, sigma, next_sigma, want_denoised)
        return (x_out, den) if want_denoised else x_out


# ------------------------------------------------------------------------------------------------------------
# samplers
# ------------------------------------------------------------------------------------------------------------
DEFAULT_GUIDER = {"target": "sgm.modules.diffusionmodules.guiders.IdentityGuider"}


class BaseDiffusionSampler:
    def __init__(self, discretization_config, num_steps: Union[int, None] = None, guider_config=None,
                 verbose: bool = False, device: str = "cuda"):
        self.num_steps = num_steps
        self.discretization = instantiate_from_config(discretization_config)
        self.guider = instantiate_from_config(default(guider_config, DEFAULT_GUIDER))
        self.verbose = verbose
        self.device = device
        self._fused: Dict[tuple, _FusedState] = {}
        self.noise_sampler = lambda x: torch.randn_like(x)
        # one generator per object (frames object-major): each stochastic step draws object i's noise from generator i, so an
        # object's result does not depend on the batch it is sampled in.  None: `noise_sampler`, i.e. the global generator.
        self.noise_generators: Optional[List[torch.Generator]] = None

    def draw_noise(self, x: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """This step's eps ~ N(0, 1) in the shape of x, written to `out` when given."""
        gens = self.noise_generators
        if not gens:
            e = self.noise_sampler(x)
            return e if out is None else out.copy_(e)
        if x.shape[0] % len(gens):
            raise ValueError(f"{x.shape[0]} frames cannot be split over {len(gens)} objects")
        out = torch.empty_like(x) if out is None else out
        n = x.shape[0] // len(gens)
        for i, g in enumerate(gens):
            out[i * n:(i + 1) * n].normal_(generator=g)
        return out

    def prepare_sampling_loop(self, x, cond, uc=None, num_steps=None):
        sigmas = self.discretization(self.num_steps if num_steps is None else num_steps, device=self.device)
        uc = default(uc, cond)
        x *= torch.sqrt(1.0 + sigmas[0] ** 2.0)
        num_sigmas = len(sigmas)
        s_in = x.new_ones([x.shape[0]])
        return x, s_in, sigmas, num_sigmas, cond, uc

    def denoise(self, x, denoiser, sigma, cond, uc):
        """sampling.py:54-57.  When `denoiser` is a fusable binding the guided D(x, sigma) comes from the fused kernels (one
        network evaluation = sampler_pre -> launch plan -> sampler_post), whatever the solver around it is."""
        st = self._fused_state(denoiser, x, cond, default(uc, cond), refresh=False)
        if st is not None:
            return st.denoise(x, sigma)
        if isinstance(denoiser, FusedDenoiser) and denoiser.shard is not None:
            raise NotImplementedError("frame-sharded sampling needs the fused path (LinearPredictionGuider + "
                                      f"VScalingWithEDMcNoise, fp32 CUDA latents); got {type(self.guider).__name__}, x {x.dtype}")
        denoised = denoiser(*self.guider.prepare_inputs(x, sigma, cond, uc))
        return self.guider(denoised, sigma)

    # -- fused path (shared by every sampler) -------------------------------------------------------------------
    frame_sharded = False        # whether the sampler runs frame-sharded plans (those that ran them before the other samplers)

    def _fused_state(self, denoiser, x, cond, uc, refresh: bool) -> Optional[_FusedState]:
        if not (isinstance(denoiser, FusedDenoiser) and denoiser.fusable() and x.is_cuda and x.dtype == torch.float32):
            return None
        unet = denoiser.network.diffusion_model
        T = int(denoiser.kwargs["num_video_frames"])
        shard = denoiser.shard
        g = self.guider
        if shard is not None and not (self.frame_sharded and isinstance(g, LinearPredictionGuider)):
            raise NotImplementedError(f"frame-sharded sampling runs EulerEDMSampler, HeunEDMSampler and DPMPP2MSampler with "
                                      f"LinearPredictionGuider; got {type(self).__name__} with {type(g).__name__}")
        if isinstance(g, LinearPredictionGuider):
            if T != g.num_frames:
                return None
            scale = g.scale.reshape(-1)
        elif isinstance(g, VanillaCFG):
            scale = torch.tensor([float(g.scale)])
        elif isinstance(g, IdentityGuider):
            scale = None
        else:
            return None
        if shard is not None:             # this rank holds frames [rank*Tl, (rank+1)*Tl) of every clip
            if T % shard[1]:
                raise ValueError(f"{T} frames cannot be sharded over {shard[1]} ranks")
            Tl = T // shard[1]
            scale = scale[shard[0] * Tl:(shard[0] + 1) * Tl]
            T = Tl
        if x.shape[0] % T:
            return None
        F_, _, H, W = x.shape
        rows = F_ if scale is None else 2 * F_
        key = (id(unet), F_, H, W, T, unet.engine, shard, rows)
        pkey = (rows, H, W, T, unet.engine) if shard is None else (rows, H, W, T, unet.engine, shard)
        st = self._fused.get(key)
        if st is None or st.plan is not unet._plans.get(pkey):
            st = self._fused[key] = _FusedState(unet, F_, H, W, T, scale, shard)
        ck = _FusedState.cond_key(cond, uc)
        if refresh or st.key != ck:
            st.set_conditioning(cond, uc)
            st.key = ck
        return st

    def get_sigma_gen(self, num_sigmas):
        sigma_generator = range(num_sigmas - 1)
        if self.verbose:
            try:
                from tqdm import tqdm
                sigma_generator = tqdm(sigma_generator, total=num_sigmas,
                                       desc=f"Sampling with {self.__class__.__name__} for {num_sigmas} steps")
            except ImportError:
                pass
        return sigma_generator


class SingleStepDiffusionSampler(BaseDiffusionSampler):
    def sampler_step(self, sigma, next_sigma, denoiser, x, cond, uc, *args, **kwargs):
        raise NotImplementedError

    def euler_step(self, x, d, dt):
        return x + dt * d


class EDMSampler(SingleStepDiffusionSampler):
    frame_sharded = True

    def __init__(self, s_churn=0.0, s_tmin=0.0, s_tmax=float("inf"), s_noise=1.0, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.s_churn, self.s_tmin, self.s_tmax, self.s_noise = s_churn, s_tmin, s_tmax, s_noise

    def _gamma(self, sigmas, i, num_sigmas):
        if self.s_churn == 0.0:       # avoids the reference's per-step D2H sync (sampling.py:112,134)
            return 0.0
        return min(self.s_churn / (num_sigmas - 1), 2 ** 0.5 - 1) if self.s_tmin <= sigmas[i] <= self.s_tmax else 0.0

    def possible_correction_step(self, euler_step, x, d, dt, next_sigma, denoiser, cond, uc):
        return euler_step

    def sampler_step(self, sigma, next_sigma, denoiser, x, cond, uc=None, gamma=0.0, _refresh=False):
        st = self._fused_state(denoiser, x, cond, default(uc, cond), _refresh)
        sigma_hat = sigma if gamma == 0 else sigma * (gamma + 1.0)
        churn = None
        if gamma > 0:
            if st is not None and denoiser.shard is None:
                # x_hat = x + s_noise sqrt(sigma_hat^2 - sigma^2) eps inside the pre kernel, eps drawn before the replay
                churn = (sigma, self.draw_noise(x, st.noise_buffer()), self.s_noise)
            else:
                eps = self.draw_noise(x) * self.s_noise
                x = x + eps * append_dims(sigma_hat ** 2 - sigma ** 2, x.ndim) ** 0.5
        if st is not None and type(self).possible_correction_step is EDMSampler.possible_correction_step:
            return st.run(x, sigma_hat, next_sigma, churn=churn)[0]
        if churn is not None:
            denoised, x = st.denoise(x, sigma_hat, churn)
        else:
            denoised = self.denoise(x, denoiser, sigma_hat, cond, uc)
        d = (x - denoised) / append_dims(sigma_hat, x.ndim)            # to_d, sampling_utils.py:34
        dt = append_dims(next_sigma - sigma_hat, x.ndim)
        self._heun_ctx = (next_sigma - sigma_hat).float().contiguous() if x.is_cuda else None
        euler_step = self.euler_step(x, d, dt)
        return self.possible_correction_step(euler_step, x, d, dt, next_sigma, denoiser, cond, uc)

    def step_call(self, denoiser, x, i, s_in, sigmas, num_sigmas, cond, uc):
        """Hi3D addition (sampling.py:109-124): one externally driven step of the loop."""
        gamma = self._gamma(sigmas, i, num_sigmas)
        return self.sampler_step(s_in * sigmas[i], s_in * sigmas[i + 1], denoiser, x, cond, uc, gamma,
                                 _refresh=(i == 0))

    def __call__(self, denoiser, x, cond, uc=None, num_steps=None):
        x, s_in, sigmas, num_sigmas, cond, uc = self.prepare_sampling_loop(x, cond, uc, num_steps)
        for i in self.get_sigma_gen(num_sigmas):
            gamma = self._gamma(sigmas, i, num_sigmas)
            x = self.sampler_step(s_in * sigmas[i], s_in * sigmas[i + 1], denoiser, x, cond, uc, gamma,
                                  _refresh=(i == 0))
        return x


class EulerEDMSampler(EDMSampler):
    """sampling.py:228-232: EDMSampler whose correction step is the identity (inherited)."""


# ------------------------------------------------------------------------------------------------------------
# SURVEY §8(f) N4: the two other samplers of the sgm surface that Hi3D-style configs can name.  Every network evaluation goes
# through `self.denoise`, i.e. the fused sampler_pre -> launch plan -> sampler_post kernels when the denoiser binding is fusable
# (guider, Denoiser scalings and the OpenAIWrapper concat included); the solver algebra on the (F, 4, h, w) fp32 state is one
# hi3d_sampler_lincomb4 launch per update on CUDA (plain tensor expressions on CPU, where they are checked against the
# unmodified reference classes).
# ------------------------------------------------------------------------------------------------------------
class HeunEDMSampler(EDMSampler):
    """sampling.py:236-254.  Second order: the slope at (x, sigma_hat) is averaged with the slope at the Euler point
    (x_e, sigma_next); the last step (sigma_next = 0) stays first order, which also saves one evaluation."""

    def possible_correction_step(self, euler_step, x, d, dt, next_sigma, denoiser, cond, uc):
        if float(next_sigma.sum()) < 1e-14:
            return euler_step
        sig_n = append_dims(next_sigma, x.ndim)
        den_next = self.denoise(euler_step, denoiser, next_sigma, cond, uc)
        if x.is_cuda and x.dtype == torch.float32 and getattr(self, "_heun_ctx", None) is not None:
            # x + dt/2 (d + d'),  d' = (x_e - D')/sigma':  one hi3d_sampler_lincomb4 launch over (x, d, x_e, D')
            dtv = self._heun_ctx                                                  # dt per sample, fp32 [F]
            h = 0.5 * dtv
            one = torch.ones_like(dtv)
            return ops.sampler_lincomb(torch.empty_like(x), [(x.contiguous(), one), (d.contiguous(), h),
                                                             (euler_step.contiguous(), h / next_sigma),
                                                             (den_next.contiguous(), -h / next_sigma)])
        d_next = (euler_step - den_next) / sig_n
        heun = x + (d + d_next) / 2.0 * dt
        return torch.where(sig_n > 0.0, heun, euler_step)


class DPMPP2MSampler(BaseDiffusionSampler):
    """sampling.py:305-379 (DPM-Solver++(2M), Lu et al. 2022) in t = -log(sigma): one evaluation per step; from the
    second step on the denoised estimate is extrapolated with the previous one (ratio r of the two log-step sizes)."""
    frame_sharded = True

    @staticmethod
    def _t(sigma):                       # sampling_utils.py: to_neg_log_sigma
        return sigma.log().neg()

    @staticmethod
    def _sigma(t):                       # sampling_utils.py: to_sigma
        return t.neg().exp()

    def sampler_step(self, old_denoised, previous_sigma, sigma, next_sigma, denoiser, x, cond, uc=None):
        denoised = self.denoise(x, denoiser, sigma, cond, uc)
        t, t_next = self._t(sigma), self._t(next_sigma)
        h = t_next - t
        keep = append_dims(self._sigma(t_next) / self._sigma(t), x.ndim)     # sigma_next / sigma
        gain = append_dims((-h).expm1(), x.ndim)                             # exp(-h) - 1 <= 0
        fused = x.is_cuda and x.dtype == torch.float32
        if old_denoised is None or float(next_sigma.sum()) < 1e-14:
            if fused:        # (sigma'/sigma) x - expm1(-h) D : one hi3d_sampler_lincomb4 launch
                k1, g1 = (self._sigma(t_next) / self._sigma(t)).float().contiguous(), (-(-h).expm1()).float().contiguous()
                return ops.sampler_lincomb(torch.empty_like(x), [(x.contiguous(), k1), (denoised.contiguous(), g1)]), denoised
            return keep * x - gain * denoised, denoised
        r = (t - self._t(previous_sigma)) / h
        if fused:            # (sigma'/sigma) x - expm1(-h) ((1 + 1/(2r)) D - 1/(2r) D_old)
            k1, g1 = (self._sigma(t_next) / self._sigma(t)).float().contiguous(), (-(-h).expm1()).float()
            return ops.sampler_lincomb(torch.empty_like(x), [(x.contiguous(), k1),
                                                             (denoised.contiguous(), (g1 * (1 + 1 / (2 * r))).contiguous()),
                                                             (old_denoised.contiguous(), (-g1 / (2 * r)).contiguous())]), denoised
        x_first = keep * x - gain * denoised
        w_new, w_old = append_dims(1 + 1 / (2 * r), x.ndim), append_dims(1 / (2 * r), x.ndim)
        x_second = keep * x - gain * (w_new * denoised - w_old * old_denoised)
        return torch.where(append_dims(next_sigma, x.ndim) > 0.0, x_second, x_first), denoised

    def __call__(self, denoiser, x, cond, uc=None, num_steps=None, **kwargs):
        x, s_in, sigmas, num_sigmas, cond, uc = self.prepare_sampling_loop(x, cond, uc, num_steps)
        prev_d = None
        for i in self.get_sigma_gen(num_sigmas):
            x, prev_d = self.sampler_step(prev_d, None if i == 0 else s_in * sigmas[i - 1], s_in * sigmas[i],
                                          s_in * sigmas[i + 1], denoiser, x, cond, uc=uc)
        return x


# ------------------------------------------------------------------------------------------------------------
# The ancestral and linear multistep samplers of the sgm surface (sampling.py:150-226, 254-302).  On the fused path every network
# evaluation is a graph replay; the Euler ancestral step is ONE replay (hi3d_sampler_post_ancestral adds the noise), and the
# solver algebra of DPM-Solver++(2S) and LMS is one hi3d_sampler_lincomb launch per update.
# ------------------------------------------------------------------------------------------------------------
def ancestral_sigmas(sigma_from: torch.Tensor, sigma_to: torch.Tensor, eta: float = 1.0):
    """The ancestral split of a step from sigma_from to sigma_to (Karras et al. 2022, k-diffusion): the deterministic part goes
    to sigma_down, and fresh noise of standard deviation sigma_up brings it back to sigma_to (sigma_down^2 + sigma_up^2 =
    sigma_to^2).  eta = 0 gives the deterministic step."""
    if not eta:
        return sigma_to, torch.zeros_like(sigma_to)
    up = (sigma_to ** 2 * (sigma_from ** 2 - sigma_to ** 2) / sigma_from ** 2) ** 0.5 * eta
    sigma_up = torch.minimum(sigma_to, up)
    return (sigma_to ** 2 - sigma_up ** 2) ** 0.5, sigma_up


def lms_coefficients(sigmas, i: int, order: int) -> List[float]:
    """Linear multistep weights of step i: c_j = integral over [sigma_i, sigma_{i+1}] of the Lagrange basis polynomial through
    sigma_i, ..., sigma_{i-order+1} that is 1 at sigma_{i-j}.  The integrand has degree order - 1, so Gauss-Legendre quadrature
    with `order` nodes is exact."""
    import numpy as np
    if order - 1 > i:
        raise ValueError(f"order {order} too high for step {i}")
    s = [float(v) for v in sigmas]
    a, b = s[i], s[i + 1]
    nodes, weights = np.polynomial.legendre.leggauss(max(order, 1))
    tau = 0.5 * (b - a) * nodes + 0.5 * (a + b)
    out = []
    for j in range(order):
        basis = np.ones_like(tau)
        for k in range(order):
            if k != j:
                basis *= (tau - s[i - k]) / (s[i - j] - s[i - k])
        out.append(float(0.5 * (b - a) * np.dot(weights, basis)))
    return out


def _lincomb(terms) -> torch.Tensor:
    """sum_k c_k x_k over any number of (x_k, c_k [F]) terms: hi3d_sampler_lincomb, 8 terms per launch."""
    out = ops.sampler_lincomb8(torch.empty_like(terms[0][0]), terms[:8])
    rest = terms[8:]
    while rest:
        out = ops.sampler_lincomb8(out, [(out, torch.ones_like(terms[0][1]))] + rest[:7])
        rest = rest[7:]
    return out


class AncestralSampler(SingleStepDiffusionSampler):
    """sampling.py:150-187."""

    def __init__(self, eta=1.0, s_noise=1.0, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.eta, self.s_noise = eta, s_noise

    def ancestral_euler_step(self, x, denoised, sigma, sigma_down):
        return self.euler_step(x, (x - denoised) / append_dims(sigma, x.ndim), append_dims(sigma_down - sigma, x.ndim))

    def ancestral_step(self, x, sigma, next_sigma, sigma_up):
        noised = x + self.draw_noise(x) * self.s_noise * append_dims(sigma_up, x.ndim)
        return torch.where(append_dims(next_sigma, x.ndim) > 0.0, noised, x)

    def __call__(self, denoiser, x, cond, uc=None, num_steps=None):
        x, s_in, sigmas, num_sigmas, cond, uc = self.prepare_sampling_loop(x, cond, uc, num_steps)
        self._fused_state(denoiser, x, cond, uc, refresh=True)
        for i in self.get_sigma_gen(num_sigmas):
            x = self.sampler_step(s_in * sigmas[i], s_in * sigmas[i + 1], denoiser, x, cond, uc)
        return x


class EulerAncestralSampler(AncestralSampler):
    """sampling.py:254-261: Euler to sigma_down, then noise up to sigma_next; on the fused path one graph replay a step."""

    def sampler_step(self, sigma, next_sigma, denoiser, x, cond, uc=None):
        sigma_down, sigma_up = ancestral_sigmas(sigma, next_sigma, self.eta)
        st = self._fused_state(denoiser, x, cond, default(uc, cond), refresh=False)
        if st is not None:
            eps = self.draw_noise(x, st.noise_buffer())
            return st.run(x, sigma, sigma_down, noise=(eps, self.s_noise, sigma_up, next_sigma))[0]
        denoised = self.denoise(x, denoiser, sigma, cond, uc)
        x = self.ancestral_euler_step(x, denoised, sigma, sigma_down)
        return self.ancestral_step(x, sigma, next_sigma, sigma_up)


class DPMPP2SAncestralSampler(AncestralSampler):
    """sampling.py:264-301: DPM-Solver++(2S) to sigma_down (a second evaluation at the log-midpoint), then ancestral noise."""

    def sampler_step(self, sigma, next_sigma, denoiser, x, cond, uc=None, **kwargs):
        sigma_down, sigma_up = ancestral_sigmas(sigma, next_sigma, self.eta)
        st = self._fused_state(denoiser, x, cond, default(uc, cond), refresh=False)
        if st is not None:
            eps = self.draw_noise(x)
            x_euler, denoised, _ = st.run(x, sigma, sigma_down, want_denoised=True)
        else:
            denoised = self.denoise(x, denoiser, sigma, cond, uc)
            x_euler = self.ancestral_euler_step(x, denoised, sigma, sigma_down)
        second = float(sigma_down.sum()) >= 1e-14          # saves the second evaluation when every sigma_down is 0
        if second:
            t, t_down = sigma.log().neg(), sigma_down.log().neg()
            h = t_down - t
            sigma_mid = (t + 0.5 * h).neg().exp()
            k_mid, g_mid = sigma_mid / sigma, (-0.5 * h).expm1()
            k_down, g_down = sigma_down / sigma, (-h).expm1()
        if st is None:
            if second:
                x2 = append_dims(k_mid, x.ndim) * x - append_dims(g_mid, x.ndim) * denoised
                denoised2 = self.denoise(x2, denoiser, sigma_mid, cond, uc)
                x_2s = append_dims(k_down, x.ndim) * x - append_dims(g_down, x.ndim) * denoised2
                x_euler = torch.where(append_dims(sigma_down, x.ndim) > 0.0, x_2s, x_euler)
            return self.ancestral_step(x_euler, sigma, next_sigma, sigma_up)
        f32 = lambda v: v.float().contiguous()                                         # noqa: E731
        noise = f32(self.s_noise * sigma_up * (next_sigma > 0.0))
        if not second:
            return _lincomb([(x_euler, f32(torch.ones_like(sigma))), (eps, noise)])
        x2 = _lincomb([(x, f32(k_mid)), (denoised, f32(-g_mid))])
        denoised2 = st.denoise(x2, f32(sigma_mid))
        sel = f32(sigma_down > 0.0)
        # where(sigma_down > 0, (sigma_down/sigma) x - expm1(-h) D2, x_euler) + s_noise sigma_up eps [sigma_next > 0]
        return _lincomb([(x, f32(k_down) * sel), (x_euler, 1.0 - sel), (denoised2, -f32(g_down) * sel), (eps, noise)])


class LinearMultistepSampler(BaseDiffusionSampler):
    """sampling.py:190-225: linear multistep of `order` over the slopes d = (x - D)/sigma of the last steps.  On the fused path
    the slopes are never formed: the update is one launch over the (x, D) pairs of the last `order` steps (8 terms at order 4)."""

    def __init__(self, order=4, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.order = order

    def __call__(self, denoiser, x, cond, uc=None, num_steps=None, **kwargs):
        x, s_in, sigmas, num_sigmas, cond, uc = self.prepare_sampling_loop(x, cond, uc, num_steps)
        st = None if kwargs else self._fused_state(denoiser, x, cond, uc, refresh=True)
        sig = sigmas.detach().cpu().numpy()
        hist = []                                          # (x_j, D_j, sigma_j) or d_j, newest last
        for i in self.get_sigma_gen(num_sigmas):
            sigma = s_in * sigmas[i]
            coeffs = lms_coefficients(sig, i, min(i + 1, self.order))
            if st is not None:
                denoised = st.denoise(x, sigma)
                hist = (hist + [(x, denoised, float(sig[i]))])[-self.order:]
                terms = [(x, 1.0)]
                for c, (xj, dj, sj) in zip(coeffs, reversed(hist)):
                    terms += [(xj, c / sj), (dj, -c / sj)]
                terms[1] = (terms[1][0], terms[0][1] + terms[1][1])           # x_i appears twice: one coefficient
                terms = terms[1:]
                x = _lincomb([(t, torch.full_like(sigma, w)) for t, w in terms])
                continue
            if kwargs:
                denoised = self.guider(denoiser(*self.guider.prepare_inputs(x, sigma, cond, uc), **kwargs), sigma)
            else:
                denoised = self.denoise(x, denoiser, sigma, cond, uc)
            hist = (hist + [(x - denoised) / append_dims(sigma, x.ndim)])[-self.order:]
            x = x + sum(c * d for c, d in zip(coeffs, reversed(hist)))
        return x


# ------------------------------------------------------------------------------------------------------------
# the pipelines' --sampler / --steps / --guidance / --cfg_scale / --s_churn / --eta
# ------------------------------------------------------------------------------------------------------------
SAMPLER_CHOICES = {"euler": EulerEDMSampler, "heun": HeunEDMSampler, "dpmpp2m": DPMPP2MSampler,
                   "euler_ancestral": EulerAncestralSampler, "dpmpp2s_ancestral": DPMPP2SAncestralSampler,
                   "lms": LinearMultistepSampler}
GUIDANCE_CHOICES = ("config", "linear", "vanilla", "none")


def configure_sampler(base: BaseDiffusionSampler, sampler: str = "config", steps: Optional[int] = None,
                      guidance: str = "config", cfg_scale: Optional[float] = None, s_churn: Optional[float] = None,
                      eta: Optional[float] = None, num_frames: Optional[int] = None) -> BaseDiffusionSampler:
    """The model's sampler with the command line's choices applied; `base` itself when every choice is 'config' / None.
    The discretisation, the noise range and the guidance scales not overridden are the configuration's."""
    if sampler == "config" and steps is None and guidance == "config" and cfg_scale is None and s_churn is None and eta is None:
        return base
    cls = type(base) if sampler == "config" else SAMPLER_CHOICES[sampler]
    old = base.guider
    if guidance == "config":
        if cfg_scale is not None:
            raise ValueError("--cfg_scale needs --guidance linear or vanilla")
        guider = old
    elif guidance == "none":
        if cfg_scale is not None:
            raise ValueError("--guidance none has no scale")
        guider = IdentityGuider()
    else:
        max_scale = cfg_scale if cfg_scale is not None else getattr(old, "max_scale", getattr(old, "scale", None))
        if not isinstance(max_scale, (int, float)):
            raise ValueError(f"--guidance {guidance} needs --cfg_scale (the configuration's guider has no scale)")
        if guidance == "vanilla":
            guider = VanillaCFG(float(max_scale))
        else:
            frames = num_frames if num_frames is not None else getattr(old, "num_frames", None)
            if frames is None:
                raise ValueError("--guidance linear needs the number of frames")
            guider = LinearPredictionGuider(float(max_scale), int(frames), min_scale=getattr(old, "min_scale", 1.0))
    kw = {}
    if issubclass(cls, EDMSampler):
        if eta is not None:
            raise ValueError(f"--eta applies to the ancestral samplers, not {cls.__name__}")
        kw = dict(s_churn=getattr(base, "s_churn", 0.0) if s_churn is None else float(s_churn),
                  s_tmin=getattr(base, "s_tmin", 0.0), s_tmax=getattr(base, "s_tmax", float("inf")),
                  s_noise=getattr(base, "s_noise", 1.0))
    elif issubclass(cls, AncestralSampler):
        if s_churn is not None:
            raise ValueError(f"--s_churn applies to the EDM samplers (euler, heun), not {cls.__name__}")
        kw = dict(eta=getattr(base, "eta", 1.0) if eta is None else float(eta), s_noise=getattr(base, "s_noise", 1.0))
    elif s_churn is not None or eta is not None:
        raise ValueError(f"--s_churn / --eta do not apply to {cls.__name__}")
    if cls is LinearMultistepSampler:
        kw["order"] = getattr(base, "order", 4)
    out = cls(discretization_config={"target": "torch.nn.Identity"}, num_steps=base.num_steps if steps is None else int(steps),
              verbose=base.verbose, device=base.device, **kw)
    out.discretization, out.guider = base.discretization, guider
    return out
