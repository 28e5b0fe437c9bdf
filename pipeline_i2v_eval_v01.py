#!/usr/bin/env python
"""Stage-1 entry point, same CLI as the reference's pipeline_i2v_eval_v01.py (:39-45) on the H100 engine.

    python pipeline_i2v_eval_v01.py --denoise_config configs/inference-v01.yaml --denoise_checkpoint ckpts/first_stage.pt \
        --image_path demo/15_out.png --output_dir outputs/15_out --elevation 0  [--cond cond.pt | --synthetic]

The hot path (25-step fused Euler-EDM over VideoUNet + VAE decode) runs here.  The conditioner's image towers (OpenCLIP
ViT-H/14, CLIP ViT-L/14 + aesthetic MLP) run natively when their weights are available -- the reference's files
(ckpts/open_clip_pytorch_model.bin, ckpts/ViT-L-14.pt, ckpts/metric_models/sac+logos+ava1-l14-linearMSE.pth under the working
directory) or their tensors inside the checkpoint -- and then --image_path alone builds c / uc through the model's own
GeneralConditioner, as below.  Otherwise three ways to supply what the towers produce:
  --towers t.pt   {'clip': (1, 1024) image embedding, 'aes': (1, 1) aesthetic score}: the image is pre-processed as in the
                  reference (cv2 resize, centre crop, [-1, 1]; v01:131-149), `add_custom_cond` and the model's own
                  GeneralConditioner (elevation / cond_aug timestep embeddings, VAE-mode latent of the cond frame) build c / uc
                  exactly like v01:62-78;
  --cond c.pt     torch.save({'c': .., 'uc': ..}) from the reference's conditioner.get_unconditional_conditioning;
  --synthetic     seeded stand-ins.
Output: <output_dir>/first_step/first.mp4 (8 fps, like v01:96-98,129) + first.pt (the frames as a tensor, which stage 2
prefers over re-reading the lossy mp4).  Without a checkpoint file the seeded synthetic weights of spec.synth_fill_ are used
(said loudly).  --tiny builds a reduced-width 2-step model: the smoke size the tests execute this script at.

Several images: --image_path a.png b.png ... writes <output_dir>/<image stem>/{temp_image,first_step}; --elevation, --seed and
--towers take one value for all or one per image; --batch K samples K objects per batch (background removal, conditioner
towers, UNet and VAE each run once over the K).  Object i's output is what a run over image i alone with the same seed gives.
"""
import argparse
import os
import random

import torch

from hi3d_official_b200 import configs, spec
from hi3d_official_b200.engine import create_model
from hi3d_official_b200.util import get_obj_from_str


def load_model(config_path, ckpt, stage, tiny=False, precision="fp16"):
    """The stage's DiffusionEngine on the GPU; `precision` = operand precision of the denoising UNet's GEMMs
    (VideoUNet.set_precision), the VAE and the conditioner towers stay fp16."""
    if os.path.exists(config_path) and not tiny:
        model = create_model(config_path)
    else:
        if not tiny:
            print(f"[hi3d-b200] {config_path} not found: using the built-in copy of the stage-{stage} inference config")
        cfg = (configs.stage1_config(True) if stage == 1 else configs.stage2_config(True))["model"]
        if tiny:
            cfg["params"]["network_config"]["params"]["model_channels"] = 64
            cfg["params"]["first_stage_config"]["params"]["ddconfig"]["ch"] = 64
            cfg["params"]["sampler_config"]["params"]["num_steps"] = 2
            for e in cfg["params"]["conditioner_config"]["params"]["emb_models"]:
                if "encoder_config" in e.get("params", {}):
                    e["params"]["encoder_config"]["params"]["ddconfig"]["ch"] = 64
        model = get_obj_from_str(cfg["target"])(**cfg["params"])
    if os.path.exists(ckpt):
        model.init_from_ckpt(ckpt)
        model = model.cuda().half()
    else:
        print(f"[hi3d-b200] checkpoint {ckpt} not found: SEEDED SYNTHETIC WEIGHTS (outputs are not images)")
        model = model.cuda().half()
        spec.synth_fill_(model, seed=0, fast=True)
    model.model.diffusion_model.set_precision(precision)
    return model


def synthetic_cond(stage, T, h, device, seed):
    g = torch.Generator().manual_seed(seed)
    adm, cc = (768, 4) if stage == 1 else (512, 13)
    c = dict(crossattn=torch.randn(1, 1, 1024, generator=g), vector=torch.randn(1, adm, generator=g),
             concat=(torch.randn(T, cc, h, h, generator=g) * 0.18).half())
    c = {k: v.to(device) for k, v in c.items()}
    uc = dict(crossattn=torch.zeros_like(c["crossattn"]), vector=c["vector"].clone(), concat=torch.zeros_like(c["concat"]))
    return c, uc


def save_frames(frames, out_dir, name, fps=8):
    """frames: (T, 3, H, W) in [-1, 1] -> <out_dir>/<name>.mp4 through tensor2vid / export_to_video (vtdm/util.py:12-49,
    v01:96-98) and <out_dir>/<name>.pt."""
    from hi3d_official_b200 import video_io
    os.makedirs(out_dir, exist_ok=True)
    torch.save(frames.cpu(), os.path.join(out_dir, name + ".pt"))
    vid = frames.float().cpu().permute(1, 0, 2, 3)[None]                      # "t c h w -> 1 c t h w"
    return video_io.export_to_video(video_io.tensor2vid(vid.clone()), os.path.join(out_dir, name + ".mp4"), fps=fps)


def load_image(path, size):
    """v01:131-149: cv2 read -> resize so the short side is `size` -> centre crop -> [-1, 1], (3, size, size)."""
    import cv2
    import numpy as np
    img = cv2.cvtColor(cv2.imread(path), cv2.COLOR_BGR2RGB)
    hh, ww = img.shape[:2]
    sc = size / min(hh, ww)
    img = cv2.resize(img, (max(size, round(ww * sc)), max(size, round(hh * sc))), interpolation=cv2.INTER_AREA)
    y0, x0 = (img.shape[0] - size) // 2, (img.shape[1] - size) // 2
    img = img[y0:y0 + size, x0:x0 + size]
    return torch.from_numpy(np.ascontiguousarray(img)).permute(2, 0, 1).float() / 127.5 - 1.0


def remove_background(image_path, output_dir):
    """v01:153-168: rembg.remove with U^2-Net (hi3d_official_b200/rembg.py, weights ckpts/u2net.pth under the working directory),
    the cut-out saved as <output_dir>/temp_image/rgba.png and pasted onto white through its alpha as temp_image/white.png, at
    the input's size.  Returns the image stage 1 reads: white.png, or `image_path` itself when ckpts/u2net.pth is absent."""
    return remove_backgrounds([image_path], [output_dir])[0]


def remove_backgrounds(image_paths, output_dirs):
    """remove_background for several images with one U^2-Net call (rembg.remove_batch); image i's files go under
    output_dirs[i]."""
    from PIL import Image
    from hi3d_official_b200 import rembg
    if not os.path.exists(rembg.DEFAULT_WEIGHTS):
        for image_path in image_paths:
            print(f"[hi3d-b200] WARNING: {rembg.DEFAULT_WEIGHTS} not found, background removal SKIPPED: stage 1 conditions on "
                  f"{image_path} as given, background included", flush=True)
        return list(image_paths)
    images = rembg.remove_batch([Image.open(p) for p in image_paths], session=rembg.new_session())
    out = []
    for image_path, output_dir, image in zip(image_paths, output_dirs, images):
        temp_dir = os.path.join(output_dir, "temp_image")
        os.makedirs(temp_dir, exist_ok=True)
        image.save(os.path.join(temp_dir, "rgba.png"))
        white_path = os.path.join(temp_dir, "white.png")
        white = Image.new("RGB", image.size, "WHITE")
        white.paste(image, mask=image.split()[3])
        white.save(white_path)
        print(f"[hi3d-b200] removed the background of {image_path}: {white_path}", flush=True)
        out.append(white_path)
    return out


def cond_from_towers(model, frames, towers, elevation, stage, generators=None):
    """v01:62-78 / v02:104-118: batch -> add_custom_cond -> GeneralConditioner with the third-party towers' outputs supplied.
    frames: (3, T, H, W) for one object or (B, 3, T, H, W) for B, in [-1, 1] on the GPU (stage 1: the image repeated T times).
    elevation: one number, or one per object.  towers: the objects' tower outputs stacked ('clip' (B, 1024), 'aes' (B, 1),
    'depth' (B*T, h', w')).  generators: one CUDA generator per object for the condition-frame noise (None: the global one).
    The conditioner's towers and the VAE encode run once over the whole batch."""
    video = frames if frames.dim() == 5 else frames[None]
    B, dev = video.shape[0], frames.device
    elevs = [float(e) for e in (elevation if isinstance(elevation, (list, tuple)) else [elevation] * B)]
    batch = {"video": video, "elevation": torch.tensor(elevs, device=dev),
             "fps_id": torch.full((B,), 7.0, device=dev), "motion_bucket_id": torch.full((B,), 127.0, device=dev)}
    batch = model.add_custom_cond(batch, infer=True, generators=generators)
    towers = towers or {}                     # a tower missing here runs natively in the conditioner (or raises)
    if "clip" in towers:
        batch["cond_frames_without_noise:clip"] = towers["clip"].to(dev).float().reshape(B, -1)
    if stage == 1 and "aes" in towers:
        batch["video:aes"] = towers["aes"].to(dev).float().reshape(B, 1)
    elif stage == 2 and "depth" in towers:
        batch["cond_frames:depth"] = towers["depth"].to(frames.device).float()
    c, uc = model.conditioner.get_unconditional_conditioning(
        batch, force_uc_zero_embeddings=["cond_frames", "cond_frames_without_noise"])
    return c, uc


def native_towers_ready(model, allowed_missing=()):
    """True when the model's GeneralConditioner runs every tower natively (weights loaded), except `allowed_missing`."""
    missing = getattr(model.conditioner, "missing_towers", None)
    return missing is not None and not set(missing()) - set(allowed_missing)


# ---- several images per run ---------------------------------------------------------------------------------------------
def add_cli_args(ap, stage):
    """The flags both entry points share.  --image_path, --elevation, --seed and --towers take one value or one per image."""
    ap.add_argument("--denoise_config", type=str, default=f"configs/inference-v0{stage}.yaml")
    ap.add_argument("--denoise_checkpoint", type=str, default="ckpts/first_stage.pt" if stage == 1 else "ckpts/second_stage.pt")
    ap.add_argument("--image_path", type=str, nargs="+", default=["demo/15_out.png"])
    ap.add_argument("--output_dir", type=str, default="outputs/15_out")
    ap.add_argument("--elevation", type=int, nargs="+", default=[0])
    ap.add_argument("--cond", type=str, default=None)
    ap.add_argument("--towers", type=str, nargs="+", default=None)
    ap.add_argument("--synthetic", action="store_true")
    ap.add_argument("--tiny", action="store_true")
    ap.add_argument("--seed", type=int, nargs="+", default=None)
    ap.add_argument("--batch", type=int, default=1,
                    help="objects per sampling batch (several images): trades device memory for throughput, same results")
    ap.add_argument("--precision", choices=("fp16", "fp8", "fp8_attn"), default="fp16",
                    help="operand precision of the denoising UNet's convolutions, projections and feed-forwards: fp8 runs them "
                         "on e4m3 tensor cores, which changes the result (the VAE and the conditioner stay fp16); fp8_attn "
                         "also runs every spatial self-attention core on e4m3 tensor cores, which changes the result again")
    from hi3d_official_b200.sampling import GUIDANCE_CHOICES, SAMPLER_CHOICES
    ap.add_argument("--sampler", choices=("config",) + tuple(SAMPLER_CHOICES), default="config",
                    help="the sampler; 'config' keeps the configuration's" + ("" if stage == 1 else
                         " (stage 2 re-noises between EDM steps: euler or heun only)"))
    ap.add_argument("--steps", type=int, default=None, help="sampler steps (default: the configuration's)")
    ap.add_argument("--guidance", choices=GUIDANCE_CHOICES, default="config",
                    help="linear: the scale rises from 1 to --cfg_scale over the frames (LinearPredictionGuider); vanilla: "
                         "--cfg_scale for every frame (VanillaCFG); none: no unconditional evaluation (IdentityGuider), half "
                         "the network rows")
    ap.add_argument("--cfg_scale", type=float, default=None,
                    help="guidance scale of --guidance linear / vanilla (default: the configuration's maximum scale)")
    ap.add_argument("--s_churn", type=float, default=None, help="EDM churn of euler / heun (default: the configuration's)")
    ap.add_argument("--eta", type=float, default=None, help="ancestral noise of euler_ancestral / dpmpp2s_ancestral (default 1)")


def configure_sampler(model, params, stage):
    """Applies --sampler, --steps, --guidance, --cfg_scale, --s_churn and --eta to the model's sampler (the configuration's
    when none is given)."""
    from hi3d_official_b200.sampling import EDMSampler, configure_sampler as configure
    if params.steps is not None and params.steps < 1:
        raise SystemExit(f"--steps must be at least 1, got {params.steps}")
    try:
        smp = configure(model.sampler, params.sampler, params.steps, params.guidance, params.cfg_scale, params.s_churn,
                        params.eta, num_frames=model.num_samples)
    except ValueError as e:
        raise SystemExit(str(e))
    if stage == 2 and not isinstance(smp, EDMSampler):
        raise SystemExit(f"stage 2 drives the sampler one step at a time between re-noise blends (EDMSampler.step_call), which "
                         f"only the EDM samplers have: --sampler euler or heun, not {type(smp).__name__}")
    model.sampler = smp


def per_image(values, n, flag):
    """One value for all n images, or one per image."""
    if values is None:
        return [None] * n
    if len(values) == 1:
        return list(values) * n
    if len(values) != n:
        raise SystemExit(f"{flag}: give one value or one per image ({n}), got {len(values)}")
    return list(values)


def batch_plan(params):
    """Several images: per image its output directory <output_dir>/<image stem>, elevation, seed (random when not given)
    and tower file, and the groups of image indices that share a sampling batch (--batch)."""
    paths = params.image_path
    n = len(paths)
    stems = [os.path.splitext(os.path.basename(p))[0] for p in paths]
    dup = sorted({s for s in stems if stems.count(s) > 1})
    if dup:
        raise SystemExit(f"images with the same file name stem would share an output directory: {dup}")
    if params.batch < 1:
        raise SystemExit(f"--batch must be at least 1, got {params.batch}")
    if params.cond:
        raise SystemExit("--cond holds one image's conditioning: with several images use --towers, --synthetic or the towers' "
                         "weights")
    return dict(dirs=[os.path.join(params.output_dir, s) for s in stems],
                elevations=per_image(params.elevation, n, "--elevation"),
                seeds=[random.randint(0, 65535) if s is None else s for s in per_image(params.seed, n, "--seed")],
                towers=per_image(params.towers, n, "--towers"),
                groups=[list(range(i, min(n, i + params.batch))) for i in range(0, n, params.batch)])


def cat_cond(dicts):
    """c / uc dictionaries of single objects -> one batch (per-key concatenation, object-major)."""
    return {k: torch.cat([d[k] for d in dicts], 0) for k in dicts[0]}


def load_towers(paths):
    """--towers files of several images, stacked per key: 'clip' (B, 1024), 'aes' (B, 1), 'depth' (B*T, h', w')."""
    ts = [torch.load(p) for p in paths]
    keys = set.intersection(*(set(t) for t in ts))
    return {k: torch.cat([t[k].float().reshape((-1,) + tuple(t[k].shape[-2:])) if k == "depth" else t[k].float().reshape(1, -1)
                          for t in ts], 0) for k in keys}


def main_batch(params, model, T, h):
    """Stage 1 over several images, --batch objects per sampling batch; object i draws from its own generators exactly what
    a single-image run with its seed draws (condition-frame noise, then the initial latents)."""
    from hi3d_official_b200.engine import per_object_randn
    plan = batch_plan(params)
    if not (params.towers or params.synthetic or native_towers_ready(model)):
        raise SystemExit("the conditioner towers are outside the H100 hot path: pass --towers <file> or --synthetic")
    for idx in plan["groups"]:
        seeds, dirs = [plan["seeds"][i] for i in idx], [plan["dirs"][i] for i in idx]
        gens = [torch.Generator("cuda").manual_seed(s) for s in seeds]
        if params.synthetic and not params.towers:
            c, uc = (cat_cond(d) for d in zip(*[synthetic_cond(1, T, h, "cuda", s) for s in seeds]))
        else:
            paths = remove_backgrounds([params.image_path[i] for i in idx], dirs)
            img = torch.stack([load_image(p, 8 * h) for p in paths]).cuda()              # (B, 3, H, W)
            towers = load_towers([plan["towers"][i] for i in idx]) if params.towers else None
            c, uc = cond_from_towers(model, img[:, :, None].repeat(1, 1, T, 1, 1), towers,
                                     [plan["elevations"][i] for i in idx], 1, generators=gens)
        randn = per_object_randn((T, 4, h, h), gens, "cuda")
        with torch.no_grad():
            frames = model.sample_stage1(c, uc, randn, generators=gens)
        for j, (d, s) in enumerate(zip(dirs, seeds)):
            mp4 = save_frames(frames[j * T:(j + 1) * T], os.path.join(d, "first_step"), "first")
            print(f"[hi3d-b200] wrote {T} frames {tuple(frames.shape[1:])} to {mp4} (seed {s})")


def main():
    ap = argparse.ArgumentParser()
    add_cli_args(ap, 1)
    params = ap.parse_args()
    if len(params.image_path) > 1:
        batch_plan(params)                                                       # argument errors before the model loads
        model = load_model(params.denoise_config, params.denoise_checkpoint, 1, params.tiny, params.precision)
        configure_sampler(model, params, 1)
        return main_batch(params, model, model.num_samples, 16 if params.tiny else 64)
    image_path, elevation = params.image_path[0], params.elevation[0]
    towers = params.towers[0] if params.towers else None
    if len(params.elevation) > 1 or (params.seed and len(params.seed) > 1) or (params.towers and len(params.towers) > 1):
        raise SystemExit("one image takes one --elevation, --seed and --towers value")
    seed = random.randint(0, 65535) if params.seed is None else params.seed[0]   # v01:33-34
    torch.manual_seed(seed)
    model = load_model(params.denoise_config, params.denoise_checkpoint, 1, params.tiny, params.precision)
    configure_sampler(model, params, 1)
    T = model.num_samples                                                        # 16 frames
    h = 16 if params.tiny else 64                                                # 512^2 / 8
    if params.cond:
        d = torch.load(params.cond, map_location="cuda")
        c, uc = d["c"], d["uc"]
    elif towers:
        img = load_image(remove_background(image_path, params.output_dir), 8 * h).cuda()
        c, uc = cond_from_towers(model, img[:, None].repeat(1, T, 1, 1), torch.load(towers), elevation, 1)
    elif params.synthetic:
        c, uc = synthetic_cond(1, T, h, "cuda", seed)
    elif native_towers_ready(model):
        img = load_image(remove_background(image_path, params.output_dir), 8 * h).cuda()
        c, uc = cond_from_towers(model, img[:, None].repeat(1, T, 1, 1), None, elevation, 1)
    else:
        raise SystemExit("the conditioner towers are outside the H100 hot path: pass --towers / --cond <file> or --synthetic")
    randn = torch.randn(T, 4, h, h, device="cuda")                               # v01:91
    with torch.no_grad():
        frames = model.sample_stage1(c, uc, randn)                               # v01:92-94
    mp4 = save_frames(frames, os.path.join(params.output_dir, "first_step"), "first")
    print(f"[hi3d-b200] wrote {T} frames {tuple(frames.shape[1:])} to {mp4} (seed {seed})")


if __name__ == "__main__":
    main()
