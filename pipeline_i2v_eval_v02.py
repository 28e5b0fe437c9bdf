#!/usr/bin/env python
"""Stage-2 (1024^2 refiner) entry point, same CLI as the reference's pipeline_i2v_eval_v02.py (:38-44) on the H100
engine.  Reads <output_dir>/first_step/first.pt (stage-1 frames written by pipeline_i2v_eval_v01.py; first.mp4 through
OpenCV when the tensor is absent, like v02:169-176), up-samples them to 1024^2, VAE-encodes each frame (posterior sample,
CPU RNG like the reference), runs the 25-step re-noise/blend loop of pipeline_i2v_eval_v02.py:127-135 on the fused sampler,
decodes and writes second_step_video/second.mp4.  Conditioning, in v01's order: --cond, --towers {'clip': (1,1024), 'depth':
(T,h',w') MiDaS maps}, --synthetic, and otherwise, when the OpenCLIP and MiDaS DPT-Hybrid towers have weights (their files under
the working directory or their tensors in the checkpoint), the model's own conditioner builds c / uc from the frames.  A tower
left out of --towers runs natively; --tiny = the smoke size the tests run.

Several images (the same --image_path list as stage 1): each object's stage-1 output is read from <output_dir>/<image stem>/
and its video written there; --batch K refines K objects per batch, object i drawing from generators seeded with its seed
exactly what a single-image run draws."""
import argparse
import os
import random

import torch
import torch.nn.functional as F

from pipeline_i2v_eval_v01 import (add_cli_args, batch_plan, cat_cond, cond_from_towers, configure_sampler, load_model,
                                   load_towers, native_towers_ready, save_frames, synthetic_cond)


def replace_first_frame(frames, output_dir, size):
    """v02:184-188: frame 0 of the stage-1 video becomes the cut-out input <output_dir>/temp_image/white.png (written by
    pipeline_i2v_eval_v01.py) -- cv2.imread, cv2.resize to size x size (INTER_LINEAR), BGR -> RGB, [-1, 1] -- when that file
    exists.  frames: (T, 3, size, size) in [-1, 1], changed in place.  Returns whether frame 0 was replaced."""
    import cv2
    import numpy as np
    path = os.path.join(output_dir, "temp_image", "white.png")
    if not os.path.exists(path):
        return False
    img = cv2.cvtColor(cv2.resize(cv2.imread(path), [size, size]), cv2.COLOR_BGR2RGB)
    frames[0] = (torch.from_numpy(np.ascontiguousarray(img)).permute(2, 0, 1).float() / 255.0 - 0.5) * 2.0
    print(f"[hi3d-b200] frame 0 replaced by {path}", flush=True)
    return True


def load_first_frames(output_dir, T, h, synthetic, generator=None):
    """One object's stage-1 frames from <output_dir>/first_step, up-sampled to (T, 3, 8h, 8h) on the GPU, frame 0 replaced
    by the cut-out input; random frames (from `generator`, or the global one) when there are none and `synthetic`."""
    first = os.path.join(output_dir, "first_step", "first.pt")
    first_mp4 = os.path.join(output_dir, "first_step", "first.mp4")
    if os.path.exists(first):
        frames = torch.load(first).cuda().float()
        frames = F.interpolate(frames, size=(8 * h, 8 * h), mode="bilinear", align_corners=False)   # cv2.resize, v02:186
    elif os.path.exists(first_mp4):
        import numpy as np
        from hi3d_official_b200 import video_io
        fr = np.stack(video_io.read_video_frames(first_mp4)[:T], 0)
        frames = torch.from_numpy(fr).permute(0, 3, 1, 2).float().cuda() / 127.5 - 1.0
        frames = F.interpolate(frames, size=(8 * h, 8 * h), mode="bilinear", align_corners=False)
    elif synthetic:
        frames = torch.rand(T, 3, 8 * h, 8 * h, device="cuda", generator=generator) * 2 - 1
    else:
        raise SystemExit(f"{first} not found (run pipeline_i2v_eval_v01.py first) and --synthetic not given")
    replace_first_frame(frames, output_dir, 8 * h)
    return frames


def posterior_noise(model, T, h, generators):
    """The CPU draws encode_first_stage makes for T frames without `noise` (one randn per chunk of
    en_and_decode_n_samples_a_time frames), from each object's CPU generator in turn: (B*T, 4, h, h)."""
    k = model.en_and_decode_n_samples_a_time or T
    return torch.cat([torch.randn((min(k, T - t), 4, h, h), generator=g) for g in generators for t in range(0, T, k)], 0)


def main_batch(params, model, T, h):
    from hi3d_official_b200.engine import per_object_randn
    plan = batch_plan(params)
    if not (params.towers or params.synthetic or native_towers_ready(model)):
        raise SystemExit(f"the conditioner's towers {model.conditioner.missing_towers()} have no weights: put their files under "
                         f"ckpts/ (open_clip_pytorch_model.bin, dpt_hybrid_384.pt), or pass --towers <file> or --synthetic")
    for idx in plan["groups"]:
        seeds, dirs, B = [plan["seeds"][i] for i in idx], [plan["dirs"][i] for i in idx], len(idx)
        gens = [torch.Generator("cuda").manual_seed(s) for s in seeds]
        frames = torch.cat([load_first_frames(d, T, h, params.synthetic, g) for d, g in zip(dirs, gens)], 0)
        if params.towers:
            video = frames.view(B, T, *frames.shape[1:]).permute(0, 2, 1, 3, 4).contiguous()
            c, uc = cond_from_towers(model, video, load_towers([plan["towers"][i] for i in idx]),
                                     [plan["elevations"][i] for i in idx], 2, generators=gens)
        elif params.synthetic:
            c, uc = (cat_cond(d) for d in zip(*[synthetic_cond(2, T, h, "cuda", s) for s in seeds]))
        else:
            video = frames.view(B, T, *frames.shape[1:]).permute(0, 2, 1, 3, 4).contiguous()
            c, uc = cond_from_towers(model, video, None, [plan["elevations"][i] for i in idx], 2, generators=gens)
        with torch.no_grad():
            init_latents = per_object_randn((T, 4, h, h), gens, "cuda")
            noise = posterior_noise(model, T, h, [torch.Generator().manual_seed(s) for s in seeds]).cuda()
            z = model.encode_first_stage(frames.half(), noise=noise)
            out = model.sample_stage2(c, uc, init_latents, z.float(), generators=gens)
        for j, (d, s) in enumerate(zip(dirs, seeds)):
            mp4 = save_frames(out[j * T:(j + 1) * T], os.path.join(d, "second_step_video"), "second")
            print(f"[hi3d-b200] wrote {T} frames {tuple(out.shape[1:])} to {mp4} (seed {s})")


def main():
    ap = argparse.ArgumentParser()
    add_cli_args(ap, 2)
    params = ap.parse_args()
    if params.sampler not in ("config", "euler", "heun"):
        raise SystemExit(f"stage 2 drives the sampler one step at a time between re-noise blends (EDMSampler.step_call), which "
                         f"only the EDM samplers have: --sampler euler or heun, not {params.sampler}")
    if len(params.image_path) > 1:
        batch_plan(params)                                                       # argument errors before the model loads
        model = load_model(params.denoise_config, params.denoise_checkpoint, 2, params.tiny, params.precision)
        configure_sampler(model, params, 2)
        return main_batch(params, model, model.num_samples, 32 if params.tiny else 128)
    elevation = params.elevation[0]
    towers = params.towers[0] if params.towers else None
    if len(params.elevation) > 1 or (params.seed and len(params.seed) > 1) or (params.towers and len(params.towers) > 1):
        raise SystemExit("one image takes one --elevation, --seed and --towers value")
    seed = random.randint(0, 65535) if params.seed is None else params.seed[0]
    torch.manual_seed(seed)
    model = load_model(params.denoise_config, params.denoise_checkpoint, 2, params.tiny, params.precision)
    configure_sampler(model, params, 2)
    T = model.num_samples
    h = 32 if params.tiny else 128
    frames = load_first_frames(params.output_dir, T, h, params.synthetic)
    if params.cond:
        d = torch.load(params.cond, map_location="cuda")
        c, uc = d["c"], d["uc"]
    elif towers:
        c, uc = cond_from_towers(model, frames.permute(1, 0, 2, 3).contiguous(), torch.load(towers), elevation, 2)
    elif params.synthetic:
        c, uc = synthetic_cond(2, T, h, "cuda", seed)
    elif native_towers_ready(model):
        c, uc = cond_from_towers(model, frames.permute(1, 0, 2, 3).contiguous(), None, elevation, 2)
    else:
        raise SystemExit(f"the conditioner's towers {model.conditioner.missing_towers()} have no weights: put their files under ckpts/ "
                         f"(open_clip_pytorch_model.bin, dpt_hybrid_384.pt), or pass --towers / --cond <file> or --synthetic")
    with torch.no_grad():
        init_latents = torch.randn(T, 4, h, h, device="cuda")                                      # v02:93
        z = model.encode_first_stage(frames.half())              # v02:96-101: en_and_decode_n_samples_a_time frames a call
        out = model.sample_stage2(c, uc, init_latents, z.float())                                  # v02:103-137
    mp4 = save_frames(out, os.path.join(params.output_dir, "second_step_video"), "second")
    print(f"[hi3d-b200] wrote {T} frames {tuple(out.shape[1:])} to {mp4} (seed {seed})")


if __name__ == "__main__":
    main()
