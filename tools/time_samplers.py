#!/usr/bin/env python
"""Time one video's sampling for every sampler, step count and guidance the pipelines offer (--sampler, --steps, --guidance),
on the full-width stage-1 (16 x 64^2 latents) and stage-2 (16 x 128^2, the re-noise loop of sample_stage2) models with
synthetic weights and conditioning.  Stage 2 runs the EDM samplers only, as its pipeline does.  Each (sampler, guidance) is
warmed up with a 2-step video (plans built, CUDA graphs captured), then each step count is timed as the wall time of one
video between device synchronisations, VAE decode excluded; the median of --reps videos is reported.  Also the eager-to-graph
gain of Heun and DPM-Solver++(2M) (HI3D_CUDA_GRAPH=0 against graph replay) at stage 1.  The card's name, power limit and
maximum SM clock are read in the same run.  Needs a GPU.
Usage: python tools/time_samplers.py [--stages 1 2] [--steps 10 15 25] [--reps 1] [--json out.json]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

T = 16
STAGE = {1: dict(h=64, cc=4, adm=768), 2: dict(h=128, cc=13, adm=512)}
SAMPLERS = {1: ("euler", "heun", "dpmpp2m", "euler_ancestral", "dpmpp2s_ancestral", "lms"), 2: ("euler", "heun")}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else \
        torch.cuda.get_device_name(0) + ", power limit not readable"


def inputs(stage, seed=0):
    s = STAGE[stage]
    g = torch.Generator().manual_seed(seed)
    h = s["h"]
    c = dict(crossattn=torch.randn(1, 1, 1024, generator=g), vector=torch.randn(1, s["adm"], generator=g),
             concat=(torch.randn(T, s["cc"], h, h, generator=g) * 0.18).half())
    c = {k: v.cuda() for k, v in c.items()}
    uc = dict(crossattn=torch.zeros_like(c["crossattn"]), vector=c["vector"], concat=torch.zeros_like(c["concat"]))
    randn = torch.randn(T, 4, h, h, generator=g).cuda()
    z = (torch.randn(T, 4, h, h, generator=g) * 0.18).cuda()
    return c, uc, randn, z


def video(model, stage, inp):
    c, uc, randn, z = inp
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    if stage == 1:
        model.sample_stage1(c, uc, randn.clone(), decode=False)
    else:
        model.sample_stage2(c, uc, randn.clone(), z, decode=False)
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def time_config(model, stage, base, name, guidance, steps_list, reps, inp):
    from hi3d_official_b200.sampling import configure_sampler
    model.sampler = configure_sampler(base, name, 2, guidance, num_frames=T)
    video(model, stage, inp)                                   # warm-up: plans, graph captures
    out = {}
    for steps in steps_list:
        model.sampler.num_steps = steps
        out[steps] = statistics.median(video(model, stage, inp) for _ in range(reps))
    model.sampler = base
    return out


@torch.no_grad()
def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--stages", type=int, nargs="+", default=[1, 2])
    ap.add_argument("--steps", type=int, nargs="+", default=[10, 15, 25])
    ap.add_argument("--reps", type=int, default=1)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    from hi3d_official_b200 import configs, spec
    res = {"card": card(), "frames": T, "seconds_per_video": {}, "eager_vs_graph": {}}
    print(res["card"], flush=True)
    for stage in args.stages:
        model = configs.build_engine(stage, device="cuda")
        spec.synth_fill_(model, seed=0, fast=True)
        base, inp = model.sampler, inputs(stage)
        for name in SAMPLERS[stage]:
            for guidance in ("linear", "none"):
                t = time_config(model, stage, base, name, guidance, args.steps, args.reps, inp)
                res["seconds_per_video"][f"stage{stage}/{name}/{guidance}"] = t
                print(f"stage {stage} {name:18s} guidance {guidance:6s} " +
                      "  ".join(f"{s:3d} steps {v:7.3f} s" for s, v in t.items()), flush=True)
        if stage == 1:
            for name in ("heun", "dpmpp2m"):
                gain = {}
                for mode in ("0", "1"):
                    os.environ["HI3D_CUDA_GRAPH"] = mode
                    gain["graph" if mode == "1" else "eager"] = time_config(model, stage, base, name, "linear", [25],
                                                                             args.reps, inp)[25]
                res["eager_vs_graph"][f"stage{stage}/{name}/25"] = gain
                print(f"stage {stage} {name}: 25 steps eager {gain['eager']:.3f} s, graph replay {gain['graph']:.3f} s "
                      f"({gain['eager'] / gain['graph']:.3f}x)", flush=True)
            os.environ.pop("HI3D_CUDA_GRAPH", None)
        del model, base
        torch.cuda.empty_cache()
    res["card_after"] = card()
    print(res["card_after"])
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        json.dump(res, open(args.json, "w"), indent=1)


if __name__ == "__main__":
    main()
