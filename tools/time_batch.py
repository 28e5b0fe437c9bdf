#!/usr/bin/env python
"""Throughput of sampling several objects in one batch: stage 1 (16 x 512^2, 25 EDM steps + VAE decode) at B = 1, 2, 4 objects
and stage 2 (16 x 1024^2, 25 re-noise steps + decode) at B = 1, 2, on seeded synthetic full-size weights through the fused
CUDA-graph sampler -- what pipeline_i2v_eval_v0{1,2}.py --batch B runs after conditioning.  Prints, per (stage, B), the output
frames per second (B * 16 frames per batch over the wall time of whole batches, timed with CUDA events after a warm-up batch)
and the peak device memory, plus the card's name and power limit read in the same run.  Needs a GPU.
Usage: python tools/time_batch.py [--reps 2] [--stage1 1 2 4] [--stage2 1 2] [--json out.json]"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

T = 16


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def inputs(stage, B, dev):
    g = torch.Generator().manual_seed(100 + B)
    h, cc, adm = (64, 4, 768) if stage == 1 else (128, 13, 512)
    c = dict(crossattn=torch.randn(B, 1, 1024, generator=g), vector=torch.randn(B, adm, generator=g),
             concat=(torch.randn(B * T, cc, h, h, generator=g) * 0.18).half())
    c = {k: v.to(dev) for k, v in c.items()}
    uc = dict(crossattn=torch.zeros_like(c["crossattn"]), vector=c["vector"], concat=torch.zeros_like(c["concat"]))
    x = torch.randn(B * T, 4, h, h, generator=g).to(dev)
    z = (torch.randn(B * T, 4, h, h, generator=g) * 0.18).to(dev)
    return c, uc, x, z


def measure(model, stage, B, reps, dev):
    c, uc, x, z = inputs(stage, B, dev)

    def batch():
        if stage == 1:
            return model.sample_stage1(c, uc, x.clone())
        return model.sample_stage2(c, uc, x.clone(), z)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(dev)
    with torch.no_grad():
        out = batch()                                  # warm-up: launch plans, CUDA-graph capture, VAE plans
        assert out.shape[0] == B * T
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            batch()
        e1.record()
        torch.cuda.synchronize()
    s = e0.elapsed_time(e1) / 1e3 / reps
    return dict(stage=stage, objects=B, frames=B * T, s_per_batch=round(s, 3), frames_per_s=round(B * T / s, 3),
                peak_mem_gib=round(torch.cuda.max_memory_allocated(dev) / 2 ** 30, 2))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2, help="timed batches per (stage, B), after one warm-up batch")
    ap.add_argument("--stage1", type=int, nargs="*", default=[1, 2, 4])
    ap.add_argument("--stage2", type=int, nargs="*", default=[1, 2])
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_batch.py measures on a GPU; none is visible")
    from hi3d_official_b200 import configs, spec
    dev = torch.device("cuda", 0)
    gpu = card()
    print(f"card: {gpu}", flush=True)
    rows = []
    for stage, Bs in ((1, args.stage1), (2, args.stage2)):
        if not Bs:
            continue
        model = configs.build_engine(stage, device=dev)
        spec.synth_fill_(model, seed=0, fast=True)
        for B in Bs:
            r = measure(model, stage, B, args.reps, dev)
            rows.append(r)
            print(json.dumps(r), flush=True)
            model.sampler._fused.clear()                  # drop this B's captured graph and plan before the next B
            model.model.diffusion_model._plans.clear()
            model.first_stage_model._plans.clear()
            torch.cuda.empty_cache()
        del model
        torch.cuda.empty_cache()
    for stage in (1, 2):
        base = next((r for r in rows if r["stage"] == stage and r["objects"] == 1), None)
        for r in rows:
            if base is not None and r["stage"] == stage:
                r["speedup_vs_B1"] = round(r["frames_per_s"] / base["frames_per_s"], 3)
    result = {"card": gpu, "reps": args.reps, "results": rows}
    print(json.dumps(result))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
