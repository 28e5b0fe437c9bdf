#!/usr/bin/env python
"""Time the conditioner's CLIP image towers (clip_vision.ClipVisionTower) at full width on seeded weights: OpenCLIP
ViT-H/14 and OpenAI ViT-L/14, one 224^2 image per call (what one video needs), CUDA events around --iters calls after
--warmup.  Prints one JSON line with the card's name and power limit beside the times.

    python tools/time_clip_towers.py [--iters 20] [--warmup 3] [--batch 1]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from hi3d_official_b200.clip_vision import ClipVisionTower  # noqa: E402
import clip_oracle as CO  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=1)
    a = ap.parse_args()
    res = {"gpu": card(), "batch": a.batch}
    for name, (width, layers, hw, out, qg) in {"vit_h14": (1280, 32, 80, 1024, False),
                                               "vit_l14": (1024, 24, 64, 768, True)}.items():
        tower = ClipVisionTower(CO.random_visual_sd(width, layers, hw, out, seed=1), hw, qg, device="cuda")
        img = torch.rand(a.batch, 3, 224, 224, device="cuda")
        for _ in range(a.warmup):
            tower(img)
        torch.cuda.synchronize()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(a.iters):
            tower(img)
        t1.record()
        torch.cuda.synchronize()
        ms = t0.elapsed_time(t1) / a.iters
        res[name] = {"ms_per_call": round(ms, 3), "tflops": round(tower.flops_per_image * a.batch / ms / 1e9, 1)}
        del tower
    print(json.dumps(res))


if __name__ == "__main__":
    main()
