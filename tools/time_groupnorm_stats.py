#!/usr/bin/env python
"""Time the GroupNorm unit-statistics launch (hi3d_groupnorm_unit_stats) at the shapes the plans give it: the VAE at 1024^2 and
512^2, one frame per call (n_images = 1), and the stage-2 / stage-1 UNet at 2 x 16 frames (n_images = 32).  Each shape is timed
with CUDA events over back-to-back launches into one table; the rate is the tensor's bytes (one fp16 read) over the time,
reported against the H100 SXM's 3.35 TB/s HBM3 data-sheet bandwidth, with the card's name and power limit.  Needs a GPU.
Usage: python tools/time_groupnorm_stats.py [--iters 50] [--json out.json]"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_TBS = 3.35
SHAPES = [  # (what, C, unit, rows per image, n_images)
    ("VAE 1024^2 x 128", 128, 4, 1 << 20, 1),
    ("VAE 1024^2 x 256", 256, 4, 1 << 20, 1),
    ("VAE 512^2 x 256", 256, 4, 1 << 18, 1),
    ("VAE 512^2 x 512", 512, 4, 1 << 18, 1),
    ("VAE 256^2 x 512", 512, 4, 1 << 16, 1),
    ("UNet s2 128^2 x 320", 320, 10, 16384, 32),
    ("UNet s2 64^2 x 640", 640, 10, 4096, 32),
    ("UNet s2 32^2 x 1280", 1280, 10, 1024, 32),
    ("UNet s2 16^2 x 1280", 1280, 10, 256, 32),
    ("UNet s1 64^2 x 320", 320, 10, 4096, 32),
    ("UNet s1 8^2 x 1280", 1280, 10, 64, 32),
]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        q = torch.cuda.get_device_name(0) + ", power limit unknown"
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--json", type=str, default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "time_groupnorm_stats.py needs a GPU"
    from hi3d_official_b200 import ops
    dev = torch.device("cuda", 0)
    res = {"card": card(), "shapes": {}}
    for what, C, unit, rows, n in SHAPES:
        x = torch.randn(n * rows, C, generator=torch.Generator(device=dev).manual_seed(1), device=dev).half()
        st = torch.zeros(n * (C // unit) * 2, device=dev)
        for _ in range(3):
            ops.groupnorm_unit_stats(x, n, rows, unit, st)
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(a.iters):
            ops.groupnorm_unit_stats(x, n, rows, unit, st)
        e.record()
        torch.cuda.synchronize()
        us = s.elapsed_time(e) / a.iters * 1e3
        gbs = x.numel() * 2 / us / 1e3
        res["shapes"][what] = dict(C=C, unit=unit, rows=rows, n_images=n, us=round(us, 2), gbs=round(gbs, 1),
                                   hbm_frac=round(gbs / (HBM_TBS * 1e3), 3))
        print(f"{what:22s} rows {rows:8d} x n {n:3d}: {us:9.2f} us  {gbs:7.1f} GB/s  {100 * gbs / (HBM_TBS * 1e3):5.1f} % of "
              f"{HBM_TBS} TB/s")
        del x, st
    print(f"card: {res['card']}")
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
