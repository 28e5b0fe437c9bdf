#!/usr/bin/env python
"""Time the conditioner's MiDaS DPT-Hybrid depth tower (midas.DPTHybridTower) at full size on seeded weights: one call of
16 frames at 384^2, what DepthEmbedder runs once per stage-2 video at 1024^2.  CUDA events around --iters calls after --warmup;
the same for the fp32 oracle (tests/midas_oracle.py) under fp16 autocast, the reference's own precision, for comparison.
Prints one JSON line with the card's name and power limit beside the times.

    python tools/time_depth_tower.py [--iters 5] [--warmup 2] [--frames 16] [--size 384]
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

from hi3d_official_b200.midas import DPTHybridTower  # noqa: E402
import midas_oracle as MO  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def flops_per_image(H, W, stem=64, stage_out=(256, 512, 1024), stage_mid=(64, 128, 256), depths=(3, 4, 9), width=768, mlp=3072,
                    blocks=12, features=256):
    """2 x multiply-adds of DPT-Hybrid's convs, linears and attention products at an H x W input, as the reference computes them
    (out_conv at the upsampled resolution, no channel padding)."""
    conv = lambda hw, ci, co, k: 2.0 * hw * ci * co * k * k   # noqa: E731
    f = conv(H * W / 4, 3, stem, 7)
    h, cin = H * W / 16, stem
    for si, (co, mid, d) in enumerate(zip(stage_out, stage_mid, depths)):
        for b in range(d):
            ho = h / 4 if (b == 0 and si > 0) else h
            f += conv(h, cin if b == 0 else co, mid, 1) + conv(ho, mid, mid, 3) + conv(ho, mid, co, 1)
            if b == 0:
                f += conv(ho, cin, co, 1)
            h = ho
        cin = co
    P = h
    L = P + 1
    f += conv(P, cin, width, 1)
    f += blocks * (2.0 * L * (4 * width * width + 2 * width * mlp) + 4.0 * L * L * width)
    f += 2 * (conv(P, 2 * width, width, 1) + conv(P, width, width, 1)) + conv(P / 4, width, width, 3)
    grids = [H * W / 16, H * W / 64, P, P / 4]
    for hw, ci in zip(grids, (stage_out[0], stage_out[1], width, width)):
        f += conv(hw, ci, features, 3)
    for i, hw in enumerate(grids):
        units = 1 if i == 3 else 2
        f += units * 2 * conv(hw, features, features, 3) + conv(4 * hw, features, features, 1)
    f += conv(H * W / 4, features, features // 2, 3) + conv(H * W, features // 2, 32, 3) + conv(H * W, 32, 1, 1)
    return f


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--size", type=int, default=384)
    a = ap.parse_args()
    sd = MO.random_dpt_hybrid_sd(seed=1, device="cuda", **MO.FULL)
    x = torch.rand(a.frames, 3, a.size, a.size, device="cuda") * 2 - 1
    tower = DPTHybridTower(sd, device="cuda")
    fl = flops_per_image(a.size, a.size) * a.frames
    ms = timed(lambda: tower(x), a.iters, a.warmup)

    def oracle():
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
            MO.dpt_forward(sd, x)
    ms_ref = timed(oracle, a.iters, a.warmup)
    print(json.dumps({"gpu": card(), "frames": a.frames, "size": a.size, "gflop_per_call": round(fl / 1e9, 1),
                      "native": {"ms_per_call": round(ms, 2), "tflops": round(fl / ms / 1e9, 1)},
                      "oracle_fp16_autocast": {"ms_per_call": round(ms_ref, 2), "tflops": round(fl / ms_ref / 1e9, 1)},
                      "speedup": round(ms_ref / ms, 2)}))


if __name__ == "__main__":
    main()
