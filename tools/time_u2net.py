#!/usr/bin/env python
"""Time the native U^2-Net (hi3d_official_b200/u2net.py) on seeded full-size weights: one 320^2 image (what rembg.remove runs per
video) and a batch of 16.  Prints ms per call, the rate against U^2-Net's 117.2 GFLOP per 320^2 image (torch.utils.flop_counter
on the fp32 graph), the share of conv time that went to the mma.sync engine (geometries hi3d_gemm_tc5 forwards: N < 32, or
feature maps whose tile does not divide the batch, e.g. the 40^2, 20^2 and 10^2 levels at batch 1), and the card's name and
power limit.  Also the summed kernel time of one call (torch.profiler), which tells whether the call is bound by the GPU or
by the host's launches.  Needs a GPU.  Usage: python tools/time_u2net.py [--iters 20] [--json out.json]"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

GFLOP_PER_IMAGE = 117.2


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        q = torch.cuda.get_device_name(0) + ", power limit unknown"
    return q


def time_calls(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def engine_shares(fn):
    """Kernel time by engine over one call, from torch.profiler (CUDA activities)."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    tot = {"tc5": 0.0, "mma": 0.0, "other": 0.0}
    from torch.autograd import DeviceType
    for ev in prof.key_averages():
        if ev.device_type != DeviceType.CUDA:     # kernels only: a host op's device time repeats its kernels'
            continue
        t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
        name = ev.key
        if "gemm_tc5_kernel" in name:
            tot["tc5"] += t
        elif "gemm_kernel" in name or "gemm_mma" in name:
            tot["mma"] += t
        else:
            tot["other"] += t
    return tot


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--json", type=str, default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "time_u2net.py needs a GPU"
    import u2net_oracle as UO
    from hi3d_official_b200.u2net import U2NetTower
    dev = torch.device("cuda", 0)
    tower = U2NetTower(UO.random_u2net_sd(seed=1, variant="full"), device=dev)
    res = {"card": card()}
    for n in (1, 16):
        x = torch.randn(n, 3, 320, 320, generator=torch.Generator().manual_seed(2)).to(dev)
        ms = time_calls(lambda: tower(x), a.iters)
        sh = engine_shares(lambda: tower(x))
        conv = sh["tc5"] + sh["mma"]
        r = dict(ms=round(ms, 3), tflops=round(GFLOP_PER_IMAGE * n / ms, 1), mma_share_of_conv_time=round(sh["mma"] / conv, 3),
                 conv_share_of_kernel_time=round(conv / (conv + sh["other"]), 3),
                 kernel_ms=round((conv + sh["other"]) / 1000.0, 3))
        res[f"batch{n}"] = r
        print(f"U^2-Net {n} x 320^2: {ms:.2f} ms/call, {r['tflops']} TFLOP/s ({GFLOP_PER_IMAGE * n:.1f} GFLOP); convs on mma.sync "
              f"{100 * r['mma_share_of_conv_time']:.0f} % of conv time; convs {100 * r['conv_share_of_kernel_time']:.0f} % of "
              f"kernel time; kernels {r['kernel_ms']:.2f} ms of the call (the rest is host / launch time)")
    print(f"card: {res['card']}")
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
