#!/usr/bin/env python
"""Time every distinct GEMM shape of one stage-2 UNet forward (32 x 128^2 latents: the CFG batch of 2 x 16 frames, synthetic
weights) on the wgmma engine (hi3d_gemm_tc5), with the engine's automatic choice and with single 128-row tiles forced
(hi3d_gemm_tc5_set_pair_mode(0)), alternated in the same process.

The plan's ops.Gemm launches are grouped by (rows mode, M, N, K, activation, residual, blend, upsample class, stride), as
bench.py's gemm_shapes_top groups them.  After one eager forward (so every buffer holds the values a forward leaves there) and
warm-up, each shape is timed --reps times per mode: CUDA events around all of its launches back to back, divided by the
launch count.  Per shape it prints the schedule the engine picks (hi3d_gemm_tc5_schedule), the median ms per launch of both
modes and their run-to-run spread ((max - min) / median), TFLOP/s, and two lower bounds from the shape alone: the FLOPs at
--tflops and the bytes that must cross HBM at least once (every distinct A channel range, W, the output, residual and blend)
at --tbs.  The card's name, power limit and maximum SM clock are read in the same run.  Needs a GPU.

    python tools/time_gemm.py [--reps 20] [--tflops 800] [--tbs 3.0] [--json out.json]
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

H, T = 128, 16          # stage 2: 1024^2 / 8 latents, 16 frames; the sampler's UNet batch is 2 x 16 (CFG)
SCHEDULES = {0: "mma.sync", 1: "single", 2: "pair", 3: "pingpong"}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else \
        torch.cuda.get_device_name(0) + ", power limit not readable"


def stage2_plan():
    from hi3d_official_b200 import configs, ops, spec
    from hi3d_official_b200.unet import VideoUNet
    cfg = configs.stage2_config()["model"]["params"]["network_config"]["params"]
    net = VideoUNet(**cfg).cuda().half()
    spec.synth_fill_(net, seed=0, fast=True)
    net.set_engine("tc5")
    N = 2 * T
    g = torch.Generator(device="cuda").manual_seed(2)
    x = torch.randn(N, net.cfg.in_channels, H, H, device="cuda", generator=g)
    ctx = torch.randn(N // T, 1, net.cfg.context_dim, device="cuda", generator=g)
    y = torch.randn(N // T, net.cfg.adm_in_channels, device="cuda", generator=g)
    plan = net.get_plan(N, H, H, T)
    plan.prepare_conditioning(ctx, y)
    ops.nchw_to_nhwc(x.contiguous(), plan.xin.t.view(N, H, H, -1))
    plan.set_timesteps(torch.full((N,), 0.7, device="cuda"))
    plan.run()
    torch.cuda.synchronize()
    return net, plan


def shape_key(p):
    return (p.mode, p.M, p.N, p.K, p.act, bool(p.residual), bool(p.blend_x), p.out_up, p.stride)


def key_str(k):
    mode, M, N, K, act, res, bl, up, st = k
    return f"mode{mode} M={M} N={N} K={K} act={act}" + (" res" if res else "") + (" blend" if bl else "") + \
        (" up" if up else "") + (" s2" if st == 2 else "")


def min_bytes(g):
    """Bytes one launch must move through HBM at least once: each distinct channel range of each A source, W, out, residual,
    blend."""
    p = g.p
    segs = g._keep[0]
    ranges = {}
    for s in segs:
        rows = s.src.numel() // s.ld
        ranges.setdefault((s.src.data_ptr(), rows), set()).add((s.c_off, s.C))
    a = sum(rows * sum(c for _, c in rs) for (_, rows), rs in ranges.items())
    n_out = p.N // 2 if p.act == 2 else p.N
    rows_out = p.M
    b = a + p.N * p.K + rows_out * n_out * (1 + bool(p.residual) + bool(p.blend_x))
    return 2.0 * b


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--tflops", type=float, default=800.0, help="tensor-core rate of the FLOP bound, TFLOP/s")
    ap.add_argument("--tbs", type=float, default=3.0, help="HBM rate of the byte bound, TB/s")
    ap.add_argument("--json", type=str, default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_gemm.py needs a GPU")
    if a.reps < 20:
        raise SystemExit("time at least 20 repetitions per shape and mode")
    from hi3d_official_b200 import _native, ops
    lib = _native.load()
    schedule = getattr(lib, "hi3d_gemm_tc5_schedule", None)    # absent in builds that predate the query
    net, plan = stage2_plan()
    groups = {}
    for s in plan.steps:
        if isinstance(s, ops.Gemm) and not s.fp8:
            groups.setdefault(shape_key(s.p), []).append(s)

    def time_group(steps, mode):
        _native.check(lib.hi3d_gemm_tc5_set_pair_mode(mode), "set_pair_mode")
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for s in steps:
            s()
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1) / len(steps)

    rows = []
    try:
        for k, steps in groups.items():
            for mode in (-1, 0, -1, 0):
                time_group(steps, mode)
            t = {-1: [], 0: []}
            for _ in range(a.reps):
                for mode in (-1, 0):
                    t[mode].append(time_group(steps, mode))
            _native.check(lib.hi3d_gemm_tc5_set_pair_mode(-1), "set_pair_mode")
            sc = None
            if schedule is not None:
                r = schedule(ctypes.byref(steps[0].p))
                sc = f"{SCHEDULES.get(r // 1000, r)}/{r % 1000}" if r >= 0 else f"error {r}"
            fl = steps[0].flops
            by = min_bytes(steps[0])
            auto, single = statistics.median(t[-1]), statistics.median(t[0])
            rows.append(dict(
                shape=key_str(k), launches=len(steps), schedule=sc, gflop=round(fl / 1e9, 2),
                auto_ms=round(auto, 4), auto_spread=round((max(t[-1]) - min(t[-1])) / auto, 4),
                single_ms=round(single, 4), single_spread=round((max(t[0]) - min(t[0])) / single, 4),
                speedup=round(single / auto, 3), auto_tflops=round(fl / auto / 1e9, 1),
                flop_bound_ms=round(fl / (a.tflops * 1e9), 4), byte_bound_ms=round(by / (a.tbs * 1e9), 4),
                auto_vs_bound=round(max(fl / (a.tflops * 1e9), by / (a.tbs * 1e9)) / auto, 3)))
    finally:
        lib.hi3d_gemm_tc5_set_pair_mode(-1)
    rows.sort(key=lambda r: -r["auto_ms"] * r["launches"])
    tot = {m: sum(r[f"{m}_ms"] * r["launches"] for r in rows) for m in ("auto", "single")}
    bound = sum(max(r["flop_bound_ms"], r["byte_bound_ms"]) * r["launches"] for r in rows)
    res = dict(card=card(), reps=a.reps, rates=dict(tflops=a.tflops, tbs=a.tbs), shapes=rows,
               total_ms=dict(auto=round(tot["auto"], 2), single=round(tot["single"], 2), bound=round(bound, 2)))
    print(f"card: {res['card']}")
    print(f"{'shape':<58} {'n':>3} {'schedule':>13} {'auto ms':>8} {'spread':>6} {'single ms':>9} {'spread':>6} "
          f"{'x':>6} {'TF/s':>6} {'flop bd':>8} {'byte bd':>8} {'bd/auto':>7}")
    for r in rows:
        print(f"{r['shape']:<58} {r['launches']:>3} {str(r['schedule']):>13} {r['auto_ms']:>8.4f} {r['auto_spread']:>6.3f} "
              f"{r['single_ms']:>9.4f} {r['single_spread']:>6.3f} {r['speedup']:>6.3f} {r['auto_tflops']:>6.1f} "
              f"{r['flop_bound_ms']:>8.4f} {r['byte_bound_ms']:>8.4f} {r['auto_vs_bound']:>7.3f}")
    print(f"one forward's GEMMs (sum of per-shape medians x launches): auto {res['total_ms']['auto']} ms, single "
          f"{res['total_ms']['single']} ms, bound {res['total_ms']['bound']} ms")
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
