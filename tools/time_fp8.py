#!/usr/bin/env python
"""Time the UNet forward in fp16, fp8 and fp8_attn precision (VideoUNet.set_precision) at the stage-1 (32 x 64^2 latents) and
stage-2 (32 x 128^2) shapes of the sampler: the CFG batch of 2 x 16 frames, synthetic weights, one forward = one CUDA-graph replay
of the launch plan, as the fused sampler step replays it.  The three plans are alternated in rounds; each reports the median of the
timed forwards after warm-up, the split of one eager forward by kind of launch (CUDA events around every launch; spatial and
temporal attention apart), and the relative L2 differences of the outputs on the same seeded inputs.  The card's name, power limit and maximum SM
clock are read in the same run.  Needs a GPU.
Usage: python tools/time_fp8.py [--stages 1 2] [--rounds 4] [--reps 6] [--json out.json]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = {1: 64, 2: 128}        # latent side per stage (512^2 / 8, 1024^2 / 8); T = 16 frames, CFG batch 2 x 16
T = 16
PRECS = ("fp16", "fp8", "fp8_attn")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else \
        torch.cuda.get_device_name(0) + ", power limit not readable"


def unet(stage):
    from hi3d_official_b200 import configs, spec
    from hi3d_official_b200.unet import VideoUNet
    cfg = (configs.stage1_config() if stage == 1 else configs.stage2_config())["model"]["params"]["network_config"]["params"]
    net = VideoUNet(**cfg).cuda().half()
    spec.synth_fill_(net, seed=0, fast=True)
    return net


def graph_of(plan):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        plan.run()                      # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        plan.run()
    return g


def split(plan):
    """ms per kind of launch over one eager forward (events around each launch)."""
    from hi3d_official_b200 import ops
    recs = []
    for s in plan.steps:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); s(); e1.record()
        recs.append((s, e0, e1))
    torch.cuda.synchronize()
    out = {}
    for s, e0, e1 in recs:
        if isinstance(s, ops.Gemm):
            k = "gemm_fp8" if s.fp8 else "gemm_fp16"
        else:
            k = getattr(s, "kind", "other")
        out[k] = out.get(k, 0.0) + e0.elapsed_time(e1)
    return {k: round(v, 2) for k, v in sorted(out.items())}


def run_stage(stage, rounds, reps):
    from hi3d_official_b200 import ops
    net = unet(stage)
    h = SHAPES[stage]
    N = 2 * T
    cfg = net.cfg
    g = torch.Generator(device="cuda").manual_seed(stage)
    x = torch.randn(N, cfg.in_channels, h, h, device="cuda", generator=g)
    ctx = torch.randn(N // T, 1, cfg.context_dim, device="cuda", generator=g)
    y = torch.randn(N // T, cfg.adm_in_channels, device="cuda", generator=g)
    t = torch.full((N,), 0.7, device="cuda")
    plans, graphs = {}, {}
    for prec in PRECS:
        net.set_precision(prec)
        p = plans[prec] = net.get_plan(N, h, h, T)      # set_precision drops the cache, the plan object stays alive here
        p.prepare_conditioning(ctx, y)
        ops.nchw_to_nhwc(x.contiguous(), p.xin.t.view(N, h, h, -1))
        p.set_timesteps(t)
        graphs[prec] = graph_of(p)
    torch.cuda.synchronize()
    res = {"latents": f"{N} x {h}^2", "fp8_layers": len(plans["fp8"].fp8_layers)}
    outs = {}
    for prec, p in plans.items():
        graphs[prec].replay()
        torch.cuda.synchronize()
        outs[prec] = p.net_out.t[:, :cfg.out_channels].float().clone()
    for a, b in (("fp8", "fp16"), ("fp8_attn", "fp16"), ("fp8_attn", "fp8")):
        res[f"rel_l2_{a}_vs_{b}"] = float((outs[a] - outs[b]).norm() / outs[b].norm())
    times = {prec: [] for prec in PRECS}
    for prec in PRECS:
        for _ in range(3):
            graphs[prec].replay()
    for _ in range(rounds):
        for prec in PRECS:
            for _ in range(reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(); graphs[prec].replay(); e1.record()
                e1.synchronize()
                times[prec].append(e0.elapsed_time(e1))
    for prec in PRECS:
        res[prec] = dict(median_ms=round(statistics.median(times[prec]), 2), n=len(times[prec]),
                         min_ms=round(min(times[prec]), 2), max_ms=round(max(times[prec]), 2), split_ms=split(plans[prec]))
    res["speedup"] = round(res["fp16"]["median_ms"] / res["fp8"]["median_ms"], 3)
    res["speedup_fp8_attn_vs_fp8"] = round(res["fp8"]["median_ms"] / res["fp8_attn"]["median_ms"], 3)
    res["fp8_attention_blocks"] = len(plans["fp8_attn"].fp8_attention)
    del graphs, plans, net
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--stages", type=int, nargs="+", default=[1, 2])
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--reps", type=int, default=6)
    ap.add_argument("--json", type=str, default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_fp8.py needs a GPU")
    if a.rounds * a.reps < 20:
        raise SystemExit("time at least 20 forwards per precision (--rounds x --reps)")
    res = {"card": card(), "stages": {}}
    for st in a.stages:
        r = res["stages"][st] = run_stage(st, a.rounds, a.reps)
        print(f"stage {st} ({r['latents']}, {r['fp8_layers']} fp8 layers): fp16 {r['fp16']['median_ms']} ms, fp8 "
              f"{r['fp8']['median_ms']} ms per forward (median of {r['fp8']['n']}), x{r['speedup']}; rel. L2 fp8 vs fp16 "
              f"{r['rel_l2_fp8_vs_fp16']:.3e}")
        print(f"  fp8_attn ({r['fp8_attention_blocks']} e4m3 attention blocks): {r['fp8_attn']['median_ms']} ms, x"
              f"{r['speedup_fp8_attn_vs_fp8']} vs fp8; rel. L2 vs fp16 {r['rel_l2_fp8_attn_vs_fp16']:.3e}, vs fp8 "
              f"{r['rel_l2_fp8_attn_vs_fp8']:.3e}")
        for prec in PRECS:
            print(f"  {prec} split (one eager forward, ms): {r[prec]['split_ms']}")
    print(f"card: {res['card']}")
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
