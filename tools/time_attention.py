#!/usr/bin/env python
"""Time the d = 64 spatial attention kernel (hi3d_attention_d64_tc5) at the four stage-2 UNet shapes (32 images x L tokens
x heads: 16384 x 5, 4096 x 10, 1024 x 20, 256 x 20).  Each measurement is CUDA events around as many back-to-back calls as
fill --window seconds, after warm-up.  Several libraries (--lib, any build of libhi3d_b200.so with the same C signature,
e.g. one built from an earlier commit) are timed in one process, alternating between them over --rounds rounds, so that
clock and power drift hits them alike.  --variants / --emus sweep hi3d_attention_tc5_set_variant and
hi3d_attention_tc5_set_exp_emulation; without them each library runs its own default.  --fp8 adds, for every library, the e4m3
path (hi3d_attention_vt_e4m3 + hi3d_attention_d64_tc5_fp8, reported as "fp8_path") and its kernel alone ("fp8_kernel"),
alternated with the fp16 kernel in the same rounds, on the same (e4m3-representable) values; every entry's TFLOP/s counts the
same 4 L^2 C n_img.  Prints one JSON line with the card's name, power limit and max SM clock beside the times.

    python tools/time_attention.py [--lib PATH ...] [--rounds 3] [--window 1.0] [--variants 0,6] [--emus 0,1] [--fp8]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = {"ds1": (32, 16384, 5), "ds2": (32, 4096, 10), "ds4": (32, 1024, 20), "ds8": (32, 256, 20)}


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def load(path):
    lib = C.CDLL(os.path.abspath(path))
    lib.hi3d_attention_d64_tc5.restype = C.c_int
    lib.hi3d_attention_d64_tc5.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_float, C.c_void_p, C.c_void_p]
    for f in ("hi3d_attention_tc5_set_variant", "hi3d_attention_tc5_set_exp_emulation"):
        getattr(lib, f).restype = C.c_int
        getattr(lib, f).argtypes = [C.c_int]
    lib.hi3d_last_error.restype = C.c_char_p
    if hasattr(lib, "hi3d_attention_d64_tc5_fp8"):
        lib.hi3d_attention_vt_e4m3.restype = C.c_int
        lib.hi3d_attention_vt_e4m3.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
        lib.hi3d_attention_vt_e4m3_bytes.restype = C.c_int64
        lib.hi3d_attention_vt_e4m3_bytes.argtypes = [C.c_int, C.c_int, C.c_int]
        lib.hi3d_attention_d64_tc5_fp8.restype = C.c_int
        lib.hi3d_attention_d64_tc5_fp8.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_float, C.c_void_p,
                                                   C.c_void_p]
    return lib


def check(lib, rc, what):
    if rc != 0:
        raise RuntimeError(f"{what}: {lib.hi3d_last_error().decode()}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", help="library to time (repeatable); default: this tree's build")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--window", type=float, default=1.0, help="seconds of calls per measurement")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--variants", help="comma-separated hi3d_attention_tc5_set_variant values")
    ap.add_argument("--emus", help="comma-separated hi3d_attention_tc5_set_exp_emulation values")
    ap.add_argument("--fp8", action="store_true", help="also time the e4m3 path (transpose + kernel) and its kernel alone")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_attention.py needs a CUDA device")
    if not a.lib:
        from hi3d_official_b200 import build
        a.lib = [build.build()]
    libs = [(p, load(p)) for p in a.lib]
    variants = [int(v) for v in a.variants.split(",")] if a.variants else [None]
    emus = [int(e) for e in a.emus.split(",")] if a.emus else [None]
    configs = [(v, e) for v in variants for e in emus]
    if a.fp8:
        missing = [p for p, lib in libs if not hasattr(lib, "hi3d_attention_d64_tc5_fp8")]
        if missing:
            sys.exit(f"--fp8: {missing} have no hi3d_attention_d64_tc5_fp8")
    # entries: (library index, config, what) -- what = "fp16", "fp8_path" or "fp8_kernel"; configs only apply to fp16
    entries = [(li, cfg, "fp16") for li in range(len(libs)) for cfg in configs]
    if a.fp8:
        entries += [(li, (None, None), w) for li in range(len(libs)) for w in ("fp8_path", "fp8_kernel")]
    stream = torch.cuda.current_stream()
    res = {"gpu": card(), "rounds": a.rounds, "window_s": a.window, "libs": a.lib, "results": []}

    def setup(lib, cfg):
        v, e = cfg
        if v is not None:
            check(lib, lib.hi3d_attention_tc5_set_variant(v), "set_variant")
        if e is not None:
            check(lib, lib.hi3d_attention_tc5_set_exp_emulation(e), "set_exp_emulation")

    for name in a.shapes.split(","):
        n_img, L, heads = SHAPES[name]
        C_ = heads * 64
        g = torch.Generator(device="cuda").manual_seed(1)
        qkv = torch.randn(n_img * L, 3 * C_, device="cuda", generator=g).half()
        qkv8 = None
        if a.fp8:       # both paths see the same values: e4m3 for the e4m3 path, the same values in fp16 for the fp16 kernel
            qkv8 = qkv.to(torch.float8_e4m3fn)
            qkv = qkv8.half()
            vt = torch.empty(int(libs[0][1].hi3d_attention_vt_e4m3_bytes(n_img, L, heads)), dtype=torch.uint8, device="cuda")
        out = torch.empty(n_img * L, C_, device="cuda", dtype=torch.float16)
        flop = 4.0 * n_img * heads * L * L * 64
        st = C.c_void_p(stream.cuda_stream)

        def call(lib, what):
            if what == "fp16":
                check(lib, lib.hi3d_attention_d64_tc5(qkv.data_ptr(), n_img, L, heads, 0.125, out.data_ptr(), st),
                      "hi3d_attention_d64_tc5")
                return
            if what == "fp8_path":
                check(lib, lib.hi3d_attention_vt_e4m3(qkv8.data_ptr(), n_img, L, heads, vt.data_ptr(), st), "hi3d_attention_vt_e4m3")
            check(lib, lib.hi3d_attention_d64_tc5_fp8(qkv8.data_ptr(), vt.data_ptr(), n_img, L, heads, 0.125, out.data_ptr(), st),
                  "hi3d_attention_d64_tc5_fp8")

        def timed(lib, what, n):
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(n):
                call(lib, what)
            t1.record()
            torch.cuda.synchronize()
            return t0.elapsed_time(t1) / n

        # warm-up and the call count of every entry: enough calls to fill the window
        calls, times = {}, {}
        for e in entries:
            li, cfg, what = e
            lib = libs[li][1]
            setup(lib, cfg)
            for _ in range(a.warmup):
                call(lib, "fp8_path" if what == "fp8_kernel" else what)
            calls[e] = max(3, int(a.window * 1e3 / timed(lib, what, 3)) + 1)
            times[e] = []
        for _ in range(a.rounds):
            for e in entries:
                li, cfg, what = e
                setup(libs[li][1], cfg)
                times[e].append(timed(libs[li][1], what, calls[e]))
        for (li, cfg, what), ts in times.items():
            ms = sorted(ts)[len(ts) // 2]
            res["results"].append({"shape": name, "n_img": n_img, "L": L, "heads": heads, "lib": li, "path": what,
                                   "variant": cfg[0], "emu": cfg[1], "calls": calls[li, cfg, what], "ms": round(ms, 4),
                                   "ms_min": round(min(ts), 4), "ms_max": round(max(ts), 4),
                                   "tflops": round(flop / ms / 1e9, 1)})
        del qkv, qkv8, out
    print(json.dumps(res))


if __name__ == "__main__":
    main()
