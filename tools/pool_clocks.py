#!/usr/bin/env python
"""Where the pooled kernel's time goes, per step kind, on the GPU (needs a library built with RT_POOL_CLOCKS).

    python tools/build_variants.py clocks                      # here or anywhere nvcc runs; no GPU needed
    python tools/pool_clocks.py [--lib ray_tracing_b200/variants/librt_b200_clocks.so ...] [--frames 2] [--out FILE]

Renders the default benchmark workload (the 87k-triangle knot room, 1920x1080, 8 bounces, 256 spp) with each library given and
prints, per step kind of the kernel (census, inner, leaf, next model, shade, refill, camera rays, ray queue): the share of the
warps' cycles, the number of steps per frame and the lanes (or slots) a step served on average.  The cycles are clock64()
differences taken by lane 0 of every warp, so they are warp-resident cycles: a step's share includes the time its warp waited
for issue slots and for memory, not only its own instructions.  The card's name and power limit are printed with the numbers.
"""
import argparse
import ctypes
import os
import subprocess
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import ray_tracing_b200 as rt                      # noqa: E402
from ray_tracing_b200 import build, scenes         # noqa: E402

KINDS = ["census", "inner", "leaf", "next", "shade", "refill", "camera", "queue"]
DEFAULT_LIB = os.path.join(build.PKG_DIR, "variants", "librt_b200_clocks.so")


def smi(fields):
    r = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={fields}", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True, timeout=30)
    return [x.strip() for x in r.stdout.strip().split(",")] if r.returncode == 0 else None


def profile(lib, frames, log):
    lib = os.path.abspath(lib)
    so = ctypes.CDLL(lib)
    if not hasattr(so, "rtxPoolClocks"):
        sys.exit(f"pool_clocks: {lib} was not built with RT_POOL_CLOCKS (tools/build_variants.py clocks)")
    so.rtxPoolClocks.argtypes = [ctypes.POINTER(ctypes.c_ulonglong), ctypes.c_int, ctypes.c_int]
    buf = (ctypes.c_ulonglong * (3 * len(KINDS)))()
    sc = scenes.knot_room(1920, 1080, 8, 256)
    mgr = rt.RayComputeManager(lib)
    scenes.apply(sc, mgr)
    mgr.OnEnable()
    ctx = mgr.context
    ctx.set_int("Frame", 1)
    ctx.dispatch_full(0)                                    # warm-up: modules, upload
    ctx.synchronize()
    so.rtxPoolClocks(buf, len(buf), 1)
    ctx.reset_stats()
    for f in range(frames):
        ctx.set_int("Frame", 2 + f)
        ctx.dispatch_full(0)
    ctx.synchronize()
    kms = ctx.stats()["kernelMs"] / frames
    if so.rtxPoolClocks(buf, len(buf), 1) != len(buf):
        sys.exit("pool_clocks: rtxPoolClocks failed")
    a = np.array(buf[:], dtype=np.float64).reshape(len(KINDS), 3)
    total = a[:, 0].sum()
    log(f"{os.path.basename(lib)}: kernel {kms:.1f} ms/frame (the marks included), {total / frames:.4g} warp-cycles per frame")
    log(f"  {'step kind':10s} {'cycles %':>9s} {'steps/frame':>13s} {'cycles/step':>12s} {'lanes/step':>11s}")
    for k, name in enumerate(KINDS):
        cyc, steps, lanes = a[k]
        log(f"  {name:10s} {100 * cyc / total:8.1f}% {steps / frames:13.4g} {cyc / max(steps, 1):12.1f} {lanes / max(steps, 1):11.1f}")
    mgr.OnDestroy()


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--lib", nargs="+", default=[DEFAULT_LIB])
    ap.add_argument("--frames", type=int, default=2)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    lines = []

    def log(s):
        print(s, flush=True)
        lines.append(s)

    card = smi("name,power.limit,clocks.max.sm")
    if card is None:
        sys.exit("pool_clocks: nvidia-smi found no GPU; this tool measures on the GPU only")
    log(f"card: {card[0]}, power limit {card[1]} W, max SM clock {card[2]} MHz; knot room 1920x1080, 8 bounces, 256 spp")
    for lib in args.lib:
        profile(lib, args.frames, log)
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
