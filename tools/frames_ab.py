#!/usr/bin/env python
"""How much faster is one rtDispatchFrames(n) than the n rtDispatch calls it replaces?  (1 spp per frame, accumulate on.)

    python tools/frames_ab.py [--n 8 64] [--rounds 3] [--workloads cornell knot cluster] [--out FILE]

Per workload, in one process: one context, the two arms alternated `rounds` times (A = n rtDispatch calls with "Frame" stepped,
B = one rtDispatchFrames(n)), each arm timed by the library's CUDA events (RtStats.kernelMs: the sum over the arm's launches) and by a
host clock around the arm, ended by a synchronise.  Both are reported per frame.  The two arms' images are then compared bitwise at
the timed size, from the same zeroed accumulation and the same first frame.  On a box with two or more GPUs the runs repeat on a group
context over all of them (rtCreateMulti: row-band tiles, one exchange per dispatch for A, one per batch for B).
The card's name, power limit and SM clock (sampled while the arms run) are printed with the numbers.
"""
import argparse
import os
import subprocess
import sys
import threading
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import ray_tracing_b200 as rt                      # noqa: E402
from ray_tracing_b200 import capi, scenes          # noqa: E402
from ray_tracing_b200.build import LIB_CUDA        # noqa: E402

WORKLOADS = {
    "cornell": ("9-sphere Cornell box (configs[1]), 1920x1080, 8 bounces", lambda: scenes.cornell_spheres(1920, 1080, 8, 1)),
    "knot": ("87,132-triangle knot room, 1920x1080, 8 bounces", lambda: scenes.knot_room(1920, 1080, 8, 1)),
    "cluster": ("871,212-triangle glass knot cluster, 3840x2160, 12 bounces", lambda: scenes.knot_cluster(3840, 2160, 12, 1)),
}


def smi(fields, index=0):
    r = subprocess.run(["nvidia-smi", "-i", str(index), f"--query-gpu={fields}", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True, timeout=30)
    return [x.strip() for x in r.stdout.strip().split(",")] if r.returncode == 0 else None


class ClockSampler:
    """SM clock (MHz) of GPU 0, polled while the arms run."""
    def __init__(self):
        self.samples, self._stop = [], threading.Event()
        self._t = threading.Thread(target=self._run, daemon=True)

    def _run(self):
        while not self._stop.is_set():
            v = smi("clocks.sm")
            if v and v[0].isdigit():
                self.samples.append(int(v[0]))
            self._stop.wait(0.25)

    def __enter__(self):
        self._t.start()
        return self

    def __exit__(self, *exc):
        self._stop.set()
        self._t.join()

    def summary(self):
        if not self.samples:
            return "SM clock not sampled"
        s = np.array(self.samples)
        return f"SM clock median {int(np.median(s))} MHz (min {s.min()}, max {s.max()}, {len(s)} samples)"


def arm(ctx, n, batched, F, groups):
    ctx.reset_stats()
    ctx.set_int("Frame", F)
    t0 = time.perf_counter()
    if batched:
        ctx.dispatch_frames(n, *groups)
    else:
        for k in range(n):
            ctx.set_int("Frame", F + k)
            ctx.dispatch(capi.RT_KERNEL_RAYTRACE, *groups)
        ctx.set_int("Frame", F)
    ctx.synchronize()
    wall = (time.perf_counter() - t0) * 1e3
    st = ctx.stats()
    return st["kernelMs"], wall, st["exchangeMs"]


def measure(name, devices, ns, rounds, log):
    desc, make = WORKLOADS[name]
    sc = make()
    mgr = rt.RayComputeManager(LIB_CUDA, devices=devices) if devices else rt.RayComputeManager(LIB_CUDA)
    scenes.apply(sc, mgr)
    mgr.OnEnable()
    ctx = mgr.context
    groups = ((sc.width + 7) // 8, (sc.height + 7) // 8, 1)
    where = f"group of {len(devices)} GPUs" if devices else "1 GPU"
    arm(ctx, 2, False, 1, groups)                          # warm-up: modules, scene upload, both kernel families
    arm(ctx, 2, True, 1, groups)
    with ClockSampler() as clk:
        for n in ns:
            res = {False: [], True: []}
            for r in range(rounds):
                for batched in ((False, True) if r % 2 == 0 else (True, False)):
                    res[batched].append(arm(ctx, n, batched, 1 + r * n, groups))
            a, b = np.array(res[False]), np.array(res[True])
            # bitwise: both arms from a zeroed accumulation and the same first frame
            imgs = []
            for batched in (False, True):
                ctx.dispatch(capi.RT_KERNEL_RESET_ACCUMULATED, *groups)
                arm(ctx, n, batched, 1, groups)
                imgs.append((ctx.readback("FrameRender"), ctx.readback("AccumulatedRender")))
            same = all(np.array_equal(x.view(np.uint32), y.view(np.uint32)) for x, y in zip(imgs[0], imgs[1]))
            assert same, f"{name} n={n} {where}: the batch's images differ from the dispatches'"
            line = (f"{name:8s} {where:16s} n={n:3d}  kernel ms/frame: dispatches {np.median(a[:, 0]) / n:8.3f}  batch {np.median(b[:, 0]) / n:8.3f}"
                    f"  ({np.median(a[:, 0]) / np.median(b[:, 0]):5.3f}x)   host ms/frame: dispatches {np.median(a[:, 1]) / n:8.3f}  batch {np.median(b[:, 1]) / n:8.3f}"
                    f"  ({np.median(a[:, 1]) / np.median(b[:, 1]):5.3f}x)"
                    + (f"   exchange ms/frame: {np.median(a[:, 2]) / n:.3f} vs {np.median(b[:, 2]) / n:.3f}" if devices else "")
                    + f"   [medians of {rounds}; spread kernel {a[:, 0].min() / n:.3f}-{a[:, 0].max() / n:.3f} / {b[:, 0].min() / n:.3f}-{b[:, 0].max() / n:.3f}; images bitwise equal]")
            log(line)
    log(f"         {desc}: {clk.summary()}")
    mgr.OnDestroy()


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--n", type=int, nargs="+", default=[8, 64])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--workloads", nargs="+", default=list(WORKLOADS), choices=list(WORKLOADS))
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    lines = []

    def log(s):
        print(s, flush=True)
        lines.append(s)

    card = smi("name,power.limit,clocks.max.sm")
    if card is None:
        sys.exit("frames_ab: nvidia-smi found no GPU; this tool measures on the GPU only")
    log(f"card: {card[0]}, power limit {card[1]} W, max SM clock {card[2]} MHz")
    import torch
    n_gpu = torch.cuda.device_count()
    for name in args.workloads:
        measure(name, None, args.n, args.rounds, log)
        if n_gpu >= 2:
            measure(name, list(range(n_gpu)), args.n, args.rounds, log)
    if n_gpu < 2:
        log("group context: not measured (one GPU)")
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
