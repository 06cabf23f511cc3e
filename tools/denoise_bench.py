#!/usr/bin/env python
"""Cost and quality of rtDenoise (the a-trous denoiser) on the GPU.

    python tools/denoise_bench.py [--quick] [--min-seconds 0.3] [--ab ray_tracing_b200/variants/librt_b200_denoise_plain.so]

Timing, per image size (1080p, 4K of the knot room with glass, one accumulated 1-spp frame and its feature images): rtDenoise for
iterations 1 / 3 / 5 and both sources, CUDA events around the call on the context's stream, after a warm-up call, each arm repeated
over at least --min-seconds, the arms alternated three times (median and min..max of the three reported in ms); the 1-spp frame of
the same workload beside it (RtStats.kernelMs).  With --ab, a second library (the -DRT_DENOISE_PLAIN build: every tap from global
memory) is timed in the same rounds, and its DenoisedRender must equal this build's bit for bit.  Counted from shapes: bytes moved at
the minimum (prepare: 48 read + 48 written per pixel; a pass: 32 read + 16 written, the last 16 more read) and the exp_rt calls at
most made (24 per pixel per iteration).

Quality, at 320 x 180: relative MSE of the noisy mean and of the denoised mean (managers' defaults) against a 1024-sample render of
the same scene, after 1 / 4 / 16 frames, on the Cornell box, the knot room and the 871k-triangle cluster.
Prints the card name, power limit and max SM clock read in the same run.  Fails without a GPU.
"""
import argparse
import json
import os
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tests"))
sys.path.insert(0, os.path.join(REPO, "tools"))
from conftest import CUDA_LIB                                     # noqa: E402
import ray_tracing_b200 as rt                                     # noqa: E402
from ray_tracing_b200 import capi, scenes                         # noqa: E402
from trace_rays_bench import card, timed                          # noqa: E402


def open_scene(lib, sc, frames, rays_per_pixel=1):
    sc.settings = dict(sc.settings, numRaysPerPixel=rays_per_pixel)
    mgr = rt.RayComputeManager(lib)
    scenes.apply(sc, mgr)
    mgr.OnEnable()
    ctx = mgr.context
    for f in range(1, frames + 1):
        ctx.set_int("Frame", f)
        ctx.dispatch_features()
        ctx.dispatch_full()
    ctx.synchronize()
    return mgr, ctx


def timing_rows(args, torch, hd, uhd):
    libs = {"tiled": CUDA_LIB}
    if args.ab:
        libs["plain"] = os.path.abspath(args.ab)
    for size in (hd, uhd):
        W, H = size
        n = W * H
        ctxs, mgrs, streams = {}, [], {}
        for arm, lib in libs.items():
            mgr, ctx = open_scene(lib, scenes.knot_room(W, H, 8, 1, glass=True), 1)
            streams[arm] = torch.cuda.Stream()
            ctx.set_stream(streams[arm].cuda_stream)
            ctxs[arm] = ctx
            mgrs.append(mgr)
        first = ctxs["tiled"]
        first.synchronize()
        t0 = first.stats()["kernelMs"]
        first.dispatch_full()
        first.synchronize()
        frame_ms = first.stats()["kernelMs"] - t0
        cases = [(acc, k) for acc in (1, 0) for k in (1, 3, 5)]
        for acc, k in cases:                                  # the arms compute the same bits
            imgs = {}
            for arm, ctx in ctxs.items():
                ctx.denoise(bool(acc), k)
                imgs[arm] = ctx.readback("DenoisedRender")
            for arm, img in imgs.items():
                same = (img.view(np.uint32) == imgs["tiled"].view(np.uint32)) | (np.isnan(img) & np.isnan(imgs["tiled"]))
                if not same.all():
                    sys.exit(f"denoise_bench: {arm} differs from tiled at {W}x{H} acc={acc} iterations={k}")
        ms = {(arm, acc, k): [] for arm in ctxs for acc, k in cases}
        for _ in range(3):
            for acc, k in cases:
                for arm, ctx in ctxs.items():
                    stream = streams[arm]

                    def clock(fn):
                        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        a.record(stream)
                        fn()
                        b.record(stream)
                        b.synchronize()
                        return a.elapsed_time(b) / 1e3
                    ms[(arm, acc, k)].append(timed(lambda: ctx.denoise(bool(acc), k), args.min_seconds, clock) * 1e3)
        for acc, k in cases:
            bytes_ = n * (96 + 48 * k + 16)
            exps = 24 * n * k
            row = {"size": f"{W}x{H}", "source": "accumulated" if acc else "frame", "iterations": k, "frame_1spp_ms": round(frame_ms, 3)}
            for arm in ctxs:
                v = ms[(arm, acc, k)]
                med = float(np.median(v))
                row[arm + "_ms"] = round(med, 4)
                row[arm + "_spread"] = [round(float(min(v)), 4), round(float(max(v)), 4)]
                row[arm + "_GBps"] = round(bytes_ / med / 1e6, 1)
                row[arm + "_Gexp_per_s"] = round(exps / med / 1e6, 1)
            print(json.dumps(row), flush=True)
        for ctx in ctxs.values():
            ctx.set_stream(0)
        for mgr in mgrs:
            mgr.OnDestroy()


def rel_mse(x, ref):
    return float(np.mean((x[..., :3].astype(np.float64) - ref[..., :3]) ** 2 / (ref[..., :3].astype(np.float64) ** 2 + 0.01)))


def quality_rows(size):
    W, H = size
    for name, make in (("cornell", lambda: scenes.cornell_spheres(W, H, 4, 1)),
                       ("knot_room", lambda: scenes.knot_room(W, H, 8, 1, glass=True)),
                       ("knot_cluster 871k", lambda: scenes.knot_cluster(W, H, 12, 1))):
        mgr, ctx = open_scene(CUDA_LIB, make(), 16, rays_per_pixel=64)
        acc = ctx.readback("AccumulatedRender")
        ref = acc[..., :3] / acc[..., 3:4]
        mgr.OnDestroy()
        mgr, ctx = open_scene(CUDA_LIB, make(), 0)
        row = {"quality": name, "size": f"{W}x{H}", "reference_spp": 1024}
        for frames in (1, 4, 16):
            done = {1: 0, 4: 1, 16: 4}[frames]
            for f in range(done + 1, frames + 1):
                ctx.set_int("Frame", f)
                ctx.dispatch_features()
                ctx.dispatch_full()
            acc = ctx.readback("AccumulatedRender")
            ctx.denoise(True)
            noisy, den = rel_mse(acc[..., :3] / acc[..., 3:4], ref), rel_mse(ctx.readback("DenoisedRender"), ref)
            row[f"frames{frames}"] = {"noisy": round(noisy, 4), "denoised": round(den, 4), "factor": round(noisy / den, 1)}
        mgr.OnDestroy()
        print(json.dumps(row), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="small frames (a rehearsal, not a measurement)")
    ap.add_argument("--min-seconds", type=float, default=0.3)
    ap.add_argument("--ab", default="", help="a second librt_b200.so to time in the same rounds")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("denoise_bench: no CUDA device")
    print(json.dumps({"card": card(), "lib": os.path.relpath(CUDA_LIB, REPO), "ab": args.ab,
                      "defaults": [capi.DENOISE_ITERATIONS, capi.DENOISE_SIGMA_COLOUR, capi.DENOISE_SIGMA_NORMAL, capi.DENOISE_SIGMA_DEPTH]}),
          flush=True)
    hd, uhd = ((192, 108), (384, 216)) if args.quick else ((1920, 1080), (3840, 2160))
    timing_rows(args, torch, hd, uhd)
    quality_rows((64, 36) if args.quick else (320, 180))
    return 0


if __name__ == "__main__":
    sys.exit(main())
