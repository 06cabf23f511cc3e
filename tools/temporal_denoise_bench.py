#!/usr/bin/env python
"""Cost and quality of rtDenoiseTemporal (the temporal SVGF denoiser) on the GPU.

    python tools/temporal_denoise_bench.py [--quick] [--min-seconds 0.3]

Timing, per image size (1080p, 4K of the knot room with glass, one 1-spp frame and its feature images): rtDenoiseTemporal for
iterations 1 / 3 / 5 with a still camera after 8 calls (every pixel's history is long; the static rule: one history tap), with a
moving camera (the camera alternates between two poses 0.25 degrees apart on every call: the full reprojection with up to four taps
and, after 8 calls, a long history), and right after a jump cut (resetHistory = 1 on every call: every pixel takes the 7x7 estimate),
and rtDenoise of the same frame
(useAccumulated = 0) with the same iteration count, the three arms alternated in the same rounds.  CUDA events around the call on the
context's stream, after a warm-up call, each arm repeated over at least --min-seconds, three rounds (median and min..max of the three
reported in ms); the 1-spp frame of the same workload beside it (RtStats.kernelMs).

Quality, at 320 x 180: a 16-frame 1-spp orbit of the camera in the Cornell box and the knot room with and without its glass; per frame
the relative MSE of rtDenoiseTemporal (managers' defaults) and of rtDenoise(useAccumulated = 0) against a 1024-sample render at that
frame's camera, the mean over frames 8..16; and on a still camera the mean frame-to-frame change of both outputs over the same frames.
--ab a.so,b.so repeats the quality rows with other builds (tools/build_variants.py: the lattice prefilter, the history tolerances);
--sweep repeats them over a grid of sigmaLuminance, sigmaDepth and alpha with this build.
Prints the card name, power limit and max SM clock read in the same run.  Fails without a GPU.
"""
import argparse
import json
import math
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


def open_scene(sc, rays_per_pixel=1, lib=CUDA_LIB):
    sc.settings = dict(sc.settings, numRaysPerPixel=rays_per_pixel, accumulate=False)
    mgr = rt.RayComputeManager(lib)
    scenes.apply(sc, mgr)
    mgr.OnEnable()
    return mgr, mgr.context


def frame(ctx, f):
    ctx.set_int("Frame", f)
    ctx.dispatch_full()
    ctx.dispatch_features()


def timing_rows(args, torch, hd, uhd):
    for W, H in (hd, uhd):
        mgr, ctx = open_scene(scenes.knot_room(W, H, 8, 1, glass=True))
        stream = torch.cuda.Stream()
        ctx.set_stream(stream.cuda_stream)
        ctx.synchronize()
        t0 = ctx.stats()["kernelMs"]
        frame(ctx, 1)
        ctx.synchronize()
        frame_ms = ctx.stats()["kernelMs"] - t0
        arms = {}
        for k in (1, 3, 5):
            arms[("steady", k)] = lambda k=k: ctx.denoise_temporal(k)
            arms[("moving", k)] = lambda k=k: move(k)
            arms[("jump", k)] = lambda k=k: ctx.denoise_temporal(k, reset_history=True)
            arms[("rtDenoise", k)] = lambda k=k: ctx.denoise(False, k)

        def clock(fn):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            fn()
            b.record(stream)
            b.synchronize()
            return a.elapsed_time(b) / 1e3
        M0, M1 = np.asarray(scenes.knot_room(W, H, 8, 1, glass=True).cam_local_to_world, np.float64), None
        c, s_ = math.cos(math.radians(0.25)), math.sin(math.radians(0.25))
        M1 = M0 @ np.array([[c, 0, s_, 0], [0, 1, 0, 0], [-s_, 0, c, 0], [0, 0, 0, 1]])
        pose = [0]

        def move(k):
            pose[0] ^= 1
            ctx.set_matrix("CamLocalToWorldMatrix", M1 if pose[0] else M0)
            ctx.denoise_temporal(k)
        ms = {key: [] for key in arms}
        lens = {}
        for _ in range(3):
            for k in (1, 3, 5):
                for kind in ("steady", "moving", "jump", "rtDenoise"):
                    ctx.set_matrix("CamLocalToWorldMatrix", M0)
                    if kind in ("steady", "moving"):
                        for _ in range(8):
                            arms[(kind, k)]()            # a long history
                    ms[(kind, k)].append(timed(arms[(kind, k)], args.min_seconds, clock) * 1e3)
                    if kind in ("steady", "moving"):
                        fr = ctx.temporal_frame()
                        lens[kind] = fr[..., 2]
                        if kind == "moving":
                            moved = np.isfinite(fr[..., 0]) & (fr[..., 0] != np.arange(W)[None, :])
        for k in (1, 3, 5):
            row = {"size": f"{W}x{H}", "iterations": k, "frame_1spp_ms": round(frame_ms, 3)}
            for kind in ("steady", "moving", "jump", "rtDenoise"):
                v = ms[(kind, k)]
                row[kind + "_ms"] = round(float(np.median(v)), 4)
                row[kind + "_spread"] = [round(float(min(v)), 4), round(float(max(v)), 4)]
            print(json.dumps(row), flush=True)
        for kind, ln in lens.items():
            print(json.dumps({"size": f"{W}x{H}", "arm": kind, "history_length_median": float(np.median(ln[ln > 0])),
                              "history_length_min": float(ln[ln > 0].min())}), flush=True)
        print(json.dumps({"size": f"{W}x{H}", "arm": "moving", "pixels_reprojected_off_their_own_position": round(float(moved.mean()), 4)}),
              flush=True)
        ctx.set_stream(0)
        mgr.OnDestroy()


def rel_mse(x, ref):
    return float(np.mean((x[..., :3].astype(np.float64) - ref[..., :3]) ** 2 / (ref[..., :3].astype(np.float64) ** 2 + 0.01)))


def orbit(M0, k):
    M0 = np.asarray(M0, np.float64)
    p = M0 @ np.array([0.0, 0.0, 5.0, 1.0])
    c, s = math.cos(math.radians(0.75 * k)), math.sin(math.radians(0.75 * k))
    R = np.array([[c, 0, s, 0], [0, 1, 0, 0], [-s, 0, c, 0], [0, 0, 0, 1]])
    T = np.eye(4)
    T[:3, 3] = p[:3]
    Ti = np.eye(4)
    Ti[:3, 3] = -p[:3]
    return T @ R @ Ti @ M0


QUALITY_SCENES = (("cornell", lambda W, H: scenes.cornell_spheres(W, H, 4, 1)),
                  ("knot_room", lambda W, H: scenes.knot_room(W, H, 8, 1, glass=True)),
                  ("knot_room_no_glass", lambda W, H: scenes.knot_room(W, H, 8, 1, glass=False)))


def quality_row(lib, make, sc, refs, params):
    row = {}
    for moving in (True, False):
        mgr, ctx = open_scene(make(), lib=lib)
        t_err, s_err, t_out, s_out = [], [], [], []
        for k in range(16):
            ctx.set_matrix("CamLocalToWorldMatrix", orbit(sc.cam_local_to_world, k if moving else 0))
            frame(ctx, k + 1)
            ctx.denoise_temporal(*params)
            t = ctx.readback("DenoisedRender")
            ctx.denoise(False)
            s = ctx.readback("DenoisedRender")
            if k >= 7:
                t_err.append(rel_mse(t, refs[k if moving else 0]))
                s_err.append(rel_mse(s, refs[k if moving else 0]))
                t_out.append(t[..., :3].astype(np.float64))
                s_out.append(s[..., :3].astype(np.float64))
        mgr.OnDestroy()
        if moving:
            row["orbit_relmse_temporal"] = round(float(np.mean(t_err)), 5)
            row["orbit_relmse_spatial"] = round(float(np.mean(s_err)), 5)
            row["orbit_factor"] = round(float(np.mean(s_err) / np.mean(t_err)), 2)
        else:
            flick = lambda o: float(np.mean([np.mean(np.abs(a - b)) for a, b in zip(o[1:], o[:-1])]))
            row["still_flicker_temporal"] = round(flick(t_out), 5)
            row["still_flicker_spatial"] = round(flick(s_out), 5)
            row["still_flicker_factor"] = round(flick(s_out) / flick(t_out), 2)
    return row


def quality_rows(size, libs, grid):
    W, H = size
    for name, mk in QUALITY_SCENES:
        make = lambda: mk(W, H)
        sc = make()
        refs = []
        rmgr, rctx = open_scene(make(), rays_per_pixel=64)
        rctx.set_bool("accumulate", True)
        for k in range(16):
            rctx.set_matrix("CamLocalToWorldMatrix", orbit(sc.cam_local_to_world, k))
            rctx.dispatch_full(capi.RT_KERNEL_RESET_ACCUMULATED)
            for f in range(16):
                rctx.set_int("Frame", 1000 * k + f + 1)
                rctx.dispatch_full()
            acc = rctx.readback("AccumulatedRender")
            refs.append(acc[..., :3] / acc[..., 3:4])
        rmgr.OnDestroy()
        for lib in libs:
            for params in grid:
                row = {"quality": name, "size": f"{W}x{H}", "reference_spp": 1024, "frames": "8..16",
                       "lib": os.path.basename(lib), "params": params}
                row.update(quality_row(lib, make, sc, refs, params))
                print(json.dumps(row), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="small frames (a rehearsal, not a measurement)")
    ap.add_argument("--min-seconds", type=float, default=0.3)
    ap.add_argument("--ab", default="", help="comma-separated other librt_b200.so builds for the quality rows")
    ap.add_argument("--sweep", action="store_true", help="quality rows over a parameter grid")
    ap.add_argument("--quality-only", action="store_true")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("temporal_denoise_bench: no CUDA device")
    print(json.dumps({"card": card(), "lib": os.path.relpath(CUDA_LIB, REPO),
                      "defaults": [capi.TEMPORAL_ITERATIONS, capi.TEMPORAL_SIGMA_LUMINANCE, capi.TEMPORAL_SIGMA_NORMAL,
                                   capi.TEMPORAL_SIGMA_DEPTH, capi.TEMPORAL_ALPHA]}), flush=True)
    hd, uhd = ((192, 108), (384, 216)) if args.quick else ((1920, 1080), (3840, 2160))
    if not args.quality_only:
        timing_rows(args, torch, hd, uhd)
    default = (capi.TEMPORAL_ITERATIONS, capi.TEMPORAL_SIGMA_LUMINANCE, capi.TEMPORAL_SIGMA_NORMAL, capi.TEMPORAL_SIGMA_DEPTH,
               capi.TEMPORAL_ALPHA)
    grid = [default]
    if args.sweep:
        grid += [(5, sl, 1.0, sz, al) for sl in (2.0, 4.0, 8.0) for sz in (0.1, 1.0) for al in (0.05, 0.1, 0.2)
                 if (5, sl, 1.0, sz, al) != default]
    libs = [CUDA_LIB] + [os.path.abspath(p) for p in args.ab.split(",") if p]
    quality_rows((64, 36) if args.quick else (320, 180), libs, grid)
    return 0


if __name__ == "__main__":
    sys.exit(main())
