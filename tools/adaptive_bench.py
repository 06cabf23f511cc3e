#!/usr/bin/env python
"""Cost and quality of rtDispatchAdaptive (adaptive sampling) on the GPU.

    python tools/adaptive_bench.py [--quick] [--rounds 3] [--sweep] [--out DIR]

1. Overhead: an all-active adaptive call (minFrames = maxFrames = RT_ADAPTIVE_MAX_FRAMES: every covered pixel is below minFrames)
   against rtDispatch of the same frame, alternated call by call in the same rounds; host wall time per call until the render has
   finished (the adaptive call synchronises once before its launch, rtDispatch not at all) and the render launch's kernelMs.  1-spp
   1080p Cornell box and glass knot room frames, and bench.py's default workload (the knot room at 1080p, 256 spp per frame).
2. Selection: the three selection kernels (k_adaptive_flags, k_adaptive_scan, k_adaptive_scatter) at 1080p and 4K with every pixel
   active and with none active, timed with torch.profiler (CUDA activities, a run of its own), against the HBM bound of their
   algorithmic bytes: 16 B read per covered pixel, 4 B written per active pixel, the ballot words and block counts.
3. Time to quality: the glass knot room at 1080p, 1 spp per frame, against a 4096-frame rtDispatchFrames reference of an independent
   seed: relative MSE against elapsed GPU time (host wall time of the synchronised loop) for uniform frames and for adaptive frames
   with the capi defaults, and the factor between the uniform and adaptive errors at equal time.
4. --sweep: the capi defaults' grid (threshold x minFrames x maxFrames) at 320 x 180 on both scenes, uniform at an equal budget of
   traced pixel-frames, with this build and the RT_ADAPTIVE_EPSILON build variants of tools/build_variants.py if they are built.
Medians over --rounds rounds with min..max.  Prints the card name, power limit and max SM clock read in the same run.  Fails without a
GPU.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tests"))
sys.path.insert(0, os.path.join(REPO, "tools"))
from conftest import CUDA_LIB                                     # noqa: E402
import ray_tracing_b200 as rt                                     # noqa: E402
from ray_tracing_b200 import capi, scenes                         # noqa: E402
from trace_rays_bench import card                                 # noqa: E402

HBM_BYTES_PER_S = 3.35e12                 # H100 SXM data sheet
ALL = capi.ADAPTIVE_MAX_FRAMES_LIMIT


def open_scene(sc, lib=CUDA_LIB, spp=None, seed=None):
    mgr = rt.RayComputeManager(lib)
    scenes.apply(sc, mgr)
    if spp is not None:
        mgr.numRaysPerPixel = spp
    if seed is not None:
        mgr.renderSeed = seed
    mgr.OnEnable()
    return mgr, mgr.context


def rel_mse(x, ref):
    return float(np.mean((x[..., :3].astype(np.float64) - ref[..., :3]) ** 2 / (ref[..., :3].astype(np.float64) ** 2 + 0.01)))


def mean_image(a):
    w = a[..., 3:4]
    return np.where(w > 0, a / np.where(w > 0, w, 1), 0)


def stat(xs):
    return {"median": float(np.median(xs)), "min": float(np.min(xs)), "max": float(np.max(xs))}


def overhead_rows(args):
    rows = []
    cases = [("cornell 1080p 1 spp", scenes.cornell_spheres(1920, 1080, 8, 1), 24),
             ("knot room glass 1080p 1 spp", scenes.knot_room(1920, 1080, 8, 1, glass=True), 24),
             ("knot room 1080p 256 spp (bench.py default)", scenes.knot_room(1920, 1080, 8, 256), 3)]
    for name, sc, calls in cases:
        if args.quick:
            calls = max(2, calls // 4)
        mgr, ctx = open_scene(sc)
        frame = [1]

        def plain():
            ctx.set_int("Frame", frame[0]); frame[0] += 1
            ctx.dispatch_full()

        def adaptive():
            ctx.set_int("Frame", frame[0]); frame[0] += 1
            n = ctx.dispatch_adaptive(0.0, ALL, ALL)
            assert n == sc.width * sc.height

        for fn in (plain, adaptive):                 # warm-up: modules, scene repack, the moments' allocation
            fn(); ctx.synchronize()
        wall = {"rtDispatch": [], "rtDispatchAdaptive": []}
        kern = {"rtDispatch": [], "rtDispatchAdaptive": []}
        for _ in range(args.rounds):
            acc = {k: [0.0, 0.0] for k in wall}
            for _ in range(calls):
                for key, fn in (("rtDispatch", plain), ("rtDispatchAdaptive", adaptive)):
                    k0 = ctx.stats()["kernelMs"]
                    t0 = time.perf_counter()
                    fn()
                    ctx.synchronize()
                    acc[key][0] += (time.perf_counter() - t0) * 1e3
                    acc[key][1] += ctx.stats()["kernelMs"] - k0
            for key in wall:
                wall[key].append(acc[key][0] / calls)
                kern[key].append(acc[key][1] / calls)
        mgr.OnDestroy()
        row = {"case": name, "calls_per_round": calls,
               "wall_ms": {k: stat(v) for k, v in wall.items()}, "kernel_ms": {k: stat(v) for k, v in kern.items()},
               "overhead_ms_median": float(np.median(np.array(wall["rtDispatchAdaptive"]) - np.array(wall["rtDispatch"])))}
        print(json.dumps(row), flush=True)
        rows.append(row)
    return rows


def selection_rows(args, torch, out_dir):
    from torch.profiler import ProfilerActivity, profile
    rows = []
    for W, H in ((1920, 1080), (3840, 2160)):
        sc = scenes.cornell_spheres(W, H, 1, 1)
        mgr, ctx = open_scene(sc)
        # "all": every pixel below minFrames; "none": every pixel at maxFrames (after two frames with maxFrames = 2)
        ctx.set_int("Frame", 1); ctx.dispatch_adaptive(0.0, 2, 2)
        ctx.set_int("Frame", 2); ctx.dispatch_adaptive(0.0, 2, 2)
        ctx.synchronize()
        reps = 5 if args.quick else 20
        for label, call in (("all", lambda: ctx.dispatch_adaptive(0.0, ALL, ALL)), ("none", lambda: ctx.dispatch_adaptive(0.0, 2, 2))):
            call(); ctx.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(reps):
                    call()
                ctx.synchronize()
            times = {}
            for ev in prof.key_averages():
                if "k_adaptive_" in ev.key:
                    key = "flags" if "flags" in ev.key else "scan" if "scan" in ev.key else "scatter"
                    total_us = getattr(ev, "device_time_total", 0) or getattr(ev, "self_device_time_total", 0) or getattr(ev, "cuda_time_total", 0)
                    times[key] = [total_us / 1e3 / max(ev.count, 1)]
            if args.out:
                prof.export_chrome_trace(os.path.join(out_dir, f"adaptive_selection_{W}x{H}_{label}.json"))
            active = W * H if label == "all" else 0
            jobs = ((W + 7) // 8) * ((H + 3) // 4) * 32
            blocks = (jobs + 255) // 256
            nbytes = 16 * W * H + 4 * active + 4 * (jobs // 32) * 2 + 4 * blocks * 3
            total_ms = sum(np.median(v) for v in times.values()) if times else float("nan")
            row = {"size": f"{W}x{H}", "active": label, "kernels_ms_median": {k: float(np.median(v)) for k, v in times.items()},
                   "selection_ms": float(total_ms), "algorithmic_bytes": nbytes,
                   "hbm_bound_ms": nbytes / HBM_BYTES_PER_S * 1e3, "share_of_hbm_bound": (nbytes / HBM_BYTES_PER_S * 1e3) / total_ms}
            print(json.dumps(row), flush=True)
            rows.append(row)
        mgr.OnDestroy()
    return rows


def time_to_quality(args):
    W, H = (960, 540) if args.quick else (1920, 1080)
    sc = scenes.knot_room(W, H, 8, 1, glass=True)
    mgr, ctx = open_scene(sc, seed=977)
    ref_frames = 256 if args.quick else 4096
    t0 = time.perf_counter()
    ctx.dispatch_frames(ref_frames)
    ctx.synchronize()
    ref = mean_image(mgr.accumulatedResult)
    print(json.dumps({"reference_frames": ref_frames, "reference_s": time.perf_counter() - t0}), flush=True)
    mgr.OnDestroy()
    checkpoints = (4, 8, 16, 32, 64, 128, 256)
    out = {}
    wm, wc = open_scene(sc)                      # warm-up on a context of its own: modules, both kernels' first launches
    wc.dispatch_full(); wc.dispatch_adaptive(); wc.synchronize()
    wm.OnDestroy()
    for arm in ("uniform", "adaptive"):
        mgr, ctx = open_scene(sc)
        curve, elapsed, frame, traced = [], 0.0, 1, 0
        while frame <= checkpoints[-1]:
            t0 = time.perf_counter()
            ctx.set_int("Frame", frame)
            if arm == "uniform":
                ctx.dispatch_full(); n = W * H
            else:
                n = ctx.dispatch_adaptive()
            ctx.synchronize()
            elapsed += time.perf_counter() - t0
            traced += n
            if frame in checkpoints or n == 0:
                curve.append({"frames": frame, "gpu_s": elapsed, "pixel_frames_per_pixel": traced / (W * H),
                              "rel_mse": rel_mse(mean_image(mgr.accumulatedResult), ref)})
                print(json.dumps(dict(arm=arm, **curve[-1])), flush=True)
            if n == 0:
                break
            frame += 1
        out[arm] = curve
        mgr.OnDestroy()
    # the uniform error at the adaptive arm's end time (log-log interpolation on the uniform curve)
    end = out["adaptive"][-1]
    u = out["uniform"]
    ts, es = np.log([c["gpu_s"] for c in u]), np.log([c["rel_mse"] for c in u])
    at = float(np.exp(np.interp(np.log(end["gpu_s"]), ts, es)))
    res = {"size": f"{W}x{H}", "curves": out, "adaptive_end": end, "uniform_at_equal_time": at, "factor_at_equal_time": at / end["rel_mse"]}
    print(json.dumps({k: v for k, v in res.items() if k != "curves"}), flush=True)
    return res


def sweep(args):
    from build_variants import path as variant_path
    libs = [("default", CUDA_LIB)] + [(n, variant_path(n)) for n in ("adaptive_eps4", "adaptive_eps12") if os.path.exists(variant_path(n))]
    W, H = 320, 180
    rows = []
    for name, sc in (("cornell", scenes.cornell_spheres(W, H, 4, 1)), ("knot_room_glass", scenes.knot_room(W, H, 8, 1, glass=True))):
        mgr, ctx = open_scene(sc, seed=977)
        ctx.dispatch_frames(1024)
        ref = mean_image(mgr.accumulatedResult)
        mgr.OnDestroy()
        uni = {}

        def uniform(frames):
            if frames not in uni:
                m, c = open_scene(sc)
                c.dispatch_frames(frames) if frames > 1 else c.dispatch_full()
                uni[frames] = rel_mse(mean_image(m.accumulatedResult), ref)
                m.OnDestroy()
            return uni[frames]
        for lname, lib in libs:
            for mx in (32, 64, 128):
                for mn in (4, 8, 16):
                    for thr in (0.1, 0.2, 0.3, 0.5):
                        m, c = open_scene(sc, lib=lib)
                        used, f = 0, 1
                        while True:
                            c.set_int("Frame", f); f += 1
                            n = c.dispatch_adaptive(thr, mn, mx)
                            used += n
                            if n == 0:
                                break
                        a = rel_mse(mean_image(m.accumulatedResult), ref)
                        m.OnDestroy()
                        k = used / (W * H)
                        lo, hi = max(1, int(np.floor(k))), int(np.ceil(k))
                        u = uniform(lo) + (uniform(hi) - uniform(lo)) * (k - lo) if hi > lo else uniform(hi)
                        row = {"scene": name, "build": lname, "threshold": thr, "minFrames": mn, "maxFrames": mx,
                               "frames_per_pixel": k, "adaptive": a, "uniform": u, "factor": u / a}
                        print(json.dumps(row), flush=True)
                        rows.append(row)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--sweep", action="store_true")
    ap.add_argument("--out", default="")
    ap.add_argument("--skip", default="", help="comma-separated parts to skip: overhead,selection,quality")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("adaptive_bench: no CUDA device")
    info = {"card": card(), "torch_device": torch.cuda.get_device_name(0)}
    print(json.dumps(info), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
    skip = set(filter(None, args.skip.split(",")))
    res = {"card": info}
    if "overhead" not in skip:
        res["overhead"] = overhead_rows(args)
    if "selection" not in skip:
        res["selection"] = selection_rows(args, torch, args.out)
    if "quality" not in skip:
        res["time_to_quality"] = time_to_quality(args)
    if args.sweep:
        res["sweep"] = sweep(args)
    res["card_after"] = card()
    if args.out:
        with open(os.path.join(args.out, "adaptive_bench.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
