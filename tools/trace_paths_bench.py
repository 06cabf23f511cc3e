#!/usr/bin/env python
"""Throughput of rtTracePaths (the path tracer's radiance along caller rays) on the GPU, against the camera kernels on the same segments.

    python tools/trace_paths_bench.py [--quick] [--min-seconds 0.5] [--out DIR]

Per workload, the camera ray and post-jitter RNG state of every pixel come from the oracle's orCameraSample (HL:565-572), so the
query traces exactly the paths a 1-spp rtDispatch of the same frame traces.  Arms, alternated three times (medians and min..max spread):
  paths      rtTracePathsDevice(samples = 1) on torch CUDA tensors, CUDA events around the call on the context's stream
  kernel1    rtDispatch of the frame with "kernel" = 1 (the wavefront kernel), timed by RtStats.kernelMs
  default    rtDispatch with the automatic kernel choice (the pooled kernel on mesh scenes), timed by RtStats.kernelMs
Rates are Msegments/s: RtStats.rays (one per CalculateRayCollision) over kernel time; the tool stops with an error unless the three
arms count the same segments and the query's rgb equals the dispatch's FrameRender bit for bit for both camera kernels.  Each arm
repeats its call until at least --min-seconds of work per repetition, after a warm-up call.  Prints the card name and power limit read
in the same run.

Workloads: Cornell spheres at 1080p; the knot room with a glass knot at 1080p; the 871k-triangle cluster at 4K; 500 instances (TLAS)
and 10,000 spheres (the sphere accelerator) at 1080p.  Then, as a custom camera, a 360-degree equirectangular panorama of the knot
room from the middle of the room at 64 samples per pixel, written to DIR/knot_room_panorama.png.
"""
import argparse
import json
import os
import sys
import tempfile

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tests"))
sys.path.insert(0, os.path.join(REPO, "tools"))
from conftest import CUDA_LIB, ORACLE_LIB                        # noqa: E402
import ray_tracing_b200 as rt                                     # noqa: E402
from ray_tracing_b200 import capi, scenes                         # noqa: E402
from test_gpu_trace_paths import camera_samples                   # noqa: E402
from trace_rays_bench import card, scene_box, timed               # noqa: E402


def open_mgr(lib, sc):
    mgr = rt.RayComputeManager(lib)
    scenes.apply(sc, mgr)
    mgr.OnEnable()                   # uploads the first frame's uniforms (Frame, camera, ...) without rendering
    return mgr


def run_row(name, sc, args, torch):
    W, H = sc.width, sc.height
    sc.settings = dict(sc.settings, numRaysPerPixel=1)
    ref = open_mgr(ORACLE_LIB, sc)
    rays = camera_samples(ref.context, W, H)
    ref.OnDestroy()
    n = len(rays)

    mgr = open_mgr(CUDA_LIB, sc)
    ctx = mgr.context
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    d_rays = torch.from_numpy(rays.view(np.uint8)).to("cuda")
    d_out = torch.empty(n * 16, dtype=torch.uint8, device="cuda")

    def event_clock(fn):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        fn()
        b.record(stream)
        b.synchronize()
        return a.elapsed_time(b) / 1e3

    def kernel_ms_clock(fn):
        ctx.synchronize()
        t0 = ctx.stats()["kernelMs"]
        fn()
        ctx.synchronize()
        return (ctx.stats()["kernelMs"] - t0) / 1e3

    def paths():
        ctx.trace_paths_device(d_rays.data_ptr(), d_out.data_ptr(), n, 1)

    def camera(kernel):
        def fn():
            ctx.set_option("kernel", kernel)
            ctx.dispatch_full()          # the frame OnEnable set up: the same Frame, so the same paths every time
        return fn

    arms = {"paths": (paths, event_clock), "kernel1": (camera(1), kernel_ms_clock), "default": (camera(-1), kernel_ms_clock)}
    # segments per arm and the bitwise check, once before timing
    segments = {}
    for arm, (fn, _) in arms.items():
        ctx.synchronize()
        ctx.reset_stats()
        fn()
        ctx.synchronize()
        segments[arm] = ctx.stats()["rays"]
        if arm != "paths":
            frame = ctx.readback("FrameRender")[..., :3].reshape(-1, 3)
            got = d_out.cpu().numpy().view(capi.PATH_RADIANCE_DTYPE)["rgb"]
            a, b = got.view(np.uint32), frame.view(np.uint32)
            bad = np.flatnonzero(np.any((a != b) & ~(np.isnan(got) & np.isnan(frame)), axis=1))
            if len(bad):
                sys.exit(f"trace_paths_bench: {name}: rtTracePaths differs from the {arm} dispatch's FrameRender on {len(bad)} pixels, "
                         f"first {bad[0]}: {got[bad[0]]} vs {frame[bad[0]]}")
    if len(set(segments.values())) != 1:
        sys.exit(f"trace_paths_bench: {name}: RtStats.rays differs between the arms: {segments}")
    seg = segments["paths"]

    rates = {k: [] for k in arms}
    for _ in range(3):
        for arm, (fn, clock) in arms.items():
            rates[arm].append(seg / timed(fn, args.min_seconds, clock) / 1e6)
    ctx.set_stream(0)
    mgr.OnDestroy()
    row = {"workload": name, "pixels": n, "segments": int(seg), "segments_per_path": round(seg / n, 2)}
    for k, v in rates.items():
        row[k + "_msegs_s"] = round(float(np.median(v)), 1)
        row[k + "_spread"] = [round(float(min(v)), 1), round(float(max(v)), 1)]
    row["paths_over_kernel1"] = round(row["paths_msegs_s"] / row["kernel1_msegs_s"], 2)
    row["paths_over_default"] = round(row["paths_msegs_s"] / row["default_msegs_s"], 2)
    print(json.dumps(row), flush=True)
    return row


def panorama(args, torch, W, H, samples=64):
    """A 360-degree equirectangular view of the knot room from the middle of the room, 1.0 above the floor: a camera rtDispatch
    cannot express, through rtTracePathsDevice."""
    sc = scenes.knot_room(W, H, 8, 1, glass=True)
    lo, hi = scene_box(sc)
    centre = np.array([(lo[0] + hi[0]) / 2, 1.0, (lo[2] + hi[2]) / 2])
    v, u = np.meshgrid((np.arange(H) + 0.5) / H, (np.arange(W) + 0.5) / W, indexing="ij")     # row 0 = top of the image
    theta, phi = np.pi * v, 2.0 * np.pi * u
    d = np.stack([np.sin(theta) * np.sin(phi), np.cos(theta), -np.sin(theta) * np.cos(phi)], axis=-1).reshape(-1, 3)
    states = (np.arange(W * H, dtype=np.uint64) * 2654435761 + 12345).astype(np.uint32)
    rays = capi.make_path_rays(np.broadcast_to(centre, d.shape), d, states)
    mgr = open_mgr(CUDA_LIB, sc)
    d_rays = torch.from_numpy(rays.view(np.uint8)).to("cuda")
    d_out = torch.empty(len(rays) * 16, dtype=torch.uint8, device="cuda")
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ctx = mgr.context
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)           # the events bracket the call on the stream it runs on
    ctx.reset_stats()
    a.record(stream)
    ctx.trace_paths_device(d_rays.data_ptr(), d_out.data_ptr(), len(rays), samples)
    b.record(stream)
    b.synchronize()
    seg = ctx.stats()["rays"]
    ctx.set_stream(0)
    mgr.OnDestroy()
    rgb = d_out.cpu().numpy().view(capi.PATH_RADIANCE_DTYPE)["rgb"].reshape(H, W, 3)
    x = np.clip(np.nan_to_num(rgb, nan=0.0), 0.0, 1.0)
    srgb = np.where(x <= 0.0031308, 12.92 * x, 1.055 * x ** (1 / 2.4) - 0.055)
    os.makedirs(args.out, exist_ok=True)
    path = os.path.join(args.out, "knot_room_panorama.png")
    rt.write_png(path, (srgb * 255.0 + 0.5).astype(np.uint8))
    print(json.dumps({"panorama": os.path.relpath(path), "size": [W, H], "samples": samples, "origin": centre.round(3).tolist(),
                      "ms": round(a.elapsed_time(b), 1), "msegs_s": round(seg / (a.elapsed_time(b) / 1e3) / 1e6, 1)}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="small frames (a rehearsal, not a measurement)")
    ap.add_argument("--min-seconds", type=float, default=0.5)
    ap.add_argument("--out", default=None, help="directory for the panorama PNG (default: a new temporary directory)")
    args = ap.parse_args()
    args.out = args.out or tempfile.mkdtemp(prefix="trace_paths_bench_")
    import torch
    if not torch.cuda.is_available():
        sys.exit("trace_paths_bench: no CUDA device")
    print(json.dumps({"card": card(), "lib": os.path.relpath(CUDA_LIB, REPO)}), flush=True)
    hd, uhd = ((192, 108), (384, 216)) if args.quick else ((1920, 1080), (3840, 2160))
    for name, sc in (("cornell_spheres 1080p", scenes.cornell_spheres(*hd)),
                     ("knot_room glass 1080p", scenes.knot_room(*hd, 8, 1, glass=True)),
                     ("knot_cluster 871k 4K", scenes.knot_cluster(*uhd)),
                     ("instances500 1080p", scenes.instanced_knots(*hd, 8, 1, instances=500)),
                     ("spheres10000 1080p", scenes.random_soup(*hd, 8, 1, triangles=60, spheres=10000))):
        run_row(name, sc, args, torch)
    panorama(args, torch, *((256, 128) if args.quick else (2048, 1024)))
    return 0


if __name__ == "__main__":
    sys.exit(main())
