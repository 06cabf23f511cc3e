#!/usr/bin/env python
"""Cost of rtDispatchFeatures (first-hit feature images for denoisers) on the GPU, against the same closest hits through rtTraceRays
and against the 1-spp frame the features belong to.

    python tools/features_bench.py [--quick] [--min-seconds 0.5]

Per workload, three arms alternated three times after a warm-up call, each repetition at least --min-seconds of work (medians and
min..max spread reported, in ms per image):
  features   rtDispatchFeatures over the whole image, accumulating, CUDA events around the call on the context's stream: no ray read,
             32 bytes written per pixel and two 16-byte read-modify-writes on a hit
  closest    rtTraceRaysDevice on the rays rtCameraRaysDevice wrote, timed the same way: the same closest hits, 24 bytes read and
             48 written per ray
  frame      rtDispatch of the same frame at 1 sample per pixel with the automatic kernel, timed by RtStats.kernelMs
A row is printed only if the features' dst, normal and object equal the closest arm's hits on every pixel; otherwise the tool stops
with an error.  Prints the card name, power limit and max SM clock read in the same run.  Fails without a GPU.
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


def run_row(name, sc, args, torch):
    W, H = sc.width, sc.height
    n = W * H
    sc.settings = dict(sc.settings, numRaysPerPixel=1)
    mgr = rt.RayComputeManager(CUDA_LIB)
    scenes.apply(sc, mgr)
    mgr.OnEnable()                   # uploads the first frame's uniforms (Frame, camera, ...) without rendering
    ctx = mgr.context
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    d_rays = torch.empty(n * 28, dtype=torch.uint8, device="cuda")
    d_hits = torch.empty(n * 48, dtype=torch.uint8, device="cuda")
    ctx.camera_rays_device(d_rays.data_ptr(), n * 28)
    # rtTraceRays reads 24-byte RtRay records: the first 24 bytes of every 28-byte RtPathRay, packed
    d_rays24 = d_rays.view(n, 28)[:, :24].contiguous()

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

    def features():
        ctx.dispatch_features()

    def closest():
        ctx.trace_rays_device(d_rays24.data_ptr(), d_hits.data_ptr(), n)

    def frame():
        ctx.dispatch_full()          # the frame OnEnable set up: the same Frame, so the same paths every time

    arms = {"features": (features, event_clock), "closest": (closest, event_clock), "frame": (frame, kernel_ms_clock)}
    segments = {}
    for arm, (fn, _) in arms.items():
        ctx.synchronize()
        ctx.reset_stats()
        fn()
        ctx.synchronize()
        segments[arm] = ctx.stats()["rays"]
    feat = ctx.readback("FeatureFrame").reshape(-1)
    hits = d_hits.cpu().numpy().view(capi.RAY_HIT_DTYPE)
    obj = np.where(hits["kind"] == capi.RT_HIT_SPHERE, -2 - hits["index"], hits["index"])
    same = (feat["dst"].view(np.uint32) == hits["dst"].view(np.uint32)) & (obj == feat["object"]) & \
           np.all((feat["normal"].view(np.uint32) == hits["normal"].view(np.uint32)) | (np.isnan(feat["normal"]) & np.isnan(hits["normal"])), axis=1)
    if not same.all() or segments["features"] != n or segments["closest"] != n:
        bad = np.flatnonzero(~same)
        sys.exit(f"features_bench: {name}: FeatureFrame differs from rtTraceRays on {len(bad)} pixels"
                 + (f", first {bad[0]}: {feat[bad[0]]} vs {hits[bad[0]]}" if len(bad) else f"; rays counted: {segments}"))

    ms = {k: [] for k in arms}
    for _ in range(3):
        for arm, (fn, clock) in arms.items():
            ms[arm].append(timed(fn, args.min_seconds, clock) * 1e3)
    ctx.set_stream(0)
    mgr.OnDestroy()
    row = {"workload": name, "pixels": n, "hit_share": round(float((feat["object"] != -1).mean()), 3),
           "segments_per_path": round(segments["frame"] / n, 2)}
    for k, v in ms.items():
        row[k + "_ms"] = round(float(np.median(v)), 4)
        row[k + "_spread"] = [round(float(min(v)), 4), round(float(max(v)), 4)]
    row["features_over_closest"] = round(row["features_ms"] / row["closest_ms"], 2)
    row["features_over_frame"] = round(row["features_ms"] / row["frame_ms"], 3)
    row["one_over_segments_per_path"] = round(n / segments["frame"], 3)
    print(json.dumps(row), flush=True)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="small frames (a rehearsal, not a measurement)")
    ap.add_argument("--min-seconds", type=float, default=0.5)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("features_bench: no CUDA device")
    print(json.dumps({"card": card(), "lib": os.path.relpath(CUDA_LIB, REPO)}), flush=True)
    hd, uhd = ((192, 108), (384, 216)) if args.quick else ((1920, 1080), (3840, 2160))
    for name, sc in (("cornell_spheres 1080p", scenes.cornell_spheres(*hd)),
                     ("knot_room glass 1080p", scenes.knot_room(*hd, 8, 1, glass=True)),
                     ("knot_cluster 871k 4K", scenes.knot_cluster(*uhd)),
                     ("instances500 1080p", scenes.instanced_knots(*hd, 8, 1, instances=500)),
                     ("spheres10000 1080p", scenes.random_soup(*hd, 8, 1, triangles=60, spheres=10000))):
        run_row(name, sc, args, torch)
    return 0


if __name__ == "__main__":
    sys.exit(main())
