#!/usr/bin/env python
"""Throughput of rtTraceOcclusion (any-hit queries on segments) on the GPU, against rtTraceRays (closest hit) on the same rays.

    python tools/occlusion_bench.py [--quick] [--min-seconds 0.35] [--check 2000]

Per workload, three arms alternated three times (medians and min..max spread reported):
  occlusion  rtTraceOcclusionDevice on torch CUDA tensors, CUDA events around the call on the context's stream: Msegments/s
  closest    rtTraceRaysDevice on the same origins and directions, timed the same way: what a caller pays without the occlusion query
             (closest hit past the end of the segment, 48 bytes out per ray, dst compared afterwards)
  host       rtTraceOcclusion on host arrays, wall clock around the synchronising call: end to end, 28 + 1 bytes per segment across PCIe
Each arm repeats its call until at least --min-seconds of work per repetition, after a warm-up call.  A counting run ("countStats" = 1)
on the same batch reports box + triangle tests per ray for both queries.  A row is printed only if a seeded sample of --check of its
answers equals the oracle's; otherwise the tool stops with an error.  Prints the card name and power limit read in the same run.

Workloads:
  shadow         knot room: from the pick-hit points of every pixel (pulled back 1e-4 along the incoming ray) to a random point of the
                 ceiling light (model 2), tMax = 1 - 2^-10
  ao             knot room: from the same points, unit directions in the hemisphere the incoming ray came from, tMax = 0.25
  line of sight  between random points of the scene's box, tMax = 1 - 2^-10: knot room, the 871k-triangle cluster, 500 instances (TLAS),
                 10,000 spheres (the sphere accelerator)
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
from conftest import CUDA_LIB, ORACLE_LIB                        # noqa: E402
import ray_tracing_b200 as rt                                     # noqa: E402
from ray_tracing_b200 import capi, scenes                         # noqa: E402
from test_gpu_trace_rays import pick_rays_np                      # noqa: E402
from trace_rays_bench import card, scene_box, timed               # noqa: E402

T_SEGMENT = np.float32(1.0 - 2.0 ** -10)     # a segment to a point stops just short of it


def hit_points(sc, W, H):
    """The knot room's pick hits: points on surfaces, the incoming directions and the normals facing them."""
    xs, ys = np.meshgrid(np.arange(W), np.arange(H))
    rays = pick_rays_np(sc, W, H, xs.ravel(), ys.ravel())
    mgr = rt.RayComputeManager(CUDA_LIB)
    scenes.apply(sc, mgr)
    mgr.OnEnable()
    hits = mgr.context.trace_rays(rays)
    mgr.OnDestroy()
    ok = hits["kind"] != capi.RT_HIT_NONE
    d_in = rays["dir"][ok].astype(np.float64)
    nrm = hits["normal"][ok].astype(np.float64)
    nrm *= -np.sign(np.sum(nrm * d_in, axis=1, keepdims=True) + 1e-30)      # toward the side the ray came from
    return hits["pos"][ok].astype(np.float64) - 1e-4 * d_in, nrm


def shadow_segments(pts, n, rng):
    i = rng.randint(len(pts), size=n)
    light = np.stack([rng.uniform(-0.8, 0.8, n), np.full(n, 3.98), rng.uniform(-0.4, 1.2, n)], axis=1)     # knot_room's quad, model 2
    return capi.make_segments(pts[i], light - pts[i], T_SEGMENT)


def ao_segments(pts, nrm, n, rng, length=0.25):
    i = rng.randint(len(pts), size=n)
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    d *= np.sign(np.sum(d * nrm[i], axis=1, keepdims=True) + 1e-30)
    return capi.make_segments(pts[i], d, np.float32(length))


def sight_segments(sc, n, rng):
    lo, hi = scene_box(sc)
    a, b = rng.uniform(lo, hi, (n, 3)), rng.uniform(lo, hi, (n, 3))
    return capi.make_segments(a, b - a, T_SEGMENT)


def run_row(name, sc, segs, args, torch):
    mgr = rt.RayComputeManager(CUDA_LIB)
    scenes.apply(sc, mgr)
    mgr.OnEnable()
    ctx = mgr.context
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    n = len(segs)
    rays = capi.make_rays(segs["origin"], segs["dir"])
    d_segs = torch.from_numpy(segs.view(np.uint8)).to("cuda")
    d_occ = torch.empty(n, dtype=torch.uint8, device="cuda")
    d_rays = torch.from_numpy(rays.view(np.uint8)).to("cuda")
    d_hits = torch.empty(n * 48, dtype=torch.uint8, device="cuda")

    def kernel_clock(fn):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        fn()
        b.record(stream)
        b.synchronize()
        return a.elapsed_time(b) / 1e3

    def wall_clock(fn):
        t = time.perf_counter()
        fn()
        return time.perf_counter() - t

    host_occ = {}

    def host_call():
        host_occ["o"] = ctx.trace_occlusion(segs)

    def occlusion():
        ctx.trace_occlusion_device(d_segs.data_ptr(), d_occ.data_ptr(), n)

    def closest():
        ctx.trace_rays_device(d_rays.data_ptr(), d_hits.data_ptr(), n)

    samples = {"occlusion": [], "closest": [], "host": []}
    for _ in range(3):
        samples["occlusion"].append(n / timed(occlusion, args.min_seconds, kernel_clock) / 1e6)
        samples["closest"].append(n / timed(closest, args.min_seconds, kernel_clock) / 1e6)
        samples["host"].append(n / timed(host_call, args.min_seconds, wall_clock) / 1e6)
    torch.cuda.synchronize()
    dev_occ = d_occ.cpu().numpy().astype(bool)
    got = host_occ["o"]
    if not np.array_equal(dev_occ, got):
        sys.exit(f"occlusion_bench: {name}: device and host forms differ on {int(np.sum(dev_occ != got))} segments")
    hits = d_hits.cpu().numpy().view(capi.RAY_HIT_DTYPE)
    if np.any(got & ~(hits["dst"] < segs["tMax"])):
        sys.exit(f"occlusion_bench: {name}: occluded segments whose closest hit is not below tMax")

    work = {}
    ctx.set_option("countStats", 1)
    for arm, fn in (("occlusion", occlusion), ("closest", closest)):
        ctx.reset_stats()
        fn()
        ctx.synchronize()
        st = ctx.stats()
        work[arm] = (st["boxTests"] + st["triTests"]) / max(st["rays"], 1)
    ctx.set_option("countStats", 0)
    ctx.set_stream(0)
    mgr.OnDestroy()

    sub = np.random.RandomState(1).choice(n, min(args.check, n), replace=False)
    ref = rt.RayComputeManager(ORACLE_LIB)
    scenes.apply(sc, ref)
    ref.OnEnable()
    want = ref.context.trace_occlusion(segs[sub])
    ref.OnDestroy()
    if not np.array_equal(got[sub], want):
        sys.exit(f"occlusion_bench: {name}: {int(np.sum(got[sub] != want))} of {len(sub)} sampled answers differ from the oracle")
    row = {"workload": name, "segments": n, "occluded_share": round(float(got.mean()), 3)}
    for k, v in samples.items():
        row[k + "_msegs_s"] = round(float(np.median(v)), 1)
        row[k + "_spread"] = [round(float(min(v)), 1), round(float(max(v)), 1)]
    row["occlusion_over_closest"] = round(row["occlusion_msegs_s"] / row["closest_msegs_s"], 2)
    for k, v in work.items():
        row[k + "_box_tri_tests_per_ray"] = round(float(v), 1)
    print(json.dumps(row), flush=True)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="small batches (a rehearsal, not a measurement)")
    ap.add_argument("--min-seconds", type=float, default=0.35)
    ap.add_argument("--check", type=int, default=2000)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("occlusion_bench: no CUDA device")
    print(json.dumps({"card": card(), "lib": os.path.relpath(CUDA_LIB, REPO)}), flush=True)
    rng = np.random.RandomState(7)
    big = 1 << 16 if args.quick else 4 << 20
    W, H = (192, 108) if args.quick else (1920, 1080)
    knot = scenes.knot_room(W, H, 8, 1)
    pts, nrm = hit_points(knot, W, H)
    run_row("knot_room shadow to the ceiling light", knot, shadow_segments(pts, big, rng), args, torch)
    run_row("knot_room ao 0.25", knot, ao_segments(pts, nrm, big, rng), args, torch)
    for name, sc in (("knot_room", knot), ("knot_cluster 871k", scenes.knot_cluster(W, H, 8, 1)),
                     ("instances500", scenes.instanced_knots(W, H, 8, 1, instances=500)),
                     ("spheres10000", scenes.random_soup(W, H, 8, 1, triangles=60, spheres=10000))):
        run_row(f"{name} line of sight", sc, sight_segments(sc, big, rng), args, torch)
    return 0


if __name__ == "__main__":
    sys.exit(main())
