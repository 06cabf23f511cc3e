#!/usr/bin/env python
"""Throughput of rtTraceRays (closest-hit queries) on the GPU, with the path kernel's ray-segment rate on the same scene for context.

    python tools/trace_rays_bench.py [--quick] [--min-seconds 0.35] [--check 2000]

Per workload, three arms alternated three times (medians and min..max spread reported):
  kernel  rtTraceRaysDevice on torch CUDA tensors, CUDA events around the call on the context's stream: Mrays/s of the query kernel
  host    rtTraceRays on host arrays, wall clock around the synchronising call: end to end, 24 + 48 bytes per ray across PCIe
  path    one 1-spp frame of the scene (RayComputeManager.RenderFrame): RtStats.rays / kernelMs, the camera kernels' segment rate
Each arm repeats its call until at least --min-seconds of work per repetition, after a warm-up call.  A row is printed only if a seeded
sample of --check of its hits equals the oracle's bit for bit (NaN canonicalised); otherwise the tool stops with an error.
Prints the card name and power limit read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tests"))
from conftest import CUDA_LIB, ORACLE_LIB                        # noqa: E402
import ray_tracing_b200 as rt                                     # noqa: E402
from ray_tracing_b200 import capi, scenes                         # noqa: E402
from test_gpu_trace_rays import assert_hits_equal, pick_rays_np   # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return out.strip().splitlines()[0]
    except Exception as e:                      # noqa: BLE001
        return f"unknown ({e})"


def scene_box(sc):
    pts = [np.asarray(sc.spheres["centre"], dtype=np.float64).reshape(-1, 3)] if len(sc.spheres) else []
    for m in sc.models:
        v = sc.meshes[m.mesh].vertices.astype(np.float64)
        pts.append(v @ np.asarray(m.local_to_world)[:3, :3].T + np.asarray(m.local_to_world)[:3, 3])
    p = np.concatenate(pts)
    return p.min(axis=0), p.max(axis=0)


def random_rays(sc, n, rng, far=False):
    lo, hi = scene_box(sc)
    if far:
        d = rng.normal(size=(n, 3))
        o = (lo + hi) / 2 + d / np.linalg.norm(d, axis=1, keepdims=True) * 1e5
        return capi.make_rays(o, rng.uniform(lo, hi, (n, 3)) - o)
    return capi.make_rays(rng.uniform(lo, hi, (n, 3)), rng.normal(size=(n, 3)))


def timed(fn, min_seconds, clock):
    fn()                                         # warm-up
    reps, total = 0, 0.0
    while total < min_seconds:
        total += clock(fn)
        reps += 1
    return total / reps


def run_row(name, sc, rays, args, torch):
    mgr = rt.RayComputeManager(CUDA_LIB)
    scenes.apply(sc, mgr)
    mgr.OnEnable()
    ctx = mgr.context
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    d_rays = torch.from_numpy(rays.view(np.uint8)).to("cuda")
    d_hits = torch.empty(len(rays) * 48, dtype=torch.uint8, device="cuda")
    n = len(rays)

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

    host_hits = {}

    def host_call():
        host_hits["h"] = ctx.trace_rays(rays)

    def path_frame():
        ctx.reset_stats()
        mgr.RenderFrame()
        st = ctx.stats()
        return st["rays"] / (st["kernelMs"] / 1e3)

    samples = {"kernel": [], "host": [], "path": []}
    for _ in range(3):
        samples["kernel"].append(n / timed(lambda: ctx.trace_rays_device(d_rays.data_ptr(), d_hits.data_ptr(), n), args.min_seconds, kernel_clock) / 1e6)
        samples["host"].append(n / timed(host_call, args.min_seconds, wall_clock) / 1e6)
        rates, t0 = [], time.perf_counter()
        path_frame()
        while time.perf_counter() - t0 < args.min_seconds:
            rates.append(path_frame())
        samples["path"].append(float(np.median(rates)) / 1e6)
    torch.cuda.synchronize()
    dev_hits = d_hits.cpu().numpy().view(capi.RAY_HIT_DTYPE)
    assert_hits_equal(dev_hits, host_hits["h"], f"{name}: device vs host form")
    ctx.set_stream(0)
    mgr.OnDestroy()
    sub = np.random.RandomState(1).choice(n, min(args.check, n), replace=False)
    ref = rt.RayComputeManager(ORACLE_LIB)
    scenes.apply(sc, ref)
    ref.OnEnable()
    assert_hits_equal(host_hits["h"][sub], ref.context.trace_rays(rays[sub]), f"{name}: sampled hits vs the oracle")
    ref.OnDestroy()
    hit_share = float(np.mean(host_hits["h"]["kind"] != capi.RT_HIT_NONE))
    row = {"workload": name, "rays": n, "hit_share": round(hit_share, 3)}
    for k, v in samples.items():
        row[k + "_mrays_s"] = round(float(np.median(v)), 1)
        row[k + "_spread"] = [round(float(min(v)), 1), round(float(max(v)), 1)]
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
        sys.exit("trace_rays_bench: no CUDA device")
    print(json.dumps({"card": card(), "lib": os.path.relpath(CUDA_LIB, REPO)}), flush=True)
    rng = np.random.RandomState(7)
    big = 1 << 16 if args.quick else 8 << 20
    W, H = (192, 108) if args.quick else (1920, 1080)
    knot = scenes.knot_room(W, H, 8, 1)
    xs, ys = np.meshgrid(np.arange(W), np.arange(H))
    rows = [run_row(f"knot_room pick rays {W}x{H}", knot, pick_rays_np(knot, W, H, xs.ravel(), ys.ravel()), args, torch)]
    for name, sc in (("knot_room", knot), ("knot_cluster 871k", scenes.knot_cluster(W, H, 8, 1)),
                     ("instances500", scenes.instanced_knots(W, H, 8, 1, instances=500)),
                     ("spheres10000", scenes.random_soup(W, H, 8, 1, triangles=60, spheres=10000))):
        rows.append(run_row(f"{name} random in-scene", sc, random_rays(sc, big, rng), args, torch))
    rows.append(run_row("knot_room far origins (linear fallback)", knot, random_rays(knot, big // 8, rng, far=True), args, torch))
    return 0


if __name__ == "__main__":
    sys.exit(main())
