#!/usr/bin/env python
"""Throughput of rtBakeLightmap (lightmaps: per surface texel the mean of S paths over the cosine-weighted hemisphere of its normal)
against the route before it, rtTracePaths on materialised per-sample rays.

    python tools/lightmap_bench.py [--quick] [--min-seconds 0.5]

Arms, alternated three times per workload (medians, min..max spread):
  bake    rtBakeLightmapDevice(points, n, S) on torch CUDA tensors; CUDA events around the call on the context's stream
  paths   rtTracePathsDevice(samples = 1) on the n * S rays of orLightmapRays (each sample's origin, direction and starting state, built
          once outside the timed window: 28 bytes per sample, plus 16 of radiance), then the mean in torch with non-finite samples
          zeroed; CUDA events around both.  The same result as the bake, up to the order of the sums
Msegments/s is RtStats.rays (one per CalculateRayCollision) over the call's time; texels/s is n over it.  The tool stops with an error
unless both arms count the same segments, and unless the bake equals, bit for bit, the header's sums (numpy, binary32) of the paths
arm's radiances for a subset of texels.  Prints the card name and power limit read in the same run.

Workloads, all at S = 256 (--quick: S = 64 and at most 4,096 texels): the vertex texels of the knot room's knot (43,560), a 64 x 64
grid of texels on each of the five walls of the same Cornell-style room (20,480), and every 13th vertex of the 871k-triangle cluster's
first model (33,508).
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
from conftest import CUDA_LIB, ORACLE_LIB                        # noqa: E402
import ray_tracing_b200 as rt                                     # noqa: E402
from ray_tracing_b200 import capi, manager, scenes                # noqa: E402
from test_gpu_cubemaps import mean32                              # noqa: E402
from test_gpu_lightmaps import lightmap_rays                      # noqa: E402
from trace_rays_bench import card                                 # noqa: E402


def open_mgr(lib, sc):
    mgr = rt.RayComputeManager(lib)
    scenes.apply(sc, mgr)
    mgr.OnEnable()
    return mgr


def model_vertices(sc, model, step=1):
    m = sc.models[model]
    mesh = sc.meshes[m.mesh]
    return manager.vertex_texels(mesh.vertices, mesh.normals, m.local_to_world)[::step]


def wall_grid(sc, side=64):
    """side x side texel centres on each quad of the room mesh (model 1 of knot_room), each with the quad's normal."""
    mesh = sc.meshes[sc.models[1].mesh]
    t = (np.arange(side) + 0.5) / side
    a, b = np.meshgrid(t, t, indexing="ij")
    out = []
    for q in range(len(mesh.vertices) // 4):
        p0, p1, _, p3 = mesh.vertices[4 * q: 4 * q + 4].astype(np.float64)
        pos = p0 + a.reshape(-1, 1) * (p1 - p0) + b.reshape(-1, 1) * (p3 - p0)
        pts = np.zeros(len(pos), dtype=capi.SURFACE_POINT_DTYPE)
        pts["position"], pts["normal"] = pos, mesh.normals[4 * q]
        out.append(pts)
    return np.concatenate(out)


def run_row(name, sc, pts, samples, args, torch):
    seed = 1
    n = len(pts)
    ref = open_mgr(ORACLE_LIB, sc)
    rays = lightmap_rays(ref.context, pts, samples, seed)
    ref.OnDestroy()

    mgr = open_mgr(CUDA_LIB, sc)
    ctx = mgr.context
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    d_pts = torch.from_numpy(np.ascontiguousarray(pts).view(np.uint8)).to("cuda")
    d_out = torch.empty(n * 16, dtype=torch.uint8, device="cuda")
    d_rays = torch.from_numpy(rays.view(np.uint8)).to("cuda")
    d_rad = torch.empty(n * samples * 16, dtype=torch.uint8, device="cuda")

    def bake():
        ctx.bake_lightmap_device(d_pts.data_ptr(), d_out.data_ptr(), n, samples, seed)

    def paths():
        ctx.trace_paths_device(d_rays.data_ptr(), d_rad.data_ptr(), n * samples, 1)
        with torch.cuda.stream(stream):
            L = d_rad.view(torch.float32).view(n, samples, 4)[..., :3]
            L = torch.where(torch.isfinite(L).all(dim=-1, keepdim=True), L, torch.zeros((), device="cuda"))
            return L.sum(dim=1) / samples

    def clock(fn):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ctx.reset_stats()
        a.record(stream)
        fn()
        b.record(stream)
        b.synchronize()
        return a.elapsed_time(b) / 1e3, ctx.stats()["rays"]

    def timed(fn):
        clock(fn)                                                                          # warm-up
        reps, total, segs = 0, 0.0, None
        while total < args.min_seconds:
            t, s = clock(fn)
            assert segs is None or s == segs
            segs = s
            total += t
            reps += 1
        return total / reps, segs

    arms = (("bake", bake), ("paths", paths))
    times = {k: [] for k, _ in arms}
    segs = {}
    for _ in range(3):
        for arm, fn in arms:
            t, s = timed(fn)
            times[arm].append(t)
            segs[arm] = s
    if segs["bake"] != segs["paths"]:
        raise SystemExit(f"{name}: the bake and paths arms count different segments ({segs})")

    ctx.synchronize()
    got = d_out.cpu().numpy().view(capi.CUBE_TEXEL_DTYPE)
    rad = d_rad.cpu().numpy().view(capi.PATH_RADIANCE_DTYPE)
    for t in np.random.RandomState(5).choice(n, min(n, 64), replace=False):
        rgb, rej = mean32(rad["rgb"][t * samples: (t + 1) * samples], 1, samples)
        if got["rgb"][t].tobytes() != rgb[0].tobytes() or got["rejected"][t] != rej[0]:
            raise SystemExit(f"{name}: texel {t} of the bake differs from the sums of the paths arm")
    mgr.OnDestroy()

    med = {k: float(np.median(v)) for k, v in times.items()}
    row = {"workload": name, "texels": n, "samples": samples, "segments": int(segs["bake"]), "paths_arm_bytes": n * samples * (28 + 16)}
    for arm, _ in arms:
        row[arm] = {"ms": round(med[arm] * 1e3, 3), "spread_ms": [round(min(times[arm]) * 1e3, 3), round(max(times[arm]) * 1e3, 3)],
                    "segments": int(segs[arm]), "Msegments_per_s": round(segs[arm] / med[arm] / 1e6, 1),
                    "texels_per_s": round(n / med[arm], 1)}
    row["bake_vs_paths"] = round(med["paths"] / med["bake"], 2)
    print(json.dumps(row), flush=True)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--min-seconds", type=float, default=0.5)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("lightmap_bench needs a CUDA device")
    print(json.dumps({"card": card(), "lib": os.path.relpath(CUDA_LIB, REPO)}), flush=True)
    S = 64 if args.quick else 256
    cap = 4096 if args.quick else None
    room = scenes.knot_room(64, 36, 8, 1)
    cluster = scenes.knot_cluster(64, 36, 12, 1)
    rows = (("knot_room knot vertices", room, model_vertices(room, 0)),
            ("knot_room walls 5 x 64^2", room, wall_grid(room)),
            ("871k cluster vertices / 13", cluster, model_vertices(cluster, 0, 13)))
    for name, sc, pts in rows:
        run_row(name, sc, np.ascontiguousarray(pts[:cap]), S, args, torch)


if __name__ == "__main__":
    main()
