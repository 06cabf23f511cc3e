#!/usr/bin/env python
"""Throughput of rtBakeCubemaps (reflection probes: HDR cube maps of path-traced radiance, each texel the mean of S paths spread over
its area) against the two routes through rtTracePaths.

    python tools/cubemap_bench.py [--quick] [--min-seconds 0.5]

Arms, alternated three times per workload (medians, min..max spread):
  bake    rtBakeCubemapsDevice(positions, n, N, S) on torch CUDA tensors; CUDA events around the call on the context's stream
  paths   rtTracePathsDevice(samples = 1) on the n * 6 * N^2 * S rays of orCubemapRays (each sample's own direction and starting state,
          built once outside the timed window: 28 bytes per sample, plus 16 of radiance), then the mean in torch with non-finite samples
          zeroed; CUDA events around both.  The same result as the bake, up to the order of the sums
  centre  rtTracePathsDevice(samples = S) on one ray per texel through its centre: no memory per sample, but every sample follows the
          same direction (the texel aliases) and one NaN path spoils its texel
Msegments/s is RtStats.rays (one per CalculateRayCollision) over the call's time; texels/s is n * 6 * N^2 over it.  The tool stops with
an error unless the bake and paths arms count the same segments, and unless the bake equals, bit for bit, the header's sums (numpy,
binary32) of the paths arm's radiances for a subset of texels.  Prints the card name and power limit read in the same run.

Workloads: the Cornell box and the knot room with a glass knot, at 1 probe x 6 x 128^2 x 256 samples and 64 probes x 6 x 32^2 x 256
samples (--quick: 1 probe x 6 x 32^2 x 64).
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
from ray_tracing_b200 import capi, scenes                         # noqa: E402
from test_gpu_cubemaps import cubemap_rays, mean32                # noqa: E402
from test_gpu_probes import probe_positions                       # noqa: E402
from trace_rays_bench import card                                 # noqa: E402


def open_mgr(lib, sc):
    mgr = rt.RayComputeManager(lib)
    scenes.apply(sc, mgr)
    mgr.OnEnable()
    return mgr


def run_row(name, sc, n, N, samples, args, torch):
    seed = 1
    texels = n * 6 * N * N
    pos = probe_positions(sc, seed=3, n=n, special=False)
    ref = open_mgr(ORACLE_LIB, sc)
    rays = cubemap_rays(ref.context, pos, N, samples, seed)
    centre = cubemap_rays(ref.context, pos, N, 1, seed)                                    # sample 0's offset is the texel centre
    ref.OnDestroy()

    mgr = open_mgr(CUDA_LIB, sc)
    ctx = mgr.context
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    d_pos = torch.from_numpy(pos).to("cuda")
    d_cube = torch.empty(texels * 16, dtype=torch.uint8, device="cuda")
    d_rays = torch.from_numpy(rays.view(np.uint8)).to("cuda")
    d_rad = torch.empty(texels * samples * 16, dtype=torch.uint8, device="cuda")
    d_centre = torch.from_numpy(centre.view(np.uint8)).to("cuda")
    d_crad = torch.empty(texels * 16, dtype=torch.uint8, device="cuda")

    def bake():
        ctx.bake_cubemaps_device(d_pos.data_ptr(), d_cube.data_ptr(), n, N, samples, seed)

    def paths():
        ctx.trace_paths_device(d_rays.data_ptr(), d_rad.data_ptr(), texels * samples, 1)
        with torch.cuda.stream(stream):
            L = d_rad.view(torch.float32).view(texels, samples, 4)[..., :3]
            L = torch.where(torch.isfinite(L).all(dim=-1, keepdim=True), L, torch.zeros((), device="cuda"))
            return L.sum(dim=1) / samples

    def centre_rays():
        ctx.trace_paths_device(d_centre.data_ptr(), d_crad.data_ptr(), texels, samples)

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

    arms = (("bake", bake), ("paths", paths), ("centre", centre_rays))
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
    got = d_cube.cpu().numpy().view(capi.CUBE_TEXEL_DTYPE)
    rad = d_rad.cpu().numpy().view(capi.PATH_RADIANCE_DTYPE)
    for t in np.random.RandomState(5).choice(texels, min(texels, 64), replace=False):
        rgb, rej = mean32(rad["rgb"][t * samples: (t + 1) * samples], 1, samples)
        if got["rgb"][t].tobytes() != rgb[0].tobytes() or got["rejected"][t] != rej[0]:
            raise SystemExit(f"{name}: texel {t} of the bake differs from the sums of the paths arm")
    mgr.OnDestroy()

    med = {k: float(np.median(v)) for k, v in times.items()}
    row = {"workload": name, "probes": n, "faceSize": N, "samples": samples, "texels": texels, "segments": int(segs["bake"]),
           "paths_arm_bytes": texels * samples * (28 + 16)}
    for arm, _ in arms:
        row[arm] = {"ms": round(med[arm] * 1e3, 3), "spread_ms": [round(min(times[arm]) * 1e3, 3), round(max(times[arm]) * 1e3, 3)],
                    "segments": int(segs[arm]), "Msegments_per_s": round(segs[arm] / med[arm] / 1e6, 1),
                    "texels_per_s": round(texels / med[arm], 1)}
    row["bake_vs_paths"] = round(med["paths"] / med["bake"], 2)
    row["bake_vs_centre"] = round(med["centre"] / med["bake"], 2)
    row["bake_vs_centre_segment_rate"] = round((segs["bake"] / med["bake"]) / (segs["centre"] / med["centre"]), 2)
    print(json.dumps(row), flush=True)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--min-seconds", type=float, default=0.5)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("cubemap_bench needs a CUDA device")
    print(json.dumps({"card": card(), "lib": os.path.relpath(CUDA_LIB, REPO)}), flush=True)
    sizes = [(1, 32, 64)] if args.quick else [(1, 128, 256), (64, 32, 256)]
    for n, N, s in sizes:
        run_row(f"cornell n={n} N={N} S={s}", scenes.cornell_spheres(64, 64, 4, 1), n, N, s, args, torch)
        run_row(f"knot_room_glass n={n} N={N} S={s}", scenes.knot_room(64, 36, 8, 1, glass=True), n, N, s, args, torch)


if __name__ == "__main__":
    main()
