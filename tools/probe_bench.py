#!/usr/bin/env python
"""Throughput of rtBakeProbes (light probes: path-traced radiance projected onto L2 spherical harmonics) against the route that existed
before it: rtTracePathsDevice on materialised rays, one per (probe, sample), then an SH projection in torch.

    python tools/probe_bench.py [--quick] [--min-seconds 0.5]

Arms, alternated three times per workload (medians, min..max spread):
  bake    rtBakeProbesDevice(positions, n, S) on torch CUDA tensors; CUDA events around the call on the context's stream
  paths   rtTracePathsDevice(samples = 1) on the n * S rays of orProbeRays (each sample's position, direction and starting state,
          built once outside the timed window), then the projection in torch: non-finite samples zeroed, an einsum with the basis of
          the S directions (also built once) and the scale; CUDA events around both
Msegments/s is RtStats.rays (one per CalculateRayCollision) over the call's time; probes/s is n over it.  The tool stops with an error
unless both arms count the same segments, and unless the bake equals, bit for bit, the header's projection (numpy, binary32) of the
paths arm's radiances for a subset of probes.  Prints the card name and power limit read in the same run.

Workloads: the Cornell box and the knot room with a glass knot, at 1,024 probes x 4,096 samples and 16,384 probes x 1,024 samples
(--quick: 256 x 1,024 only).
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
from test_gpu_probes import basis32, probe_positions, probe_rays, project32   # noqa: E402
from trace_rays_bench import card                                 # noqa: E402


def open_mgr(lib, sc):
    mgr = rt.RayComputeManager(lib)
    scenes.apply(sc, mgr)
    mgr.OnEnable()
    return mgr


def run_row(name, sc, n, samples, args, torch):
    seed = 1
    pos = probe_positions(sc, seed=3, n=n, special=False)
    ref = open_mgr(ORACLE_LIB, sc)
    rays = probe_rays(ref.context, pos, samples, seed)
    ref.OnDestroy()

    mgr = open_mgr(CUDA_LIB, sc)
    ctx = mgr.context
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    d_pos = torch.from_numpy(pos).to("cuda")
    d_sh = torch.empty(n * 112, dtype=torch.uint8, device="cuda")
    d_rays = torch.from_numpy(rays.view(np.uint8)).to("cuda")
    d_rad = torch.empty(n * samples * 16, dtype=torch.uint8, device="cuda")
    d_Y = torch.from_numpy(basis32(rays["dir"][:samples])).to("cuda")                      # (S, 9), the same for every probe
    scale = float(np.float32(12.566371) / np.float32(samples))

    def bake():
        ctx.bake_probes_device(d_pos.data_ptr(), d_sh.data_ptr(), n, samples, seed)

    def paths():
        ctx.trace_paths_device(d_rays.data_ptr(), d_rad.data_ptr(), n * samples, 1)
        with torch.cuda.stream(stream):
            L = d_rad.view(torch.float32).view(n, samples, 4)[..., :3]
            L = torch.where(torch.isfinite(L).all(dim=-1, keepdim=True), L, torch.zeros((), device="cuda"))
            return torch.einsum("psc,si->pci", L, d_Y) * scale

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

    times = {"bake": [], "paths": []}
    segs = {}
    for _ in range(3):
        for arm, fn in (("bake", bake), ("paths", paths)):
            t, s = timed(fn)
            times[arm].append(t)
            segs[arm] = s
    if segs["bake"] != segs["paths"]:
        raise SystemExit(f"{name}: the arms count different segments ({segs})")

    ctx.synchronize()
    got = d_sh.cpu().numpy().view(capi.PROBE_SH_DTYPE)
    rad = d_rad.cpu().numpy().view(capi.PATH_RADIANCE_DTYPE)
    sub = np.random.RandomState(5).choice(n, min(n, 32), replace=False)
    for p in sub:
        sl = slice(p * samples, (p + 1) * samples)
        sh, rej = project32(rays[sl], rad["rgb"][sl], 1, samples)
        if got["sh"][p].tobytes() != sh[0].tobytes() or got["rejected"][p] != rej[0]:
            raise SystemExit(f"{name}: probe {p} of the bake differs from the projection of the paths arm")
    mgr.OnDestroy()

    med = {k: float(np.median(v)) for k, v in times.items()}
    row = {"workload": name, "probes": n, "samples": samples, "segments": int(segs["bake"])}
    for arm in ("bake", "paths"):
        row[arm] = {"ms": round(med[arm] * 1e3, 3), "spread_ms": [round(min(times[arm]) * 1e3, 3), round(max(times[arm]) * 1e3, 3)],
                    "Msegments_per_s": round(segs[arm] / med[arm] / 1e6, 1), "probes_per_s": round(n / med[arm], 1)}
    row["speedup"] = round(med["paths"] / med["bake"], 2)
    print(json.dumps(row), flush=True)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--min-seconds", type=float, default=0.5)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("probe_bench needs a CUDA device")
    print(json.dumps({"card": card(), "lib": os.path.relpath(CUDA_LIB, REPO)}), flush=True)
    sizes = [(256, 1024)] if args.quick else [(1024, 4096), (16384, 1024)]
    for n, s in sizes:
        run_row(f"cornell n={n} S={s}", scenes.cornell_spheres(64, 64, 4, 1), n, s, args, torch)
        run_row(f"knot_room_glass n={n} S={s}", scenes.knot_room(64, 36, 8, 1, glass=True), n, s, args, torch)


if __name__ == "__main__":
    main()
