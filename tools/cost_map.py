#!/usr/bin/env python
"""Per-pixel cost of a workload: renders it with "countStats" = 1 and writes the four heat maps of the reference's debug view
(visMode 1 box tests / ray, 2 triangle tests / ray, 3 sphere tests / ray, 4 rays per pixel) as PNG, then prints ONE JSON line with
the distribution over pixels of rays, box tests and triangle tests (mean, p50, p99, max) and, on a GPU, the card and its power limit.

    python tools/cost_map.py                                  # bench.py's default workload (1920x1080, 8 bounces, 256 spp), 1 frame
    python tools/cost_map.py --workload knot1 --frames 4 --out /tmp/cost
    python tools/cost_map.py --scene cornell_spheres --size 64x48 --spp 2 --bounces 4 --lib oracle/liboracle.so   # toy rehearsal

--lib: the library implementing include/rt_b200.h (default: the product; the oracle or the SIMT interpreter build for rehearsals).
A heat map's scale (full white) is the 99th percentile of its quantity unless --scale gives one; pixels above it are red.
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

import ray_tracing_b200 as rt  # noqa: E402
from ray_tracing_b200 import capi, scenes  # noqa: E402
from ray_tracing_b200.display import write_png  # noqa: E402

MODE_NAMES = {1: "box_per_ray", 2: "tri_per_ray", 3: "sphere_per_ray", 4: "rays"}


def gpu_info():
    """Name and power limit of GPU 0 as nvidia-smi reports them (None without one)."""
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = [s.strip() for s in out.split(",")[:2]]
        return {"gpu": name, "power_limit_w": float(limit)}
    except Exception:
        return {"gpu": None, "power_limit_w": None}


def distribution(a):
    a = a.astype(np.float64).ravel()
    return {"mean": round(float(a.mean()), 3), "p50": float(np.percentile(a, 50)), "p99": float(np.percentile(a, 99)), "max": float(a.max())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default=None, help="a bench.py workload (default: its DEFAULT_WORKLOAD)")
    ap.add_argument("--scene", default=None, help="instead of a workload: a scene function of ray_tracing_b200/scenes.py")
    ap.add_argument("--size", default="64x48", help="--scene: WxH")
    ap.add_argument("--spp", type=int, default=2, help="--scene: NumRaysPerPixel")
    ap.add_argument("--bounces", type=int, default=4, help="--scene: MaxBounceCount")
    ap.add_argument("--frames", type=int, default=1)
    ap.add_argument("--kernel", type=int, default=None)
    ap.add_argument("--scale", type=float, default=None, help="full-white value of every heat map (default: each one's p99)")
    ap.add_argument("--lib", default=None)
    ap.add_argument("--out", default="cost_map", help="directory for the PNG files")
    args = ap.parse_args()

    if args.scene:
        w, h = (int(v) for v in args.size.split("x"))
        sc = getattr(scenes, args.scene)(w, h, args.bounces, args.spp)
        name = f"{args.scene} {w}x{h}, {args.bounces} bounces, {args.spp} spp"
    else:
        import bench
        wname = args.workload or bench.DEFAULT_WORKLOAD
        sc = bench.make_scene(bench.WORKLOADS[wname])
        name = f"{wname}: {bench.WORKLOADS[wname]['desc']}"
    lib = args.lib or capi.DEFAULT_LIB
    mgr = rt.RayComputeManager(lib)
    scenes.apply(sc, mgr)
    ctx = mgr.context
    ctx.set_option("countStats", 1)
    if args.kernel is not None:
        ctx.set_option("kernel", args.kernel)
    mgr.OnEnable()
    ctx.reset_stats()
    t0 = time.perf_counter()
    for _ in range(args.frames):
        mgr.RenderFrame()
    ctx.synchronize()
    wall = time.perf_counter() - t0
    st = ctx.stats()
    pix = mgr.pixel_stats()
    for k in ("rays", "boxTests", "triTests", "sphereTests", "sphereBoxTests"):
        assert int(pix[k].astype(np.uint64).sum()) == st[k], f"PixelStats.{k} does not sum to RtStats.{k}"
    traced = pix["rays"] > 0
    rays = np.maximum(pix["rays"], 1).astype(np.float64)
    per_ray = {1: pix["boxTests"] / rays, 2: pix["triTests"] / rays, 3: (pix["sphereTests"].astype(np.float64) + pix["sphereBoxTests"]) / rays,
               4: pix["rays"].astype(np.float64)}
    os.makedirs(args.out, exist_ok=True)
    scales = {}
    for mode, vals in per_ray.items():
        s = args.scale or float(np.percentile(vals[traced], 99)) if traced.any() else 1.0
        s = s if s > 0 else 1.0
        scales[MODE_NAMES[mode]] = s
        write_png(os.path.join(args.out, f"{MODE_NAMES[mode]}.png"), mgr.debug_view(mode, s)[::-1, :, :3])
    mgr.OnDestroy()
    rec = {"scene": name, "frames": args.frames, "pixels": int(pix.size), "kernel_ms": round(st["kernelMs"], 3), "wall_s": round(wall, 3),
           "rays_per_pixel": distribution(pix["rays"]), "box_tests_per_pixel": distribution(pix["boxTests"]),
           "tri_tests_per_pixel": distribution(pix["triTests"]), "box_tests_per_ray": distribution(per_ray[1][traced]),
           "heat_map_scales": scales, "png_dir": os.path.abspath(args.out), "lib": os.path.basename(lib)}
    rec.update(gpu_info() if lib == capi.DEFAULT_LIB else {"gpu": None, "power_limit_w": None})
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
