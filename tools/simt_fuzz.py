#!/usr/bin/env python
"""Randomised parity search WITHOUT a GPU: random small scenes (spheres, instanced and transformed meshes, glass / checker /
emissive materials, sky, defocus, near / far / inside cameras, extreme scales) rendered by the kernels' own source on the SIMT
interpreter build (tests/simt) with random options, compared bit for bit with the oracle.  Found the distant-camera defect of the
model skipping in round 1 by hand-made cases; this keeps looking.  Every failure prints the seed that reproduces it.

    python tools/simt_fuzz.py [--cases 200] [--seed 1] [--lib path/to/another/build.so] [--pixel-stats] [--queries] [--occlusion] [--paths]

--pixel-stats: wherever the traversal totals are compared (counting launches of whole images), also compare the per-pixel counters
(PixelStats: rays, box and triangle tests everywhere; sphere tests too when the Spheres buffer is below the accelerator's threshold).

--queries: every scene also traces a random batch of rays (rtTraceRays, tests/test_gpu_trace_rays.py ray_sets: pick rays, origins in the
scene, inside its meshes and spheres, 1e3 - 1e5 units out, special directions and NaN / inf) with either flag, compared bit for bit
with the oracle (a NaN must be a NaN on both sides), and with "countStats" the counters the batch added.

--occlusion: every scene also traces a random batch of segments (rtTraceOcclusion): the rays of --queries with tMax at, one ulp below
and one ulp above the oracle's closest hit, fractions of it, +inf and special values (tests/test_gpu_occlusion.py tmax_sets), with
either flag, compared with the oracle's answers, and with "countStats" the early-exit counters the batch added.

--paths: every scene also traces a random batch of path rays (rtTracePaths): the rays of --queries with random RNG states
(tests/test_gpu_trace_paths.py path_rays) and a random sample count, under the scene's random MaxBounceCount / UseSky / sun, compared
bit for bit with the oracle in rgb and final state, and the segments (RtStats.rays) and, with "countStats", the counters the batch added.
"""
import argparse
import os
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tests"))
sys.path.insert(0, os.path.join(REPO, "tests", "simt"))
import build as simt_build                      # noqa: E402
from conftest import ORACLE_LIB, render        # noqa: E402
import ray_tracing_b200 as rt                   # noqa: E402
from ray_tracing_b200 import scenes             # noqa: E402
from test_gpu_trace_rays import assert_hits_equal, ray_sets      # noqa: E402  (the query batch of the rtTraceRays tests)
from test_gpu_occlusion import assert_occlusion_equal, tmax_sets  # noqa: E402  (the segment lengths of the rtTraceOcclusion tests)
from test_gpu_trace_paths import assert_radiance_equal, path_rays  # noqa: E402  (the path rays of the rtTracePaths tests)


def render_pixel_stats(lib, sc, frames, options, tile=None):
    """conftest.render plus the PixelStats image of the frames (None unless the launch counts)."""
    mgr = rt.RayComputeManager(lib)
    scenes.apply(sc, mgr)
    ctx = mgr.context
    for k, v in (options or {}).items():
        ctx.set_option(k, v)
    if tile:
        ctx.set_tile(*tile)
    mgr.OnEnable()
    ctx.reset_stats()
    for _ in range(frames):
        mgr.RenderFrame()
    out = (mgr.raytraceFrameTex, mgr.accumulatedResult, ctx.stats(), mgr.pixel_stats() if (options or {}).get("countStats") else None)
    mgr.OnDestroy()
    return out


def trace_batch(lib, sc, options, rays, no_cull, occlusion=False, samples=0):
    """rtTraceRays of `rays` (occlusion: rtTraceOcclusion of segments) on a fresh context of the scene (after OnEnable), with the
    RtStats counters the batch added."""
    mgr = rt.RayComputeManager(lib)
    scenes.apply(sc, mgr)
    ctx = mgr.context
    for k, v in (options or {}).items():
        ctx.set_option(k, v)
    mgr.OnEnable()
    ctx.reset_stats()
    if samples:                                  # rtTracePaths of path rays
        hits = ctx.trace_paths(rays, samples)
    else:
        hits = ctx.trace_occlusion(rays, no_cull=no_cull) if occlusion else ctx.trace_rays(rays, no_cull=no_cull)
    out = (hits, ctx.stats())
    mgr.OnDestroy()
    return out


def pixel_stats_differ(a, b, spheres):
    """Fields of two PixelStats images that differ (sphere tests only below the 65 spheres where the accelerator starts)."""
    keys = ("rays", "boxTests", "triTests") + (("sphereTests",) if spheres <= 64 else ())
    return [k for k in keys if not np.array_equal(a[k], b[k])]


def random_material(rng):
    kind = rng.randint(0, 6)
    if kind == 0:
        return scenes.material(flag=scenes.MAT_GLASS, ior=float(rng.uniform(1.0, 2.2)), smoothness=float(rng.uniform(0, 1)), specularProbability=float(rng.uniform(0, 1)),
                               absorption=tuple(rng.uniform(0, 1, 3)), absorptionStrength=float(rng.uniform(0, 3)))
    if kind == 1:
        return scenes.material(flag=scenes.MAT_CHECKER, diffuse=tuple(rng.uniform(0, 1, 3)), emission=tuple(rng.uniform(0, 1, 3)), specularProbability=float(rng.uniform(0, 0.5)))
    if kind == 2:
        return scenes.material(diffuse=(0, 0, 0), emission=tuple(rng.uniform(0.2, 1, 3)), emissionStrength=float(rng.uniform(1, 20)))
    return scenes.material(diffuse=tuple(rng.uniform(0.05, 1, 3)), specular=tuple(rng.uniform(0.5, 1, 3)), smoothness=float(rng.uniform(0, 1)),
                           specularProbability=float(rng.choice([0.0, 1.0, rng.uniform(0, 1)])))


def random_scene(rng, odd=0.06):
    meshes = [scenes.knot_mesh(nu=int(rng.randint(12, 60)), nv=int(rng.randint(4, 9))), scenes.room_mesh(),
              scenes.quad_mesh((-0.5, 0, -0.5), (0.5, 0, -0.5), (0.5, 0, 0.5), (-0.5, 0, 0.5))]
    soup = scenes.random_soup(8, 8, 1, 1, triangles=int(rng.randint(60, 1500)), spheres=0, seed=int(rng.randint(1, 1000)))
    meshes.append(soup.meshes[0])
    models = []
    if rng.rand() < 0.7:
        models.append(scenes.ModelDesc(1, np.eye(4), np.eye(4), random_material(rng)))
    spread = float(rng.choice([1.0, 1.0, 30.0, 1e3]))
    for _ in range(int(rng.choice([0, 1, 2, 5, 12, 30, 70]))):
        mesh = int(rng.choice([0, 2, 3]))
        base = 0.05 if mesh == 3 else 1.0
        scale = base * np.exp(rng.uniform(np.log(0.02), np.log(1.5), 3)) * (rng.choice([1, 1, 1, -1], 3) if rng.rand() < 0.2 else 1)
        l2w, w2l = scenes.trs(position=tuple(rng.uniform(-2.5, 2.5, 3) * spread + np.array([0, 2.0, 0])), euler_deg=tuple(rng.uniform(0, 360, 3)), scale=tuple(scale))
        odd = rng.rand()
        if odd < 0.04:                                # localToWorld of another transform: only the normals notice
            l2w = scenes.trs(position=tuple(rng.uniform(-5, 5, 3)), euler_deg=tuple(rng.uniform(0, 360, 3)), scale=tuple(rng.uniform(0.1, 2, 3)))[0]
        elif odd < 0.05:                              # singular worldToLocal
            w2l = w2l.copy(); w2l[int(rng.randint(0, 3)), :] = 0.0
        models.append(scenes.ModelDesc(mesh, l2w, w2l, random_material(rng)))
    ns = int(rng.choice([0, 0, 1, 5, 40, 64, 65, 200]))
    sph = np.zeros(ns, dtype=scenes.SPHERE_DTYPE)
    for i in range(ns):
        sph[i] = scenes._sphere(tuple(rng.uniform(-2.5, 2.5, 3) * spread + np.array([0, 2.0, 0])), float(np.exp(rng.uniform(np.log(0.01), np.log(1.0))) * spread ** 0.5), random_material(rng))
    dist = float(rng.choice([0.0, 2.0, 5.67, 5.67, 40.0, 3000.0, 2e5])) * (spread if spread < 100 else 1.0)
    cam = scenes.trs(position=(float(rng.uniform(-1, 1)), 1.9 + float(rng.uniform(-1, 1)), -dist), euler_deg=(float(rng.uniform(-8, 8)), float(rng.uniform(-8, 8)), float(rng.uniform(-30, 30))))[0]
    fov = float(np.clip(np.degrees(2 * np.arctan(3.0 * max(spread, 1.0) / max(dist, 3.0))), 1e-4, 100.0))
    w, h = int(rng.choice([1, 7, 16, 33, 48, 64])), int(rng.choice([1, 5, 9, 24, 36]))
    if rng.rand() < odd:                              # non-finite and degenerate numbers where a scene can carry them
        special = [np.nan, np.inf, -np.inf, 0.0, -1.0]
        for _ in range(int(rng.randint(1, 4))):
            what = int(rng.randint(0, 5))
            if what == 0 and len(sph):
                sph["radius"][int(rng.randint(0, len(sph)))] = rng.choice(special)
            elif what == 1 and len(sph):
                sph["centre"][int(rng.randint(0, len(sph)))][int(rng.randint(0, 3))] = rng.choice(special[:3])
            elif what == 2 and models:
                k = int(rng.randint(0, len(models))); m = models[k]
                w2l = m.world_to_local.copy(); w2l[int(rng.randint(0, 3)), int(rng.randint(0, 4))] = rng.choice(special[:3])
                models[k] = scenes.ModelDesc(m.mesh, m.local_to_world, w2l, m.material)
            elif what == 3 and models:
                k = int(rng.randint(0, len(models))); m = models[k]
                mat = m.material.copy(); mat["ior" if rng.rand() < 0.5 else "smoothness"] = rng.choice(special)
                models[k] = scenes.ModelDesc(m.mesh, m.local_to_world, m.world_to_local, mat)
            else:
                cam = cam.copy(); cam[int(rng.randint(0, 3)), int(rng.randint(0, 4))] = rng.choice(special[:3])
    used = sorted({m.mesh for m in models})
    remap = {old: new for new, old in enumerate(used)}
    models = [scenes.ModelDesc(remap[m.mesh], m.local_to_world, m.world_to_local, m.material) for m in models]
    return scenes.Scene(name="fuzz", width=w, height=h, spheres=sph, meshes=[meshes[i] for i in used], models=models, cam_local_to_world=cam, fov=fov,
                        settings=dict(maxBounceCount=int(rng.choice([0, 1, 3, 6, 12])), numRaysPerPixel=int(rng.choice([1, 1, 2, 3])), useSky=bool(rng.rand() < 0.5),
                                      defocusStrength=float(rng.choice([0.0, 0.0, 40.0])), divergeStrength=float(rng.choice([0.0, 0.3, 3.0])),
                                      bvhQuality=int(rng.choice([1, 1, 0, 2])), renderSeed=int(rng.randint(0, 2 ** 31 - 1))),
                        sun_forward=tuple(rng.uniform(-1, 1, 3)))


def far_scene(rng):
    """Many small models seen from very far: the class of scene that exposed the fixed padding of the model boxes."""
    meshes = [scenes.quad_mesh((-0.5, 0, -0.5), (0.5, 0, -0.5), (0.5, 0, 0.5), (-0.5, 0, 0.5)), scenes.knot_mesh(nu=12, nv=4)]
    models = []
    lo, hi = float(rng.choice([0.005, 0.02])), float(rng.choice([0.05, 0.3]))
    for _ in range(int(rng.choice([150, 500, 1200]))):
        l2w, w2l = scenes.trs(position=(rng.uniform(-2.5, 2.5), rng.uniform(0.2, 3.8), rng.uniform(-2.5, 2.5)), euler_deg=tuple(rng.uniform(0, 360, 3)),
                              scale=tuple(rng.uniform(lo, hi, 3)))
        models.append(scenes.ModelDesc(int(rng.randint(0, 2)), l2w, w2l, scenes.material(diffuse=(0.8, 0.8, 0.8), emission=(1, 1, 1), emissionStrength=1.0)))
    dist = float(np.exp(rng.uniform(np.log(2e3), np.log(2e6))))
    cam = scenes.trs(position=(float(rng.uniform(-1, 1)), 1.9, -dist), euler_deg=(0, 0, float(rng.uniform(0, 360))))[0]
    return scenes.Scene(name="far", width=128, height=72, meshes=meshes, models=models, cam_local_to_world=cam, fov=float(np.degrees(2 * np.arctan(3.2 / dist))),
                        settings=dict(maxBounceCount=int(rng.choice([0, 1, 2])), numRaysPerPixel=2, divergeStrength=0.0, renderSeed=int(rng.randint(0, 2 ** 31 - 1))))


def sphere_scene(rng):
    """Large Spheres buffers (the padded-box accelerator): nested, overlapping, duplicated, tiny and huge spheres, any camera distance."""
    n = int(rng.choice([65, 200, 1000, 3000]))
    spread = float(rng.choice([1.0, 10.0, 300.0]))
    sph = np.zeros(n, dtype=scenes.SPHERE_DTYPE)
    centres = rng.uniform(-3, 3, (n, 3)) * spread
    radii = np.exp(rng.uniform(np.log(1e-3), np.log(2.0), n)) * spread
    for i in range(n):
        if i and rng.rand() < 0.1:
            centres[i] = centres[int(rng.randint(0, i))]                   # concentric / duplicated
            if rng.rand() < 0.5:
                radii[i] = radii[int(rng.randint(0, i))]
        sph[i] = scenes._sphere(tuple(centres[i]), float(radii[i]), random_material(rng))
    dist = float(np.exp(rng.uniform(np.log(0.1), np.log(1e5)))) * spread
    cam = scenes.trs(position=(float(rng.uniform(-1, 1)) * spread, float(rng.uniform(-1, 1)) * spread, -dist), euler_deg=(float(rng.uniform(-5, 5)), float(rng.uniform(-5, 5)), 0.0))[0]
    fov = float(np.clip(np.degrees(2 * np.arctan(4.0 * spread / max(dist, spread))), 1e-4, 100.0))
    return scenes.Scene(name="spheres", width=int(rng.choice([32, 64])), height=int(rng.choice([18, 36])), spheres=sph, cam_local_to_world=cam, fov=fov,
                        settings=dict(maxBounceCount=int(rng.choice([1, 4, 8])), numRaysPerPixel=int(rng.choice([1, 2])), useSky=bool(rng.rand() < 0.5),
                                      divergeStrength=float(rng.choice([0.0, 0.3])), renderSeed=int(rng.randint(0, 2 ** 31 - 1))), sun_forward=tuple(rng.uniform(-1, 1, 3)))


def random_options(rng):
    o = {"kernel": int(rng.choice([1, 2, 2]))}
    if rng.rand() < 0.5:
        o["tlas"] = int(rng.choice([-1, 0, 1]))
    if rng.rand() < 0.2:
        o["modelSkip"] = 0
    if o["kernel"] == 2:
        if rng.rand() < 0.4:
            o["poolSlots"] = int(rng.choice([32, 64, 96]))
        if rng.rand() < 0.4:
            o["tailLanes"] = int(rng.choice([0, 3, 16, 31]))
        if rng.rand() < 0.3:
            o["sortRays"] = 1
    if rng.rand() < 0.3:
        o["smemNodes"] = int(rng.choice([1, 17, 300]))
    if rng.rand() < 0.3:
        o["pairOrder"] = int(rng.choice([1, 2, 4]))
    if rng.rand() < 0.3:
        o["gridFit"] = 1
    if rng.rand() < 0.2:
        o["extInstantiation"] = 1
    if rng.rand() < 0.15:
        o["countStats"] = 1
    if rng.rand() < 0.35:
        o["sampleChunks"] = int(rng.choice([0, 2, 3, 7]))       # round 2: a pixel's chain split over lanes / slots (scenes here have 1-3 samples per pixel)
    return o


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", type=int, default=200)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--lib", default=None)
    ap.add_argument("--odd", type=float, default=0.06, help="share of cases with NaN / inf / zero / negative numbers in spheres, matrices, materials, camera")
    ap.add_argument("--spheres", type=float, default=0.05, help="share of cases of the large-Spheres-buffer class")
    ap.add_argument("--far", type=float, default=0.05, help="share of cases of the many-small-models-from-afar class")
    ap.add_argument("--pixel-stats", action="store_true", help="also compare the per-pixel counters wherever the totals are compared")
    ap.add_argument("--queries", action="store_true", help="also trace a random batch of rays through every scene (rtTraceRays) against the oracle")
    ap.add_argument("--query-rays", type=int, default=32, help="rays per kind in a --queries batch")
    ap.add_argument("--occlusion", action="store_true", help="also trace a random batch of segments through every scene (rtTraceOcclusion) against the oracle")
    ap.add_argument("--paths", action="store_true", help="also trace a random batch of path rays through every scene (rtTracePaths) against the oracle")
    args = ap.parse_args()
    lib = args.lib or simt_build.build()
    bad, pix_cases, query_cases, occlusion_cases, path_cases, t0 = 0, 0, 0, 0, 0, time.time()
    for case in range(args.cases):
        seed = args.seed * 100003 + case
        rng = np.random.RandomState(seed)
        far = rng.rand() < args.far
        sc = far_scene(rng) if far else (sphere_scene(rng) if rng.rand() < args.spheres else random_scene(rng, args.odd))
        frames = int(rng.choice([1, 1, 2]))
        # (the pooled kernel is slow on the interpreter with 1,000 models: it gets the smaller far scenes only)
        opts = {"kernel": 2 if len(sc.models) <= 150 and rng.rand() < 0.5 else 1, "tlas": int(rng.choice([0, 1]))} if far else random_options(rng)
        tile = (int(rng.randint(0, 3)), 3, int(rng.choice([1, 4, 8]))) if rng.rand() < 0.15 else None
        pix_case = args.pixel_stats and tile is None and bool(opts.get("countStats"))
        try:
            if pix_case:
                fo, ao, so, po = render_pixel_stats(ORACLE_LIB, sc, frames, {"countStats": 1})
                fg, ag, sg, pg = render_pixel_stats(lib, sc, frames, opts)
            else:
                fo, ao, so = render(ORACLE_LIB, sc, frames=frames, want_stats=True)
                fg, ag, sg = render(lib, sc, frames=frames, options=opts, want_stats=True, tile=tile)
        except Exception as e:                    # an error code from either side is a finding too
            print(f"case seed {seed}: {type(e).__name__}: {e}   options {opts}", flush=True)
            bad += 1
            continue
        rows = slice(None) if tile is None else [y for y in range(sc.height) if (y // tile[2]) % tile[1] == tile[0]]
        a, b = ag[rows], ao[rows]
        diff = (a.view(np.uint32) != b.view(np.uint32)) & ~(np.isnan(a) & np.isnan(b))
        counters_ok = tile is not None or not opts.get("countStats") or all(sg[k] == so[k] for k in ("rays", "boxTests", "triTests"))
        pix_bad = pixel_stats_differ(pg, po, len(sc.spheres)) if pix_case else []
        if pix_case:
            pix_cases += 1
        if diff.any() or not counters_ok or pix_bad:
            bad += 1
            print(f"case seed {seed}: {int(diff.sum())} values differ, counters {'ok' if counters_ok else 'DIFFER'}, PixelStats {pix_bad or 'ok'}; {len(sc.models)} models, {len(sc.spheres)} spheres, "
                  f"{sc.width}x{sc.height}, frames {frames}, options {opts}, tile {tile}, settings {sc.settings}", flush=True)
        if args.queries:
            # pick rays, origins inside the scene and inside its meshes / spheres, 1e3 - 1e5 units out, axis-aligned / zero / NaN / inf
            sets = ray_sets(sc, seed=seed, n=args.query_rays)
            batch = np.concatenate(list(sets.values()))
            batch = batch[rng.permutation(len(batch))]
            no_cull = bool(rng.rand() < 0.5)
            q_opts = {k: v for k, v in opts.items() if k in ("tlas", "modelSkip", "extInstantiation", "countStats", "smemNodes", "pairOrder")}
            try:
                want, so = trace_batch(ORACLE_LIB, sc, {}, batch, no_cull)
                got, sg = trace_batch(lib, sc, q_opts, batch, no_cull)
                assert_hits_equal(got, want, "rtTraceRays")
                keys = ("rays", "boxTests", "triTests") + (("sphereTests",) if len(sc.spheres) <= 64 else ())
                assert not q_opts.get("countStats") or all(sg[k] == so[k] for k in keys), f"counters {sg} vs {so}"
                query_cases += 1
            except Exception as e:
                bad += 1
                print(f"case seed {seed}: queries: {type(e).__name__}: {e}   options {q_opts}, no_cull {no_cull}, {len(sc.models)} models, {len(sc.spheres)} spheres", flush=True)
        if args.occlusion:
            orng = np.random.RandomState(seed + 7)
            rays = np.concatenate(list(ray_sets(sc, seed=seed + 7, n=args.query_rays).values()))
            no_cull = bool(orng.rand() < 0.5)
            o_opts = {k: v for k, v in opts.items() if k in ("tlas", "modelSkip", "extInstantiation", "countStats", "smemNodes", "pairOrder")}
            try:
                closest, _ = trace_batch(ORACLE_LIB, sc, {}, rays, no_cull)
                segs = np.concatenate(list(tmax_sets(rays, closest, seed=seed).values()))
                segs = segs[orng.permutation(len(segs))]
                want, so = trace_batch(ORACLE_LIB, sc, {}, segs, no_cull, occlusion=True)
                got, sg = trace_batch(lib, sc, o_opts, segs, no_cull, occlusion=True)
                assert_occlusion_equal(got, want, "rtTraceOcclusion", segs)
                keys = ("rays", "boxTests", "triTests") + (("sphereTests",) if len(sc.spheres) <= 64 else ())
                assert not o_opts.get("countStats") or all(sg[k] == so[k] for k in keys), f"counters {sg} vs {so}"
                occlusion_cases += 1
            except Exception as e:
                bad += 1
                print(f"case seed {seed}: occlusion: {type(e).__name__}: {e}   options {o_opts}, no_cull {no_cull}, {len(sc.models)} models, {len(sc.spheres)} spheres", flush=True)
        if args.paths:
            prng = np.random.RandomState(seed + 11)
            rays = path_rays(sc, seed=seed + 11, n=args.query_rays)
            samples = int(prng.choice([1, 2, 3, 7]))
            p_opts = {k: v for k, v in opts.items() if k in ("tlas", "modelSkip", "extInstantiation", "countStats", "smemNodes", "pairOrder")}
            try:
                want, so = trace_batch(ORACLE_LIB, sc, {}, rays, False, samples=samples)
                got, sg = trace_batch(lib, sc, p_opts, rays, False, samples=samples)
                assert_radiance_equal(got, want, "rtTracePaths")
                keys = ("rays",) + (("boxTests", "triTests") + (("sphereTests",) if len(sc.spheres) <= 64 else ()) if p_opts.get("countStats") else ())
                assert all(sg[k] == so[k] for k in keys), f"counters {sg} vs {so}"
                path_cases += 1
            except Exception as e:
                bad += 1
                print(f"case seed {seed}: paths: {type(e).__name__}: {e}   options {p_opts}, samples {samples}, {len(sc.models)} models, {len(sc.spheres)} spheres", flush=True)
        if (case + 1) % 25 == 0:
            print(f"  {case + 1} cases, {bad} findings, {time.time() - t0:.0f} s", flush=True)
    print(f"{args.cases} cases, {bad} findings" + (f"; PixelStats compared in {pix_cases} cases" if args.pixel_stats else "")
          + (f"; query batches equal in {query_cases} cases" if args.queries else "")
          + (f"; occlusion batches equal in {occlusion_cases} cases" if args.occlusion else "")
          + (f"; path batches equal in {path_cases} cases" if args.paths else ""))
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
