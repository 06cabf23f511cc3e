#!/usr/bin/env python
"""Randomised SESSIONS on the SIMT interpreter build: not one frame of a scene but a sequence of host calls — frames, camera moves
(near, far, back), models that move / change material, Spheres buffers that shrink and grow across the accelerator's threshold,
resizes, accumulation resets, settings and kernel options that change between frames — driven identically through the host
manager against the oracle and against the kernels, compared bit for bit after every frame.  What it exercises is the host-side
state of csrc/rt_api.cu: dirty flags, cached repacks, the regions the padded boxes were built for, kernel selection.

    python tools/simt_fuzz_session.py [--cases 100] [--seed 1] [--steps 8] [--pixel-stats] [--frames] [--queries] [--adaptive]

--pixel-stats: both sides count from the start ("countStats" = 1, and the script's countStats switches reach the oracle too), and after
every frame the per-pixel counters (PixelStats rays, box and triangle tests) are compared as well: accumulation across frames, resizes,
partial state changes.

--frames: a step may render a batch of 2-6 frames as one call (RenderFrames: rtDispatchFrames) instead of one frame, on both sides.
Where the kernels' side refuses the batch because "sampleChunks" is forced to 2 or more, it renders the frames one by one instead.

--adaptive: a step may render an adaptive frame (RenderFrameAdaptive: rtDispatchAdaptive over the whole image) with a random threshold
and min / max frames, or an adaptive call over a random partial region at a random Frame straight on the context, on both sides; the
active counts, the images and "AdaptiveMoments" are compared after it, and refusals must agree.  Where the kernels' side would refuse
because "sampleChunks" is forced to 2 or more, the step renders a plain frame on both sides instead.

--queries: query steps anywhere in the script — before OnEnable, between a scene change and the next frame, right after a raw
dispatch, between frames: rtTraceRays, rtTraceOcclusion or rtTracePaths of 0, 1, 31, 32, 33 or a few hundred rays (the ray sets of
tests/test_gpu_trace_rays.py; for occlusion tMax at, one ulp below and above the oracle's closest hit and special values; for paths
random RNG states, 1-3 samples and the session's MaxBounceCount), through the manager, the context's host form or, on the kernels'
side, the context's device form (the oracle answers through the same host form).  The answers are compared bit for bit, then
RtStats.rays the batch added and, while the kernels' side counts, its traversal counters; dispatches and kernelMs must not move.  The
frames that follow compare the images as before, so a query that changed what a frame shows is found there.
"""
import argparse
import os
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tests"))
sys.path.insert(0, os.path.join(REPO, "tests", "simt"))
sys.path.insert(0, os.path.join(REPO, "tools"))
import build as simt_build                      # noqa: E402
from conftest import ORACLE_LIB                 # noqa: E402
import ray_tracing_b200 as rt                   # noqa: E402
from ray_tracing_b200 import capi, scenes       # noqa: E402
from simt_fuzz import random_material, random_scene   # noqa: E402
from test_gpu_trace_rays import assert_hits_equal, ray_sets      # noqa: E402
from test_gpu_occlusion import assert_occlusion_equal, tmax_sets  # noqa: E402
from test_gpu_trace_paths import assert_radiance_equal           # noqa: E402

QUERY_KINDS = ("trace_rays", "trace_occlusion", "trace_paths")
QUERY_FORMS = ("manager", "context", "device")


def random_query(rng):
    """('query', (kind, form, batch size, seed, no_cull, samples))"""
    n = int(rng.choice([0, 1, 31, 32, 33, int(rng.randint(100, 400))]))
    return ("query", (str(rng.choice(QUERY_KINDS)), str(rng.choice(QUERY_FORMS)), n, int(rng.randint(0, 2 ** 31 - 1)), bool(rng.rand() < 0.5),
                      int(rng.randint(1, 4))))


class DeviceMemory:
    """Buffers for the context's *_device forms: torch CUDA tensors for a CUDA build; for a build of tests/simt, whose device memory
    is host memory, numpy arrays."""

    def __init__(self, lib):
        self.torch = None
        if os.path.dirname(os.path.abspath(lib)) != os.path.abspath(simt_build.OUT_DIR):
            import torch
            self.torch = torch

    def call(self, ctx, fn, src, out_dtype, *extra):
        n = len(src)
        out = np.zeros(n, dtype=out_dtype)
        if self.torch is None:
            src = np.ascontiguousarray(src)
            getattr(ctx, fn)(src.ctypes.data, out.ctypes.data, n, *extra)
            ctx.synchronize()
            return out
        t = self.torch
        d_src = t.from_numpy(np.concatenate([src.view(np.uint8).ravel(), np.zeros(16, np.uint8)])).cuda()
        d_out = t.zeros(out.nbytes + 16, dtype=t.uint8, device="cuda")
        getattr(ctx, fn)(d_src.data_ptr(), d_out.data_ptr(), n, *extra)
        ctx.synchronize()
        return d_out.cpu().numpy()[:out.nbytes].view(out_dtype)


def query_batch(oracle, q, pool):
    """The rays, segments or path rays of query step q, drawn from the case's ray pool.  Segments take tMax from the oracle's closest
    hits in the scene as it stands, through the step's form (before either side reads its counters)."""
    kind, form, n, seed, no_cull, _ = q
    rng = np.random.RandomState(seed)
    rays = pool[rng.randint(0, len(pool), n)]
    if kind == "trace_occlusion":
        try:
            closest = (oracle if form == "manager" else oracle.context).trace_rays(rays, no_cull=no_cull)
        except rt.capi.RtError:                  # the query itself will be refused the same way: any tMax will do
            closest = np.zeros(n, dtype=capi.RAY_HIT_DTYPE)
            closest["dst"] = np.inf
        segs = np.concatenate(list(tmax_sets(rays, closest, seed=seed).values()))
        return segs[rng.permutation(len(segs))[:n]]
    if kind == "trace_paths":
        return capi.make_path_rays(rays["origin"], rays["dir"], rng.randint(0, 2 ** 32, size=n, dtype=np.uint64).astype(np.uint32))
    return rays


def run_query(mgr, q, arg, kernels_side, device):
    """One query step on one side: (answers, or the RT_E_* code of a refusal; RtStats before; RtStats after)."""
    kind, form, _, _, no_cull, samples = q
    ctx = mgr.context
    try:
        before = ctx.stats()
        if form == "device" and kernels_side:
            out_dtype = {"trace_rays": capi.RAY_HIT_DTYPE, "trace_occlusion": np.uint8, "trace_paths": capi.PATH_RADIANCE_DTYPE}[kind]
            extra = (samples,) if kind == "trace_paths" else (no_cull,)
            got = device.call(ctx, kind + "_device", arg, out_dtype, *extra)
            if kind == "trace_occlusion":
                got = got.view(np.bool_)
        else:
            target = mgr if form == "manager" else ctx
            got = getattr(target, kind)(arg, samples) if kind == "trace_paths" else getattr(target, kind)(arg, no_cull=no_cull)
        return got, before, ctx.stats()
    except rt.capi.RtError as e:
        return e.code, None, None


def compare_query(q, o, g, counting, spheres):
    """None, or what differs between the oracle's (o) and the kernels' (g) results of run_query."""
    kind = q[0]
    (wo, bo, ao), (wg, bg, ag) = o, g
    if isinstance(wo, int) or isinstance(wg, int):
        return None if (isinstance(wo, int) and isinstance(wg, int) and wo == wg) else f"{kind} refused on one side ({wo if isinstance(wo, int) else 'ok'} vs {wg if isinstance(wg, int) else 'ok'})"
    if len(wg) != len(wo):
        return f"{kind}: {len(wg)} answers vs the oracle's {len(wo)}"
    try:
        if len(wo):
            {"trace_rays": assert_hits_equal, "trace_occlusion": assert_occlusion_equal, "trace_paths": assert_radiance_equal}[kind](wg, wo, kind)
    except AssertionError as e:
        return str(e)
    keys = ("rays",) + (("boxTests", "triTests") + (("sphereTests",) if spheres <= 64 else ()) if counting else ())
    for k in keys:
        if ag[k] - bg[k] != ao[k] - bo[k]:
            return f"{kind}: RtStats.{k} grew by {ag[k] - bg[k]} vs the oracle's {ao[k] - bo[k]}"
    for side, b, a in (("kernels'", bg, ag), ("oracle's", bo, ao)):
        if a["dispatches"] != b["dispatches"] or a["kernelMs"] != b["kernelMs"]:
            return f"{kind} moved the {side} dispatches / kernelMs ({b['dispatches']}, {b['kernelMs']} -> {a['dispatches']}, {a['kernelMs']})"
    return None


def random_spheres(rng, n):
    sph = np.zeros(n, dtype=scenes.SPHERE_DTYPE)
    for i in range(n):
        sph[i] = scenes._sphere(tuple(rng.uniform(-2.5, 2.5, 3) + np.array([0, 2.0, 0])), float(np.exp(rng.uniform(np.log(0.02), np.log(0.6)))), random_material(rng))
    return sph


def random_adaptive(rng):
    """('adaptive', (threshold, minFrames, maxFrames)) or ('adaptive_partial', (threshold, minFrames, maxFrames, gx, gy, Frame))"""
    thr = float(rng.choice([0.0, 0.05, 0.2, 0.5, 1.0, float(rng.uniform(0, 2))]))
    mn = int(rng.randint(2, 6))
    mx = int(rng.choice([mn, mn + int(rng.randint(0, 6)), 1 << 24]))
    if rng.rand() < 0.3:
        return ("adaptive_partial", (thr, mn, mx, int(rng.randint(0, 9)), int(rng.randint(0, 6)), int(rng.randint(1, 1000))))
    return ("adaptive", (thr, mn, mx))


def make_script(rng, sc, steps, frames=False, queries=False, adaptive=False):
    """A list of (action, arguments) — applied to both managers; ('option', ...) only to the kernels' side.  frames: a step may end in
    ('frames', (n,)), a batch of n frames, instead of ('frame', ()).  queries: ('query', ...) steps (random_query) before OnEnable,
    among the scene changes, after raw dispatches and after frames."""
    script = [random_query(rng)] if queries and rng.rand() < 0.3 else []
    nm = len(sc.models)
    for _ in range(steps):
        for _ in range(int(rng.randint(0, 4))):
            a = int(rng.randint(0, 12 if queries else 11))
            if a == 11:
                script.append(random_query(rng))
            elif a == 10:
                # round 2: the ABI below the manager — modelCount set on its own (no ModelInfo re-send), then a dispatch
                script.append(("rawframe", (int(rng.randint(0, nm + 1)), int(rng.randint(1, 1000)))))
                if queries and rng.rand() < 0.5:
                    script.append(random_query(rng))
            elif a == 0:
                d = float(rng.choice([0.0, 3.0, 5.67, 60.0, 4000.0, 3e5]))
                script.append(("camera", (float(np.clip(np.degrees(2 * np.arctan(3.0 / max(d, 3.0))), 1e-3, 90.0)),
                                          scenes.trs(position=(float(rng.uniform(-1, 1)), 1.9, -d), euler_deg=(float(rng.uniform(-5, 5)), float(rng.uniform(-5, 5)), 0.0))[0])))
            elif a == 1 and nm:
                scale = np.exp(rng.uniform(np.log(0.02), np.log(1.2), 3))
                pos = tuple(rng.uniform(-2.5, 2.5, 3) * float(rng.choice([1.0, 1.0, 50.0])) + np.array([0, 2.0, 0]))
                script.append(("model", (int(rng.randint(0, nm)),) + scenes.trs(position=pos, euler_deg=tuple(rng.uniform(0, 360, 3)), scale=tuple(scale))))
            elif a == 2 and nm:
                script.append(("material", (int(rng.randint(0, nm)), random_material(rng))))
            elif a == 3:
                script.append(("spheres", (random_spheres(rng, int(rng.choice([0, 3, 64, 65, 150]))),)))
            elif a == 4:
                script.append(("screen", (int(rng.choice([8, 24, 40, 64])), int(rng.choice([6, 18, 36])))))
            elif a == 5:
                script.append(("reset", ()))
            elif a == 6:
                script.append(("setting", (str(rng.choice(["maxBounceCount", "numRaysPerPixel", "useSky", "accumulate", "divergeStrength", "defocusStrength"])), rng.rand())))
            else:
                name = str(rng.choice(["kernel", "tlas", "modelSkip", "poolSlots", "pairOrder", "smemNodes", "tailLanes", "sortRays", "gridFit", "extInstantiation", "countStats", "sampleChunks"]))
                value = {"kernel": [0, 1, 2, -1], "tlas": [-1, 0, 1], "modelSkip": [0, 1], "poolSlots": [0, 32, 64, 96], "pairOrder": [0, 1, 3], "smemNodes": [0, 9, 200, -1],
                         "tailLanes": [0, 5, 16, 31], "sortRays": [0, 1], "gridFit": [0, 1], "extInstantiation": [0, 1], "countStats": [0, 1], "sampleChunks": [-1, 0, 2, 3]}[name]
                script.append(("option", (name, int(rng.choice(value)))))
        if adaptive and rng.rand() < 0.6:
            script.append(random_adaptive(rng))
        elif frames and rng.rand() < 0.5:
            script.append(("frames", (int(rng.randint(2, 7)),)))
        else:
            script.append(("frame", ()))
        if queries and rng.rand() < 0.3:
            script.append(random_query(rng))
    return script


def apply(mgr, action, args, kernels_side, pixel_stats=False):
    if action == "camera":
        mgr.set_camera(*args)
    elif action == "model":
        mgr.set_model_transform(*args)
    elif action == "material":
        mgr.set_model_material(*args)
    elif action == "spheres":
        mgr.set_spheres(*args)
    elif action == "screen":
        mgr.set_screen(*args)
    elif action == "reset":
        mgr.ResetAccumulatedRender()
    elif action == "setting":
        name, u = args
        value = {"maxBounceCount": int(u * 7), "numRaysPerPixel": 1 + int(u * 3), "useSky": u < 0.5, "accumulate": u < 0.7,
                 "divergeStrength": float(u * 2), "defocusStrength": float(u < 0.3) * 30.0}[name]
        setattr(mgr, name, value)
    elif action == "option" and (kernels_side or (pixel_stats and args[0] == "countStats")):
        mgr.context.set_option(*args)


def read_pixel_stats(mgr):
    """The manager's PixelStats image, or the RT_E_* code when it has none (no counting frame yet)."""
    try:
        return mgr.pixel_stats()
    except rt.capi.RtError as e:
        return e.code


def run_adaptive(mgr, action, a):
    """One adaptive step on one side: the active count, or the RT_E_* code of a refusal."""
    try:
        if action == "adaptive":
            return mgr.RenderFrameAdaptive(*a)
        thr, mn, mx, gx, gy, frame = a
        mgr.context.set_int("Frame", frame)
        return mgr.context.dispatch_adaptive(thr, mn, mx, gx, gy, 1)
    except rt.capi.RtError as e:
        return e.code


def read_moments(mgr):
    try:
        return mgr.context.adaptive_moments()
    except rt.capi.RtError as e:
        return e.code


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", type=int, default=100)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--lib", default=None)
    ap.add_argument("--pixel-stats", action="store_true", help="also compare the per-pixel counters after every frame")
    ap.add_argument("--frames", action="store_true", help="steps may render a batch of 2-6 frames in one call (RenderFrames)")
    ap.add_argument("--queries", action="store_true", help="query steps (rtTraceRays / rtTraceOcclusion / rtTracePaths) anywhere in the script")
    ap.add_argument("--adaptive", action="store_true", help="steps may render an adaptive frame (RenderFrameAdaptive / rtDispatchAdaptive)")
    args = ap.parse_args()
    lib = args.lib or simt_build.build()
    device = DeviceMemory(lib) if args.queries else None
    bad, query_steps, adaptive_steps = 0, {k: 0 for k in QUERY_KINDS + QUERY_FORMS}, 0
    for case in range(args.cases):
        seed = args.seed * 100003 + case
        rng = np.random.RandomState(seed)
        sc = random_scene(rng, odd=0.0)
        script = make_script(rng, sc, args.steps, args.frames, args.queries, args.adaptive)
        pool = np.concatenate(list(ray_sets(sc, seed=seed, n=48).values())) if args.queries else None
        mgrs = []
        for backend in (ORACLE_LIB, lib):
            m = rt.RayComputeManager(backend)
            scenes.apply(sc, m)
            if args.pixel_stats:
                m.context.set_option("countStats", 1)
            mgrs.append(m)
        frame_no, failed, resized, chunks, enabled = 0, None, False, -1, False
        counting, spheres = args.pixel_stats, len(sc.spheres)          # the kernels' side's countStats; the Spheres buffer's length
        try:
            for action, a in script:
                if action != "query" and not enabled:
                    for m in mgrs:
                        m.OnEnable()
                    enabled = True
                if action == "query":
                    batch = query_batch(mgrs[0], a, pool)
                    o, g = (run_query(m, a, batch, i == 1, device) for i, m in enumerate(mgrs))
                    failed = compare_query(a, o, g, counting, spheres)
                    if failed:
                        failed = f"query {a[:3]} after {frame_no} frames: {failed}"
                        break
                    query_steps[a[0]] += 1
                    query_steps[a[1]] += 1
                    continue
                if action == "option" and a[0] == "countStats":
                    counting = bool(a[1])
                if action == "spheres":
                    spheres = len(a[0])
                if action == "screen":
                    resized = True                      # the textures follow at the next RenderFrame (InitFrame): no raw dispatch in between
                if action in ("rawframe", "adaptive_partial") and resized:
                    continue
                if action in ("adaptive", "adaptive_partial") and chunks >= 2:
                    action = "frame"                    # refused on the kernels' side only (a pixel list runs whole pixels)
                if action in ("frame", "frames", "adaptive"):
                    resized = False
                if action == "option" and a[0] == "sampleChunks":
                    chunks = a[1]
                if action in ("adaptive", "adaptive_partial"):
                    counts = [run_adaptive(m, action, a) for m in mgrs]
                    frame_no += 1
                    if counts[0] != counts[1]:
                        failed = f"{action} {a} after {frame_no - 1} frames: {counts[1]} vs the oracle's {counts[0]}"
                        break
                    adaptive_steps += 1
                    mo, mg = (read_moments(m) for m in mgrs)
                    if isinstance(mo, int) or isinstance(mg, int):
                        if not (isinstance(mo, int) and isinstance(mg, int) and mo == mg):
                            failed = f"AdaptiveMoments readable on one side only after {action} {a}"
                            break
                    elif mo.shape != mg.shape or ((mo.view(np.uint32) != mg.view(np.uint32)) & ~(np.isnan(mo) & np.isnan(mg))).any():
                        failed = f"AdaptiveMoments differ after {action} {a}"
                        break
                if action in ("frame", "frames", "rawframe", "adaptive", "adaptive_partial"):
                    for i, m in enumerate(mgrs):
                        if action in ("adaptive", "adaptive_partial"):
                            pass
                        elif action == "frame":
                            m.RenderFrame()
                        elif action == "frames":
                            try:
                                m.RenderFrames(a[0])
                            except rt.capi.RtError as e:
                                # a batch runs whole pixels: refused on the kernels' side while sampleChunks is forced to 2 or more
                                if not (i == 1 and chunks >= 2 and e.code == rt.capi.RT_E_STATE):
                                    raise
                                for _ in range(a[0]):
                                    m.RenderFrame()
                        else:
                            m.context.set_int("modelCount", a[0]); m.context.set_int("Frame", a[1]); m.context.dispatch_full(0)
                    frame_no += 1
                    for what in ("accumulatedResult", "raytraceFrameTex"):
                        x, y = getattr(mgrs[1], what), getattr(mgrs[0], what)
                        diff = (x.view(np.uint32) != y.view(np.uint32)) & ~(np.isnan(x) & np.isnan(y))
                        if x.shape != y.shape or diff.any():
                            failed = f"{what} differs after frame {frame_no} ({int(diff.sum()) if x.shape == y.shape else 'shape'})"
                            break
                    if not failed and args.pixel_stats:
                        # before the first counting frame (the script may switch counting off at once) both sides answer RT_E_STATE
                        got = [read_pixel_stats(m) for m in mgrs]
                        po, pg = got
                        if isinstance(po, int) or isinstance(pg, int):
                            if po != pg:
                                failed = f"PixelStats readable on one side only after frame {frame_no} ({po if isinstance(po, int) else 'ok'} vs {pg if isinstance(pg, int) else 'ok'})"
                        else:
                            bad_fields = [k for k in ("rays", "boxTests", "triTests") if po.shape != pg.shape or not np.array_equal(po[k], pg[k])]
                            if bad_fields:
                                failed = f"PixelStats {bad_fields} differ after frame {frame_no}"
                    if failed:
                        break
                else:
                    apply(mgrs[0], action, a, False, args.pixel_stats)
                    apply(mgrs[1], action, a, True, args.pixel_stats)
        except Exception as e:
            failed = f"{type(e).__name__}: {e}"
        for m in mgrs:
            m.OnDestroy()
        if failed:
            bad += 1
            brief = [(act, a if act in ("option", "setting", "screen", "query", "adaptive", "adaptive_partial") else "...") for act, a in script]
            print(f"case seed {seed}: {failed}; {len(sc.models)} models, {len(sc.spheres)} spheres; script {brief}", flush=True)
        if (case + 1) % 25 == 0:
            print(f"  {case + 1} cases, {bad} findings", flush=True)
    print(f"{args.cases} cases, {bad} findings" + (f"; adaptive steps equal: {adaptive_steps}" if args.adaptive else "") +
          (f"; query steps equal: {sum(query_steps[k] for k in QUERY_KINDS)} (" + ", ".join(f"{k} {v}" for k, v in query_steps.items()) + ")" if args.queries else ""))
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
