"""Traversal stacks where they wrap, spill and fill, checked bit for bit against the oracle.

The pooled kernel (kernel 2) keeps the top RT_SMEM_STACK = 8 entries of a lane's traversal stack in a shared-memory ring and spills
deeper ones to a local array; its 96-slot pools, the wave / mega / query kernels and the sphere and TLAS walks keep stacks of their
own.  The scenes of the other tests rarely hold more than a few pending entries, so the code past a ring boundary could be wrong
without any image changing.  The trees here are built to make it run:

- combs: every inner node's next inner child is entered before its leaf child by rays along the view axis, so each level pushes
  one entry and a ray holds as many pending entries as the comb has levels (7 .. 63, on and around every ring wrap and the cap);
- a line of thin triangles along the view axis, through the host builder, for deep stacks in a real builder's layout;
- several deep combs in one scene, with and without the sphere accelerator ("model -1"), for stack state across models;
- spheres whose radii grow along a line, so that the accelerator's surface-area levels peel one sphere per level.

The bodies take any library with the C-ABI; this file runs them on the SIMT interpreter build (tests/simt), and
tests/test_gpu_traversal_stacks.py on librt_b200.so.  The profile build of the interpreter proves the scenes reach the paths
they are meant for (push depths past 8, 16 and 31, ring spills, reloads from the local array)."""
import ctypes as C
import os
import sys
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from conftest import ORACLE_LIB, REPO, assert_bit_equal
import ray_tracing_b200 as rt
from ray_tracing_b200 import capi, scenes
from ray_tracing_b200.capi import NODE_DTYPE, TRIANGLE_DTYPE

sys.path.insert(0, os.path.join(REPO, "tests", "simt"))
import build as simt_build   # noqa: E402

COMB_DEPTHS = (7, 8, 9, 15, 16, 17, 31, 32, 33, 63)
COUNTERS = ("rays", "boxTests", "triTests", "sphereTests")


def counters_of(sc):
    """The counters that must equal the oracle's: with more than 64 spheres the kernels test the spheres the accelerator reaches and
    the oracle scans them all, so sphere tests are not comparable there."""
    return COUNTERS if len(sc.spheres) <= 64 else COUNTERS[:3]


# ---- trees ------------------------------------------------------------------------------------------------------------------------

def _tri(a, b, c, facing_camera):
    """One Triangles record; the camera looks along +z, so a front face has a winding whose normal points to -z."""
    t = np.zeros(1, dtype=TRIANGLE_DTYPE)
    if not facing_camera:
        b, c = c, b
    t["posA"], t["posB"], t["posC"] = a, b, c
    t["normA"] = t["normB"] = t["normC"] = (0.0, 0.0, -1.0 if facing_camera else 1.0)
    return t


def comb(depth, front=False, offsets=False, swap=False, twigs=False, z0=2.0, dz=0.05):
    """A comb of `depth` inner levels.  Level l has a far child (triangles in the plane z = z0 + (depth - l) * dz) and, as its near
    child, the next inner level; the last level's two children are leaves.  The deeper a level the closer its plane, so for rays along
    +z the inner child's box is entered strictly before the far child's: every level pushes its far child and descends.

    A far child is a leaf with a large triangle covering the view: back-facing (culled for opaque models, so nothing is hit and the
    stack fills and unwinds completely) or, with `front`, facing the camera.  `offsets` adds to every leaf a small front-facing
    triangle at its own place in the view, so pixels find their first hit at different levels.  With `twigs` the far child is instead
    an inner node over two upright slivers left and right of the view axis, and the bottom leaf faces away: rays enter a twig's box but
    mostly miss both children, so the inner step itself pops — past the ring, from the spilled entries — until a ray meets its sliver.  `swap` stores the far child as child B on odd levels.
    Returns (Triangles, Nodes) in the reference's layout (children of node i at startIndex and startIndex + 1)."""
    tris = []

    def leaf(*ts):
        first = len(tris)
        tris.extend(ts)
        return ("leaf", first, len(ts))

    levels = []
    for l in range(depth + 1):
        z = z0 + (depth - l) * dz
        if twigs and l < depth:
            # two upright slivers at directions of their own per level: a ray finds its first hit at some level, and the twigs it
            # passes on the way up are entered but both their children missed
            xl, xr, w = (0.1 + 0.6 * ((l * 0.618034) % 1.0)) * z, (0.1 + 0.6 * ((l * 0.414214) % 1.0)) * z, 0.03 * z
            far = ("inner", leaf(_tri((-xl - w, -4.0, z), (-xl, 4.0, z), (-xl + w, -4.0, z), front)),
                   leaf(_tri((xr - w, -4.0, z), (xr, 4.0, z), (xr + w, -4.0, z), front)))
        else:
            ts = [_tri((-12.0, -4.0, z), (0.0, 12.0, z), (12.0, -4.0, z), front and not twigs)]
            if offsets:
                ang = 2.399963 * l                               # golden-angle spiral: every level owns a patch of the image
                r = 0.15 + 1.1 * (l / max(depth, 1)) ** 0.5
                cx, cy = r * np.cos(ang) * z / 3.0, r * np.sin(ang) * z / 3.0
                sz = 0.22 * z / 3.0
                ts.append(_tri((cx - sz, cy - sz, z), (cx, cy + sz, z), (cx + sz, cy - sz, z), True))
            far = leaf(*ts)
        levels.append(far)
    node = levels[depth]
    for l in range(depth - 1, -1, -1):
        node = ("inner", node, levels[l]) if (swap and l % 2) else ("inner", levels[l], node)
    tris = np.concatenate(tris)
    lo = np.minimum(np.minimum(tris["posA"], tris["posB"]), tris["posC"])
    hi = np.maximum(np.maximum(tris["posA"], tris["posB"]), tris["posC"])
    nodes = np.zeros(2 * len(tris) + 1, dtype=NODE_DTYPE)
    used, work = 1, [(node, 0)]
    while work:
        (n, i) = work.pop()
        if n[0] == "leaf":
            nodes["startIndex"][i], nodes["triangleCount"][i] = n[1], n[2]
            rng_ = slice(n[1], n[1] + n[2])
            nodes["boundsMin"][i], nodes["boundsMax"][i] = lo[rng_].min(axis=0), hi[rng_].max(axis=0)
        else:
            nodes["startIndex"][i], nodes["triangleCount"][i] = used, 0
            work += [(n[1], used), (n[2], used + 1)]
            used += 2
    for i in range(used - 1, -1, -1):                            # inner bounds from the children (children sit after their parent)
        if nodes["triangleCount"][i] == 0:
            c = nodes["startIndex"][i]
            nodes["boundsMin"][i] = np.minimum(nodes["boundsMin"][c], nodes["boundsMin"][c + 1])
            nodes["boundsMax"][i] = np.maximum(nodes["boundsMax"][c], nodes["boundsMax"][c + 1])
    return tris, nodes[:used]


def line_mesh(k, dz=1e-4, z0=2.0):
    """2^k thin back-facing triangles, one behind the other along the view axis, as a mesh for the host builder."""
    n = 1 << k
    z = (z0 + dz * np.arange(n)).astype(np.float32)
    w = 0.05
    v = np.zeros((n, 3, 3), np.float32)
    v[:, 0] = np.stack([np.full(n, -w), np.full(n, -w), z], 1)
    v[:, 1] = np.stack([np.full(n, w), np.full(n, -w), z], 1)      # (A, C, B) order of _tri: normal along +z, a back face
    v[:, 2] = np.stack([np.zeros(n), np.full(n, w), z], 1)
    return scenes.MeshDesc(v.reshape(-1, 3), np.arange(3 * n, dtype=np.int32), np.tile(np.float32([0, 0, 1]), (3 * n, 1)))


def peel_spheres(n_line=24, n_cluster=48):
    """Spheres whose radii double along +z, then a cluster of small equal ones: the surface-area sweep splits the largest spheres off
    first, so the tree is about twice as deep as a balanced one and a ray along the line holds many pending entries.  Returns a Spheres
    buffer."""
    out = []
    mat = scenes.material(diffuse=(0.7, 0.6, 0.5))
    glass = scenes.material(diffuse=(1, 1, 1), flag=scenes.MAT_GLASS, ior=1.3)
    z, r = 3.0, 0.004
    for i in range(n_line):
        z += r
        out.append(scenes._sphere((0.0, 0.0, z), r, glass if i % 5 == 3 else mat))
        z += r
        r *= 2.0
    rng = np.random.RandomState(3)
    for i in range(n_cluster):
        c = (rng.uniform(-0.4, 0.4), rng.uniform(-0.4, 0.4), rng.uniform(1.5, 2.5))
        out.append(scenes._sphere(c, 0.03, mat))
    return np.stack(out)


# ---- scenes -----------------------------------------------------------------------------------------------------------------------

OPAQUE = scenes.material(diffuse=(0.8, 0.5, 0.3), emission=(1, 1, 1), emissionStrength=0.3)
GLASS = scenes.material(diffuse=(1, 1, 1), flag=scenes.MAT_GLASS, ior=1.45)


def comb_scene(tris, width, height, materials=(OPAQUE,), offsets=((0, 0, 0),), spheres=None, bounces=3, spp=1):
    """A scene whose models all use one mesh made of `tris` (the Nodes / Triangles buffers are replaced after OnEnable)."""
    v = np.concatenate([tris["posA"], tris["posB"], tris["posC"]], axis=1).reshape(-1, 3).astype(np.float32)
    nrm = np.concatenate([tris["normA"], tris["normB"], tris["normC"]], axis=1).reshape(-1, 3).astype(np.float32)
    mesh = scenes.MeshDesc(v, np.arange(v.shape[0], dtype=np.int32), nrm)
    models = []
    for mat, off in zip(materials, offsets):
        l2w, w2l = scenes.trs(position=off)
        models.append(scenes.ModelDesc(0, l2w, w2l, mat))
    sc = scenes.Scene(name=f"comb of {len(tris)} triangles x {len(models)}", width=width, height=height, meshes=[mesh], models=models,
                      settings=dict(maxBounceCount=bounces, numRaysPerPixel=spp, useSky=True, divergeStrength=0.3))
    if spheres is not None:
        sc.spheres = spheres
    return sc


def sphere_grid(n_side=9, z=8.0):
    """n_side^2 small spheres behind the combs: with more than 64 spheres every ray walks the sphere accelerator first."""
    out = []
    for i in range(n_side):
        for j in range(n_side):
            mat = scenes.material(diffuse=(0.3, 0.6, 0.9), emission=(1, 1, 1), emissionStrength=float((i + j) % 3 == 0))
            out.append(scenes._sphere((-3.0 + 6.0 * i / (n_side - 1), -3.0 + 6.0 * j / (n_side - 1), z + 0.1 * i), 0.3, mat))
    return np.stack(out)


def open_scene(lib, sc, tree=None, options=None):
    mgr = rt.RayComputeManager(lib)
    scenes.apply(sc, mgr)
    ctx = mgr.context
    for k, v in (options or {}).items():
        ctx.set_option(k, v)
    mgr.OnEnable()
    if tree is not None:
        ctx.set_buffer("Triangles", tree[0])
        ctx.set_int("triangleCount", len(tree[0]))
        ctx.set_buffer("Nodes", tree[1])
    return mgr


def render_tree(lib, sc, tree=None, options=None, frames=1, batch=False):
    """(FrameRender, AccumulatedRender, stats) after `frames` frames: RenderFrame calls, or with `batch` one rtDispatchFrames."""
    mgr = open_scene(lib, sc, tree, options)
    ctx = mgr.context
    ctx.reset_stats()
    if batch:
        mgr.RenderFrames(frames)
    else:
        for _ in range(frames):
            mgr.RenderFrame()
    out = (mgr.raytraceFrameTex, mgr.accumulatedResult, ctx.stats())
    mgr.OnDestroy()
    return out


def check_against_oracle(lib, sc, tree, option_sets, frames=1, batch=False):
    fo, ao, so = render_tree(ORACLE_LIB, sc, tree, frames=frames)
    for opts in option_sets:
        fg, ag, sg = render_tree(lib, sc, tree, opts, frames=frames, batch=batch)
        what = f"{sc.name} {opts}{' batch' if batch else ''}"
        assert_bit_equal(fg, fo, what + ": FrameRender")
        assert_bit_equal(ag, ao, what + ": AccumulatedRender")
        assert sg["rays"] == so["rays"], what
        if opts.get("countStats"):
            keys = counters_of(sc)
            assert {k: sg[k] for k in keys} == {k: so[k] for k in keys}, what
    return so


def stack_options(kernels=(0, 1, 2)):
    """Every stack implementation of the kernels: wave / mega stacks, the pooled kernel with its ring (32 and 64 slots) and without
    (96 slots), both queue orders, with and without the counters."""
    out = []
    for k in kernels:
        out += [{"kernel": k}, {"kernel": k, "countStats": 1}]
        if k == 2:
            out += [{"kernel": 2, "poolSlots": 96}, {"kernel": 2, "poolSlots": 96, "countStats": 1, "sortRays": 1},
                    {"kernel": 2, "poolSlots": 64, "sortRays": 1}, {"kernel": 2, "poolSlots": 32, "tailLanes": 31, "countStats": 1}]
    return out


# ---- bodies shared with the GPU file ----------------------------------------------------------------------------------------------

def combs_equal_oracle(lib, depths=COMB_DEPTHS, size=(20, 12), options=None):
    """Back-facing (nothing hit: fill and full unwind), offset front-facing (first hits at every level) and glass combs (no culling,
    refracted rays walk the other way), at every depth around the ring wraps and the 64-entry cap."""
    for depth in depths:
        for kind, tree, mats in (("back", comb(depth), (OPAQUE,)),
                                 ("offsets", comb(depth, offsets=True, swap=True), (OPAQUE,)),
                                 ("glass", comb(depth, front=True, swap=True), (GLASS,)),
                                 ("twig", comb(min(depth, 62), front=True, twigs=True, swap=True), (OPAQUE,))):   # (+1 level: the twig)
            sc = comb_scene(tree[0], *size, materials=mats)
            sc.name = f"{kind} comb of depth {depth}"
            so = check_against_oracle(lib, sc, tree, options or stack_options())
            if kind != "twig":
                assert so["triTests"] >= so["rays"], sc.name               # the combs are really walked


def builder_lines_equal_oracle(lib, ks=(10, 11, 12, 13, 14, 15, 16), size=(9, 9)):
    """A line of 2^k back-facing triangles along the view axis through the host builder ("High"); the centre pixel's ray runs down
    the line without divergence, so it visits the whole tree."""
    for k in ks:
        m = line_mesh(k)
        l2w, w2l = scenes.trs()
        sc = scenes.Scene(name=f"line of 2^{k} triangles", width=size[0], height=size[1], meshes=[m],
                          models=[scenes.ModelDesc(0, l2w, w2l, OPAQUE)],
                          settings=dict(maxBounceCount=1, numRaysPerPixel=1, useSky=True, divergeStrength=0.0, bvhQuality=1))
        so = check_against_oracle(lib, sc, None, [{"kernel": 2, "countStats": 1}, {"kernel": 2, "poolSlots": 96, "countStats": 1},
                                                  {"kernel": 2}, {"kernel": 1, "countStats": 1}, {"kernel": 0, "countStats": 1}])
        assert so["triTests"] >= 1 << k, sc.name                           # one ray tested every triangle


def multi_model_scene(depth=40, spheres=False, size=(24, 16)):
    tree = comb(depth, front=True, offsets=True)
    sc = comb_scene(tree[0], *size, materials=(OPAQUE, GLASS, OPAQUE), offsets=((0, 0, 0), (0.3, 0.2, 0.6), (-0.2, 0.1, 1.2)),
                    spheres=sphere_grid() if spheres else None)
    sc.name = f"three combs of depth {depth}" + (" and 81 spheres" if spheres else "")
    return sc, comb(depth, offsets=True)


def stack_state_across_models(lib, size=(24, 16)):
    """Deep combs as consecutive models (and the sphere accelerator before them): a ray leaves each with its stack unwound, and
    whatever one model spilled must not reach the next.  Model skipping on and off, the TLAS forced on, frame batches."""
    for spheres in (False, True):
        sc, tree = multi_model_scene(spheres=spheres, size=size)
        opts = stack_options() + [{"kernel": 2, "modelSkip": 0}, {"kernel": 2, "modelSkip": 1, "tlas": 1},
                                  {"kernel": 2, "poolSlots": 96, "tlas": 1}, {"kernel": 1, "tlas": 1}, {"kernel": 0, "modelSkip": 0}]
        check_against_oracle(lib, sc, tree, opts, frames=2)
        check_against_oracle(lib, sc, tree, [{"kernel": 2}, {"kernel": 2, "tlas": 1}, {"kernel": 2, "poolSlots": 96, "countStats": 1},
                                             {"kernel": 1}], frames=3, batch=True)


def rays_down_the_comb(n=40, seed=1):
    """Rays from the camera's side along +z (a small cone) and from behind the comb along -z."""
    rng = np.random.RandomState(seed)
    d = np.column_stack([rng.uniform(-0.25, 0.25, n), rng.uniform(-0.25, 0.25, n), np.ones(n)])
    o = np.column_stack([rng.uniform(-0.3, 0.3, n), rng.uniform(-0.3, 0.3, n), rng.uniform(-1.0, 1.0, n)])
    d[: n // 4, 2] = -1.0
    o[: n // 4, 2] = 9.0
    d[n // 4] = (0, 0, 1)
    o[n // 4] = (0, 0, 0)
    d /= np.linalg.norm(d, axis=1)[:, None]
    return o.astype(np.float32), d.astype(np.float32)


def _hits_equal(a, b, what):
    for f in ("dst", "pos", "normal"):
        assert_bit_equal(np.ascontiguousarray(a[f]), np.ascontiguousarray(b[f]), f"{what}: {f}")
    for f in ("isBackface", "kind", "index"):
        assert np.array_equal(a[f], b[f]), f"{what}: {f}"


def queries_down_the_comb(lib, depths=(8, 9, 17, 33, 63)):
    """rtTraceRays, rtTraceOcclusion with tMax just before, at and after the closest triangle (the bottom of the tree), and
    rtTracePaths, all with rays aimed down deep combs; the counters must be the oracle's."""
    o, d = rays_down_the_comb()
    for depth in depths:
        for kind, tree, mats in (("back", comb(depth), (OPAQUE,)), ("front", comb(depth, front=True, offsets=True, swap=True), (OPAQUE,)),
                                 ("glass", comb(depth, front=True), (GLASS,))):
            sc = comb_scene(tree[0], 8, 8, materials=mats, spheres=sphere_grid() if depth == 33 else None)
            what = f"{kind} comb of depth {depth}"
            res = {}
            for path in (ORACLE_LIB, lib):
                for stats in (0, 1):
                    mgr = open_scene(path, sc, tree, {"countStats": stats})
                    ctx = mgr.context
                    ctx.reset_stats()
                    r = {"hits": {nc: ctx.trace_rays(o, d, no_cull=nc) for nc in (False, True)}}
                    closest = r["hits"][True]["dst"]
                    ok = np.isfinite(closest)
                    t = closest[ok]
                    segs = [(np.nextafter(t, np.float32(0)), "before"), (t, "at"), (np.nextafter(t, np.float32(np.inf)), "after")]
                    r["occ"] = {(nc, tag): ctx.trace_occlusion(capi.make_segments(o[ok], d[ok], tm), no_cull=nc)
                                for tag_t in segs for tm, tag in (tag_t,) for nc in (False, True)}
                    r["paths"] = ctx.trace_paths(capi.make_path_rays(o, d, np.arange(1, len(o) + 1, dtype=np.uint32)), samples=2)
                    r["stats"] = ctx.stats()
                    res[(path, stats)] = r
                    mgr.OnDestroy()
            for stats in (0, 1):
                ref, got = res[(ORACLE_LIB, stats)], res[(lib, stats)]
                for nc in (False, True):
                    _hits_equal(got["hits"][nc], ref["hits"][nc], f"{what} trace_rays no_cull={nc}")
                for key in ref["occ"]:
                    assert np.array_equal(got["occ"][key], ref["occ"][key]), f"{what} occlusion {key}"
                assert_bit_equal(got["paths"]["rgb"], ref["paths"]["rgb"], f"{what} trace_paths")
                assert np.array_equal(got["paths"]["rngState"], ref["paths"]["rngState"]), what
                keys = counters_of(sc) if stats else ("rays",)
                assert {k: got["stats"][k] for k in keys} == {k: ref["stats"][k] for k in keys}, (what, stats)
            ref = res[(ORACLE_LIB, 0)]
            if kind != "back":
                assert not ref["occ"][(True, "before")].any() and ref["occ"][(True, "after")].any(), what      # tMax straddles the hits


def peeled_sphere_line(lib):
    """The sphere accelerator over spheres whose radii double along a line, rays aimed along the line: against the oracle's scan."""
    sp = peel_spheres()
    sc = scenes.Scene(name="peeled sphere line", width=12, height=12, spheres=sp,
                      settings=dict(maxBounceCount=3, numRaysPerPixel=1, useSky=True, divergeStrength=0.3))
    sc.fov = 20.0
    check_against_oracle(lib, sc, None, stack_options())
    o, d = rays_down_the_comb(n=48, seed=7)
    res = {}
    for path in (ORACLE_LIB, lib):
        for stats in (0, 1):
            mgr = open_scene(path, sc, None, {"countStats": stats})
            ctx = mgr.context
            ctx.reset_stats()
            res[(path, stats)] = (ctx.trace_rays(o, d), ctx.trace_occlusion(capi.make_segments(o, d, np.full(len(o), 50.0, np.float32))),
                                  ctx.stats())
            mgr.OnDestroy()
    for stats in (0, 1):
        (ho, oo, so), (hg, og, sg) = res[(ORACLE_LIB, stats)], res[(lib, stats)]
        _hits_equal(hg, ho, "peeled sphere line: trace_rays")
        assert np.array_equal(og, oo), "peeled sphere line: occlusion"
        keys = counters_of(sc) if stats else ("rays",)
        assert {k: sg[k] for k in keys} == {k: so[k] for k in keys}
    assert np.isfinite(res[(ORACLE_LIB, 0)][0]["dst"]).sum() > len(o) // 2


# ---- host-side trees (device-free hooks of the library) ---------------------------------------------------------------------------

PAIR_DTYPE = np.dtype([("aMin", "<f4", 3), ("aMax", "<f4", 3), ("aStart", "<i4"), ("aCount", "<i4"),
                       ("bMin", "<f4", 3), ("bMax", "<f4", 3), ("bStart", "<i4"), ("bCount", "<i4")])


def _tree_depth(pairs, root):
    """Inner nodes on the longest root-to-leaf path (the most entries a walk that pushes one child per inner node can hold)."""
    best, work = 0, [((int(root[0]), int(root[1])), 0)]
    while work:
        (start, count), depth = work.pop()
        if count > 0:
            best = max(best, depth)
            continue
        p = pairs[start]
        work.append(((int(p["aStart"]), int(p["aCount"])), depth + 1))
        work.append(((int(p["bStart"]), int(p["bCount"])), depth + 1))
    return best


def plan_spheres(lib, sp):
    """The accelerator's tree as an upload builds it, for ray origins anywhere between the camera (at 0) and the spheres."""
    L = C.CDLL(lib)
    n = len(sp)
    arr = np.ascontiguousarray(np.column_stack([sp["centre"], sp["radius"]]), dtype=np.float32)
    r = np.abs(sp["radius"])[:, None]
    box = np.ascontiguousarray(np.concatenate([np.minimum(0, (sp["centre"] - r).min(0)), np.maximum(0, (sp["centre"] + r).max(0))]), dtype=np.float32)
    pairs = np.zeros(max(n, 1), dtype=PAIR_DTYPE)
    leaves = np.zeros(n, np.int32)
    root = np.zeros(2, np.int32)
    L.rtxPlanSpheres.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    k = L.rtxPlanSpheres(arr.ctypes.data, n, box.ctypes.data, pairs.ctypes.data, len(pairs), leaves.ctypes.data, root.ctypes.data)
    assert k >= 0
    return pairs[:k], leaves, root


def tree_stack_limits(lib, which, n):
    L = C.CDLL(lib)
    L.rtxTreeStackLimits.argtypes = [C.c_int, C.c_longlong, C.c_void_p, C.c_void_p, C.c_void_p]
    sah, bound, stack = C.c_int(), C.c_int(), C.c_int()
    rc = L.rtxTreeStackLimits(which, n, C.byref(sah), C.byref(bound), C.byref(stack))
    return rc, sah.value, bound.value, stack.value


# ---- on the SIMT build ------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="session")
def simt_lib():
    return simt_build.build()


VARIANTS = {"ring4": ("RT_SMEM_STACK=4",), "ring16": ("RT_SMEM_STACK=16",), "stacktop": ("RT_STACK_TOP_REG",), "profile": ("RT_SIMT_PROFILE",)}


@pytest.fixture(scope="session")
def simt_variants(tmp_path_factory):
    """The compile-time stack variants and the profile build, compiled side by side (about a minute each)."""
    d = tmp_path_factory.mktemp("stack_variants")
    with ThreadPoolExecutor(len(VARIANTS)) as ex:
        futs = {name: ex.submit(simt_build.build, True, defs, str(d / f"{name}.so")) for name, defs in VARIANTS.items()}
        return {name: f.result() for name, f in futs.items()}


@pytest.mark.parametrize("depth", COMB_DEPTHS)
def test_simt_combs_equal_oracle(simt_lib, depth):
    combs_equal_oracle(simt_lib, depths=(depth,))


def test_simt_builder_made_lines_equal_oracle(simt_lib):
    builder_lines_equal_oracle(simt_lib, ks=(10, 12, 14, 16))


def test_simt_stack_state_across_models(simt_lib):
    stack_state_across_models(simt_lib)


def test_simt_stack_state_across_shade_phases(simt_lib, monkeypatch):
    """One 'SM' and 32-slot pools: the 40 x 24 image needs refills, and with 31 tail lanes deep rays stay in flight, mid-walk, while
    their warp shades and refills."""
    monkeypatch.setenv("RT_SIMT_SMS", "1")
    sc, tree = multi_model_scene(depth=33, spheres=True, size=(40, 24))
    check_against_oracle(simt_lib, sc, tree, [{"kernel": 2, "poolSlots": 32, "tailLanes": 31}, {"kernel": 2, "poolSlots": 32, "tailLanes": 31, "countStats": 1},
                                              {"kernel": 2, "poolSlots": 96, "tailLanes": 16, "sortRays": 1}])


def test_simt_queries_down_the_comb(simt_lib):
    queries_down_the_comb(simt_lib)


def test_simt_peeled_sphere_line(simt_lib):
    peeled_sphere_line(simt_lib)


@pytest.mark.parametrize("variant", ["ring4", "ring16", "stacktop"])
def test_simt_stack_variants_on_deep_combs(simt_variants, variant):
    """RT_SMEM_STACK = 4 and 16 move the ring boundary; RT_STACK_TOP_REG replaces the ring by a register top."""
    lib = simt_variants[variant]
    # (a 16-entry ring leaves shared memory for 32-slot pools only)
    slots = 32 if variant == "ring16" else 64
    opts = [{"kernel": 2, "poolSlots": slots}, {"kernel": 2, "poolSlots": slots, "countStats": 1}, {"kernel": 2, "poolSlots": 96},
            {"kernel": 2, "poolSlots": slots, "sortRays": 1, "tailLanes": 31}]
    combs_equal_oracle(lib, depths=(3, 4, 5, 8, 15, 16, 17, 63), options=opts)
    sc, tree = multi_model_scene(spheres=True)
    check_against_oracle(lib, sc, tree, opts + [{"kernel": 2, "poolSlots": slots, "tlas": 1}])


def test_simt_profile_shows_the_scenes_reach_deep_stacks(simt_variants):
    """Coverage of the scenes above, on the profile build: pushes at depths past 8, 16 and into the saturated bucket 31, spills of the
    ring's oldest entry to the local array (slot 28), pops that reload from it (slot 29) and among them the inner step's branchless pop
    (slot 30, reached by the twig comb) — in the ring path of 64-slot pools
    (predicated push, branchless pop) and in the local-only 96-slot path (histogram only)."""
    lib = simt_variants["profile"]
    L = C.CDLL(lib)
    prof = (C.c_ulonglong * 64).in_dll(L, "simtProf")
    cases = [(comb_scene(comb(63)[0], 8, 6), comb(63)), (comb_scene(comb(17, offsets=True)[0], 8, 6), comb(17, offsets=True)),
             (comb_scene(comb(33, front=True, twigs=True)[0], 8, 6), comb(33, front=True, twigs=True))]
    sc, tree = multi_model_scene(spheres=True, size=(8, 6))
    cases.append((sc, tree))
    for slots in (64, 96):
        for i_case, (sc, tree) in enumerate(cases):
            for i in range(64):
                prof[i] = 0
            fo, ao, _ = render_tree(ORACLE_LIB, sc, tree)
            fg, ag, _ = render_tree(lib, sc, tree, {"kernel": 2, "poolSlots": slots})
            assert_bit_equal(ag, ao, f"profile build {sc.name} {slots}")
            p = [int(prof[i]) for i in range(64)]
            hist = p[32:64]                                                  # pushes by the depth they reached (31: 31 or more)
            what = (sc.name, slots, hist)
            assert sum(hist) == p[11] > 0, what
            assert any(hist[9:]) and any(hist[17:]), what
            if i_case == 0:
                assert hist[31] > 0, what
            if slots == 64:
                assert p[28] > 0 and p[29] > 0, (sc.name, "ring spills / reloads", p[28], p[29])
                if i_case == 2:
                    assert p[30] > 0, (sc.name, "reloads of the inner step's pop", p[30])
            else:
                assert p[28] == 0 and p[29] == 0, (sc.name, "96-slot pools have no ring")


def test_sphere_tree_depth_fits_the_walks(simt_lib):
    """The deepest sphere tree the host builds for any sphere count the API accepts (up to 2^31 - 1) fits TraverseSpheres' stack;
    the surface-area levels give way to median levels where it would not.  And the bound is a bound: trees built for the peeled line
    and for a grid stay within it."""
    for n in (65, 1000, 1 << 20, 1 << 27, (1 << 27) + 1, 1 << 28, (1 << 31) - 1):
        rc, sah, bound, stack = tree_stack_limits(simt_lib, 0, n)
        assert rc == 0 and stack == 48, n
        assert bound <= stack, (n, sah, bound)
        assert sah == (20 if n <= 1 << 27 else 47 - int(np.ceil(np.log2(n)))), (n, sah)
    for sp in (peel_spheres(), peel_spheres(40, 200), sphere_grid(12)):
        pairs, leaves, root = plan_spheres(simt_lib, sp)
        assert sorted(leaves.tolist()) == list(range(len(sp)))
        depth = _tree_depth(pairs, root)
        assert depth <= tree_stack_limits(simt_lib, 0, len(sp))[2], (len(sp), depth)
    # the surface-area levels split the line's largest spheres off one or a few at a time: twice as deep as a balanced tree
    sp = peel_spheres()
    assert _tree_depth(*plan_spheres(simt_lib, sp)[::2]) >= 2 * int(np.ceil(np.log2(len(sp))))


def test_tlas_depth_fits_the_walk(simt_lib):
    """The TLAS over up to 4096 models fits the 24-entry stack of TlasCollect, for every model count and for a line of models whose
    boxes grow geometrically (surface-area levels that peel one leaf at a time)."""
    for n in (1, 4, 5, 128, 129, 1000, 4096):
        rc, sah, bound, stack = tree_stack_limits(simt_lib, 1, n)
        assert rc == 0 and stack == 24 and sah == 10 and bound <= stack, (n, bound)
    assert tree_stack_limits(simt_lib, 1, 4097)[0] != 0
    L = C.CDLL(simt_lib)
    n = 4096
    z = np.cumsum(1.02 ** np.arange(n))
    h = 0.5 * 1.02 ** np.arange(n)
    boxes = np.column_stack([-h, -h, z - h, h, h, z + h]).astype(np.float32)
    pairs = np.zeros(n, dtype=PAIR_DTYPE)
    leaves, root = np.zeros(n, np.int32), np.zeros(2, np.int32)
    L.rtxPlanTlas.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    k = L.rtxPlanTlas(boxes.ctypes.data, n, pairs.ctypes.data, len(pairs), leaves.ctypes.data, root.ctypes.data)
    assert k > 0
    assert _tree_depth(pairs[:k], root) <= tree_stack_limits(simt_lib, 1, n)[2]
