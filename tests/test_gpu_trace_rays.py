"""rtTraceRays on the H100 (`-m gpu`): the closest hit of caller-supplied rays equals the oracle's CalculateRayCollision bit for bit —
dst, pos, normal, isBackface, the winner's kind and index, and with "countStats" the traversal counters — across scenes, ray sets
(pick rays, rays inside the scene, from inside meshes and spheres, far origins that take the linear fallback, mixed batches, special
values), both flags, model skipping on and off, the context states around it and the device-pointer form.  The same bodies run in the
CPU suite against the SIMT interpreter build (tests/test_simt_trace_rays.py)."""
import numpy as np
import pytest

from conftest import CUDA_LIB, ORACLE_LIB, assert_bit_equal
import ray_tracing_b200 as rt
from ray_tracing_b200 import capi, scenes

pytestmark = pytest.mark.gpu

RAYS = 400                      # rays per set (the interpreter twin uses fewer)
# lengths of caller directions: where dot(dir, dir), b * b and 4ac of RaySphere go subnormal (1e-19 .. 1e-23) or overflow (1e18 ..),
# both sides of the range in which the queries may skip (|dir| in [2^-10, 2^10], rt_kernel_query.cuh), and ordinary lengths
DIRECTION_SCALES = (1e-23, 1e-22, 1e-21, 1e-20, 1e-19, 1e-12, 2.0 ** -10 * (1 - 2.0 ** -12), 2.0 ** -10 * (1 + 2.0 ** -12), 0.01, 1.0,
                    1e3, 2.0 ** 10 * (1 - 2.0 ** -12), 2.0 ** 10 * (1 + 2.0 ** -12), 1e12, 1e18, 1e19, 3e19)
COUNTS = ("rays", "boxTests", "triTests", "sphereTests")


def open_mgr(lib, sc, options=None, enable=True):
    mgr = rt.RayComputeManager(lib)
    scenes.apply(sc, mgr)
    for k, v in (options or {}).items():
        mgr.context.set_option(k, v)
    if enable:
        mgr.OnEnable()
    return mgr


def assert_hits_equal(a, b, what):
    for f in ("dst", "pos", "normal"):
        assert_bit_equal(np.ascontiguousarray(a[f]), np.ascontiguousarray(b[f]), f"{what}: {f}")
    for f in ("isBackface", "kind", "index", "pad"):
        bad = np.flatnonzero(np.any((a[f] != b[f]).reshape(len(a), -1), axis=1))
        assert len(bad) == 0, f"{what}: {f} differs for {len(bad)} rays, first {bad[0]}: {a[bad[0]]} vs {b[bad[0]]}"


def pick_rays_np(sc, width, height, xs, ys):
    """SetupPixel's un-jittered ray (HL:547-558) restated in numpy float32, one operation at a time, from the scene's camera."""
    f = np.float32
    M = np.asarray(sc.cam_local_to_world, dtype=np.float32)          # (row, col)
    fd = f(sc.settings.get("focusDistance", 1.0))
    plane_h = f(f(fd * f(np.tan(np.float64(f(f(f(sc.fov) * f(0.5)) * f(0.0174532924)))))) * f(2))
    plane_w = f(plane_h * f(f(width) / f(height)))
    u = (np.asarray(xs, dtype=np.float32) / f(f(width) - f(1))).astype(np.float32)
    v = (np.asarray(ys, dtype=np.float32) / f(f(height) - f(1))).astype(np.float32)
    local = [(u - f(0.5)) * plane_w, (v - f(0.5)) * plane_h, np.full_like(u, f(f(1) * fd))]
    o = np.empty((len(u), 3), np.float32)
    d = np.empty((len(u), 3), np.float32)
    for a in range(3):
        o[:, a] = f(f(f(f(M[a, 0] * f(0)) + f(M[a, 1] * f(0))) + f(M[a, 2] * f(0))) + f(M[a, 3] * f(1)))
        fp = ((M[a, 0] * local[0] + M[a, 1] * local[1]).astype(np.float32) + M[a, 2] * local[2]).astype(np.float32) + M[a, 3] * f(1)
        d[:, a] = fp.astype(np.float32) - o[:, a]
    inv = (f(1) / np.sqrt(((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]).astype(np.float32) + d[:, 2] * d[:, 2]).astype(np.float32))).astype(np.float32)
    return capi.make_rays(o, d * inv[:, None])


def ray_sets(sc, seed=0, n=None):
    """name -> RAY_DTYPE array.  Points inside the scene come from the oracle's own pick hits."""
    n = n or RAYS
    rng = np.random.RandomState(seed)
    W, H = 24, 16
    xs, ys = np.meshgrid(np.arange(W), np.arange(H))
    pick = pick_rays_np(sc, W, H, xs.ravel(), ys.ravel())
    mgr = open_mgr(ORACLE_LIB, sc, enable=False)
    hits = mgr.trace_rays(pick)
    mgr.OnDestroy()
    hit = np.isfinite(hits["dst"])
    pts = hits["pos"][hit].astype(np.float64) if hit.any() else np.zeros((1, 3))
    cam = pick["origin"][0].astype(np.float64)

    def dirs(k):
        d = rng.normal(size=(k, 3))
        return d / np.linalg.norm(d, axis=1, keepdims=True)

    k = n
    t = rng.uniform(0.05, 0.95, (k, 1))
    inside = capi.make_rays(cam + t * (pts[rng.randint(len(pts), size=k)] - cam), dirs(k))
    back = pts[rng.randint(len(pts), size=k)]
    into = capi.make_rays(back + 1e-3 * (back - cam) / np.maximum(np.linalg.norm(back - cam, axis=1, keepdims=True), 1e-9), dirs(k))
    far_o = dirs(k) * rng.choice([1e3, 1e4, 1e5], size=(k, 1)) + cam
    far = capi.make_rays(far_o, (pts[rng.randint(len(pts), size=k)] - far_o) * rng.uniform(0.1, 3.0, (k, 1)))
    special = []
    for d in ([0, 0, 0], [1, 0, 0], [0, -1, 0], [0, 0, 1], [-0.0, 0, 1], [np.nan, 0, 1], [np.inf, 0, 0], [0, -np.inf, 1], [1e-30, 1e-30, 1],
              [1e30, 1, 0]):
        for org in (cam, pts[0], [np.nan, 0, 0], [np.inf, 1, 1], [1e5, 1e5, -1e5]):
            special.append((org, d))
    spec = capi.make_rays(np.array([s[0] for s in special], dtype=np.float64), np.array([s[1] for s in special], dtype=np.float64))
    scale = rng.choice(DIRECTION_SCALES, size=(k, 1))
    scaled = capi.make_rays(inside["origin"], dirs(k) * scale)
    mixed = np.concatenate([inside[: k // 3], far[: k // 3], into[: k // 3], scaled[: k // 3], spec])
    mixed = mixed[rng.permutation(len(mixed))]
    return {"pick": pick, "inside": inside, "into": into, "far": far, "scaled": scaled, "special": spec, "mixed": mixed}


def check_scene(sc, options_list=({},), sets=None, flags=(False, True)):
    """Every ray set, both flags, against the oracle, for each option set (model skipping on and off unless given)."""
    sets = sets or ray_sets(sc)
    ref_mgr = open_mgr(ORACLE_LIB, sc)
    ref = {(name, nc): ref_mgr.context.trace_rays(r, no_cull=nc) for name, r in sets.items() for nc in flags}
    ref_mgr.OnDestroy()
    for opts in options_list:
        for skip in ((opts["modelSkip"],) if "modelSkip" in opts else (1, 0)):
            mgr = open_mgr(CUDA_LIB, sc, dict(opts, modelSkip=skip))
            for (name, nc), want in ref.items():
                assert_hits_equal(mgr.context.trace_rays(sets[name], no_cull=nc), want, f"{sc.name} {opts} modelSkip={skip} {name} no_cull={nc}")
            mgr.OnDestroy()


def _matrices_disagree(sc):
    l2w, _ = scenes.trs(position=(0.5, 1.0, 0.5), scale=(0.2, 0.2, 0.2))
    _, w2l = scenes.trs(position=(-0.8, 2.2, 0.3), euler_deg=(20, 40, 60), scale=(0.25, 0.2, 0.3))
    sc.models[3] = scenes.ModelDesc(0, l2w, w2l, sc.models[3].material)
    return sc


def _singular(sc):
    sc = _matrices_disagree(sc)
    flat = np.array(sc.models[4].world_to_local, dtype=np.float64)
    flat[1, :] = 0.0
    sc.models[4] = scenes.ModelDesc(0, sc.models[4].local_to_world, flat, sc.models[4].material)
    return sc


def test_cornell_spheres():
    check_scene(scenes.cornell_spheres(24, 16, 3, 1))


def test_ten_thousand_spheres_with_the_accelerator():
    check_scene(scenes.random_soup(24, 16, 3, 1, triangles=300, spheres=10000), ({}, {"extInstantiation": 1}))


def test_knot_room_with_glass():
    check_scene(scenes.knot_room(24, 16, 3, 1, nu=40, nv=8, glass=True))


def test_instanced_models_with_skipping():
    check_scene(scenes.instanced_knots(24, 16, 3, 1, instances=23))


@pytest.mark.parametrize("tlas", [-1, 0, 1])
def test_above_128_models_with_the_tlas(tlas):
    check_scene(scenes.instanced_knots(24, 16, 3, 1, instances=150), ({"tlas": tlas},))


def test_model_whose_matrices_disagree_and_a_singular_world_to_local():
    check_scene(_matrices_disagree(scenes.instanced_knots(24, 16, 3, 1, instances=12)))
    check_scene(_singular(scenes.instanced_knots(24, 16, 3, 1, instances=12)), ({"tlas": 1},))


def test_unity_fixture():
    from test_round2_abi import load_fixture
    check_scene(load_fixture(24, 16))


def test_accelerator_does_not_keep_a_hit_at_infinity():
    """Regression (tools/simt_fuzz.py --queries): a direction so short that dot(dir, dir) underflows gives RaySphere a 'hit' at dst = +inf
    from inside a sphere.  The reference's strict < never takes it; the sphere accelerator's tie rule (equal dst, lower index) did, and
    the query returned that sphere with pos = origin + dir * inf."""
    sc = scenes.random_soup(24, 16, 3, 1, triangles=30, spheres=200)
    centres = sc.spheres["centre"].astype(np.float64)
    rng = np.random.RandomState(29)
    d = rng.normal(size=(len(centres), 3))
    sets = {"tiny": capi.make_rays(centres, d * 1e-25), "huge": capi.make_rays(centres, d * 1e25),
            "tiny_outside": capi.make_rays(centres - 3.0, d * 1e-25)}
    check_scene(sc, ({}, {"countStats": 1}), sets=sets)


@pytest.mark.parametrize("name", ["spheres", "tlas", "knot"])
def test_directions_of_every_length(name):
    """Regression: the padding of the sphere boxes and the model world boxes holds for the reference's rounding with normal
    intermediates; with |dir| around 1e-21 the reference's discriminant is mostly rounding and it hits spheres (at dst ~ 1e22) that the
    padded boxes prune.  In-scene origins with unit directions scaled by 1e-23 .. 3e19 (each scale its own batch) must give the oracle's
    bits: directions outside |dir| in [2^-10, 2^10] take the linear loop."""
    sc = {"spheres": lambda: scenes.random_soup(24, 16, 3, 1, triangles=300, spheres=200),
          "tlas": lambda: scenes.instanced_knots(24, 16, 3, 1, instances=150),
          "knot": lambda: scenes.knot_room(24, 16, 3, 1, nu=40, nv=8, glass=True)}[name]()
    base = ray_sets(sc, seed=31, n=RAYS // 2)["inside"]
    unit = base["dir"] / np.linalg.norm(base["dir"], axis=1, keepdims=True)
    sets = {f"scale {s:g}": capi.make_rays(base["origin"], unit.astype(np.float64) * s) for s in DIRECTION_SCALES}
    check_scene(sc, ({},), sets=sets)


@pytest.mark.parametrize("name", ["knot", "spheres"])
def test_counters_equal_the_oracle(name):
    sc = scenes.knot_room(24, 16, 3, 1, nu=40, nv=8, glass=True) if name == "knot" else scenes.random_soup(24, 16, 3, 1, triangles=300, spheres=40)
    sets = ray_sets(sc, seed=3)
    for lib in (ORACLE_LIB, CUDA_LIB):
        mgr = open_mgr(lib, sc, {"countStats": 1})
        ctx = mgr.context
        ctx.reset_stats()
        got = []
        for name_, r in sets.items():
            for nc in (False, True):
                ctx.trace_rays(r, no_cull=nc)
                got.append(ctx.stats())
        if lib == ORACLE_LIB:
            want = got
        else:
            for a, b in zip(got, want):
                assert all(a[k] == b[k] for k in COUNTS), (a, b)
                assert a["dispatches"] == 0
        mgr.OnDestroy()


def test_query_before_any_resize_and_after_the_scene_changed():
    sc = scenes.instanced_knots(24, 16, 3, 1, instances=12)
    sc.spheres = scenes.cornell_spheres().spheres[6:8].copy()
    sets = ray_sets(sc, seed=5)
    out = {}
    for lib in (ORACLE_LIB, CUDA_LIB):
        mgr = open_mgr(lib, sc, enable=False)            # no OnEnable: no rtResize, no dispatch
        first = mgr.trace_rays(sets["inside"])
        mgr.OnEnable()
        mgr.RenderFrame()
        l2w, w2l = scenes.trs(position=(0.2, 1.5, 0.0), euler_deg=(10, 20, 30), scale=(0.3, 0.3, 0.3))
        mgr.set_model_transform(4, l2w, w2l)
        sph = sc.spheres.copy()
        sph["centre"][0] = (0.1, 1.6, 0.2)
        mgr.set_spheres(sph)
        second = mgr.trace_rays(sets["inside"])
        out[lib] = (first, second)
        mgr.OnDestroy()
    assert_hits_equal(out[CUDA_LIB][0], out[ORACLE_LIB][0], "before rtResize")
    assert_hits_equal(out[CUDA_LIB][1], out[ORACLE_LIB][1], "after ModelInfo / Spheres changed")
    assert not np.array_equal(out[CUDA_LIB][0]["dst"], out[CUDA_LIB][1]["dst"]), "the second query did not see the new scene"


@pytest.mark.parametrize("name", ["knot", "soup"])
def test_queries_between_frames_change_nothing_the_frames_show(name):
    sc = (scenes.instanced_knots(32, 24, 4, 2, instances=150) if name == "knot" else
          scenes.random_soup(32, 24, 4, 1, triangles=600, spheres=300))
    far = ray_sets(sc, seed=7)["far"]
    images = []
    for with_queries in (False, True):
        mgr = open_mgr(CUDA_LIB, sc)
        ctx = mgr.context
        ctx.reset_stats()
        for _ in range(3):
            mgr.RenderFrame()
            if with_queries:
                before = ctx.stats()
                ctx.trace_rays(far)
                after = ctx.stats()
                assert after["dispatches"] == before["dispatches"] and after["kernelMs"] == before["kernelMs"]
                assert after["rays"] == before["rays"] + len(far)
        images.append((mgr.raytraceFrameTex, mgr.accumulatedResult, ctx.stats()))
        mgr.OnDestroy()
    assert_bit_equal(images[1][0], images[0][0], "FrameRender with queries in between")
    assert_bit_equal(images[1][1], images[0][1], "AccumulatedRender with queries in between")
    assert images[1][2]["dispatches"] == images[0][2]["dispatches"] == 3


def test_empty_batch_and_every_error_code():
    sc = scenes.knot_room(16, 12, 3, 1, nu=30, nv=6)
    for lib in (ORACLE_LIB, CUDA_LIB):
        mgr = open_mgr(lib, sc)
        ctx, L, h = mgr.context, mgr.context._L, mgr.context.handle
        r = ray_sets(sc, n=8)["inside"]
        hits = np.zeros(len(r), dtype=capi.RAY_HIT_DTYPE)
        st = ctx.stats()
        assert L.rtTraceRays(h, None, 0, None, 0) == capi.RT_OK and ctx.stats()["rays"] == st["rays"]
        assert L.rtTraceRays(None, r.ctypes.data, len(r), hits.ctypes.data, 0) == capi.RT_E_INVALID
        assert L.rtTraceRays(h, r.ctypes.data, -1, hits.ctypes.data, 0) == capi.RT_E_INVALID
        assert L.rtTraceRays(h, None, len(r), hits.ctypes.data, 0) == capi.RT_E_INVALID
        assert L.rtTraceRays(h, r.ctypes.data, len(r), None, 0) == capi.RT_E_INVALID
        for fl in (2, -1, 3):
            assert L.rtTraceRays(h, r.ctypes.data, len(r), hits.ctypes.data, fl) == capi.RT_E_INVALID
        ctx.set_int("modelCount", 99)
        assert L.rtTraceRays(h, r.ctypes.data, len(r), hits.ctypes.data, 0) == capi.RT_E_STATE
        ctx.set_int("modelCount", 2)
        models = np.zeros(2, dtype=capi.MODEL_DTYPE)
        models[1]["nodeOffset"] = 10 ** 7
        ctx.set_buffer("ModelInfo", models)
        assert L.rtTraceRays(h, r.ctypes.data, len(r), hits.ctypes.data, 0) == capi.RT_E_STATE
        ctx.set_buffer("Nodes", np.zeros(0, dtype=capi.NODE_DTYPE))
        assert L.rtTraceRays(h, r.ctypes.data, len(r), hits.ctypes.data, 0) == capi.RT_E_STATE
        assert L.rtTraceRaysDevice(None, None, None, 0, 0) == capi.RT_E_INVALID
        mgr.OnDestroy()
    # a tree deeper than the traversal stacks (64 levels of inner nodes) is refused like rtDispatch refuses it
    from test_round2_abi import chain_bvh, one_model_scene
    for lib in (ORACLE_LIB, CUDA_LIB):
        mgr = open_mgr(lib, one_model_scene(16, 12))
        tris, nodes = chain_bvh(64)
        mgr.context.set_buffer("Triangles", tris)
        mgr.context.set_buffer("Nodes", nodes)
        with pytest.raises(capi.RtError) as e:
            mgr.context.trace_rays(np.zeros((1, 3)), np.ones((1, 3)))
        assert e.value.code == capi.RT_E_STATE and "too deep" in str(e.value), lib
        mgr.OnDestroy()


def test_device_pointer_form_on_the_context_stream_and_a_caller_stream():
    torch = pytest.importorskip("torch")
    sc = scenes.instanced_knots(24, 16, 3, 1, instances=150)
    sets = ray_sets(sc, seed=11)
    rays = np.concatenate(list(sets.values()))
    mgr = open_mgr(CUDA_LIB, sc)
    ctx = mgr.context
    want = ctx.trace_rays(rays)
    d_rays = torch.from_numpy(rays.view(np.uint8).copy()).cuda()
    for stream in (None, torch.cuda.Stream()):
        d_hits = torch.full((len(rays) * 48,), 0x5a, dtype=torch.uint8, device="cuda")
        if stream is not None:
            ctx.set_stream(stream.cuda_stream)
        ctx.trace_rays_device(d_rays.data_ptr(), d_hits.data_ptr(), len(rays))
        ctx.synchronize()
        got = d_hits.cpu().numpy().view(capi.RAY_HIT_DTYPE)
        assert_hits_equal(got, want, f"device form, stream {stream}")
    ctx.set_stream(0)
    d_hits = torch.zeros(len(rays) * 48 + 8, dtype=torch.uint8, device="cuda")
    with pytest.raises(capi.RtError) as e:
        ctx.trace_rays_device(d_rays.data_ptr(), d_hits.data_ptr() + 8, len(rays))
    assert e.value.code == capi.RT_E_INVALID
    mgr.OnDestroy()
    o = capi.RtLib(ORACLE_LIB).create(0)
    assert o._L.rtTraceRaysDevice(o.handle, None, None, 0, 0) == capi.RT_E_STATE


def test_four_million_rays_on_the_871k_triangle_cluster():
    sc = scenes.knot_cluster(64, 36, 4, 1)
    rng = np.random.RandomState(13)
    n = (4 << 20) + 12345                 # the host form's batches of RT_TRACE_CHUNK_RAYS, with a partial last one
    o = rng.uniform((-2.7, 0.05, -2.9), (2.7, 3.95, 2.7), (n, 3))
    d = rng.normal(size=(n, 3))
    rays = capi.make_rays(o, d)
    mgr = open_mgr(CUDA_LIB, sc)
    got = mgr.context.trace_rays(rays)
    mgr.OnDestroy()
    sub = rng.choice(n, 200_000, replace=False)
    ref = open_mgr(ORACLE_LIB, sc)
    want = ref.context.trace_rays(rays[sub])
    ref.OnDestroy()
    assert_hits_equal(got[sub], want, "4M rays, seeded 200k subset")
    assert (got["kind"] == capi.RT_HIT_MODEL).mean() > 0.5          # (the room encloses the origins; rays that leave through a gap miss)


def test_pick_against_numpy_and_the_oracle_and_the_cpp_manager_against_python():
    sc = scenes.knot_room(40, 30, 3, 1, nu=40, nv=8, glass=True)
    xs, ys = [0, 39, 20, 7, 33], [0, 29, 15, 22, 3]
    want_rays = pick_rays_np(sc, 40, 30, xs, ys)
    ref = open_mgr(ORACLE_LIB, sc)
    want_hits = ref.context.trace_rays(want_rays)
    ref.OnDestroy()
    mgr = open_mgr(CUDA_LIB, sc)
    for i, (x, y) in enumerate(zip(xs, ys)):
        ray = mgr.pick_ray(x, y)
        assert ray.tobytes() == want_rays[i].tobytes(), (x, y, ray, want_rays[i])
        hit = mgr.pick(x, y)
        assert_hits_equal(np.array([hit]), want_hits[i:i + 1], f"pick({x}, {y})")
    assert_hits_equal(mgr.trace_rays(want_rays), mgr.context.trace_rays(want_rays), "RayComputeManager.TraceRays vs the context")
    centre = mgr.pick(19.5, 14.5)
    assert centre["kind"] == capi.RT_HIT_MODEL and np.isfinite(centre["dst"])
    mgr.OnDestroy()
