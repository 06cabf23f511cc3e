"""rtTraceOcclusion on the H100 (`-m gpu`): whether anything lies on a caller-supplied segment equals the oracle's answer bit for bit —
the reference's collision loop from result.dst = tMax — across the scenes and rays of the rtTraceRays tests (tests/test_gpu_trace_rays.py),
tMax at, one ulp below and one ulp above each ray's closest hit, fractions of it, +inf and special values, both flags, model skipping
on and off.  Also against the library's own rtTraceRays (equal at tMax = +inf, implied at every tMax), a sphere hit at exactly
dst = tMax, the early-exit counters, the context states around it and the device-pointer form.  The same bodies run in the CPU suite
against the SIMT interpreter build (tests/test_simt_occlusion.py)."""
import numpy as np
import pytest

from conftest import CUDA_LIB, ORACLE_LIB, assert_bit_equal
from ray_tracing_b200 import capi, scenes
import test_gpu_trace_rays as T

pytestmark = pytest.mark.gpu

RAYS = 400                      # rays per set of the rtTraceRays tests (the interpreter twin uses fewer)
SPECIAL_T = np.array([0.0, -0.0, -1.0, -np.inf, np.nan, 1e-45, 3e38], dtype=np.float32)


def segments(rays, t_max) -> np.ndarray:
    return capi.make_segments(rays["origin"], rays["dir"], np.asarray(t_max, dtype=np.float32))


def tmax_sets(rays, closest, seed=0, prefix=""):
    """name -> SEGMENT_DTYPE array on `rays`: tMax = +inf, the closest hit's dst exactly (+inf on a miss), one ulp below and above it,
    random fractions of it (random lengths on a miss) and the special values, cycled."""
    rng = np.random.RandomState(seed)
    d = closest["dst"].astype(np.float32)
    n = len(rays)
    hit = np.isfinite(d)
    frac = np.where(hit, (d * rng.uniform(0.0, 1.0, n)).astype(np.float32), rng.uniform(0.0, 20.0, n).astype(np.float32))
    return {prefix + "inf": segments(rays, np.full(n, np.inf, np.float32)),
            prefix + "dst": segments(rays, d),
            prefix + "below": segments(rays, np.nextafter(d, np.float32(-np.inf))),
            prefix + "above": segments(rays, np.where(hit, np.nextafter(d, np.float32(np.inf)), d)),
            prefix + "fraction": segments(rays, frac),
            prefix + "special": segments(rays, SPECIAL_T[np.arange(n) % len(SPECIAL_T)])}


def segment_sets(sc, seed=0, n=None):
    """name -> SEGMENT_DTYPE array: every ray of the rtTraceRays tests' ray sets (pick rays, in-scene origins, just inside meshes, far
    origins, scaled directions, special values) with every tMax of tmax_sets, measured from the oracle's closest hits."""
    rays = np.concatenate(list(T.ray_sets(sc, seed=seed, n=n or RAYS).values()))
    ref = T.open_mgr(ORACLE_LIB, sc)
    closest = ref.context.trace_rays(rays)
    ref.OnDestroy()
    return tmax_sets(rays, closest, seed)


def assert_occlusion_equal(a, b, what, segs=None):
    a, b = np.asarray(a, dtype=bool), np.asarray(b, dtype=bool)
    bad = np.flatnonzero(a != b)
    assert len(bad) == 0, f"{what}: {len(bad)} of {len(a)} segments differ, first {bad[0]}: {a[bad[0]]} vs {b[bad[0]]}" + \
        (f" on {segs[bad[0]]}" if segs is not None else "")


def assert_consistent_with_trace_rays(ctx, segs, occ, no_cull, what):
    """The library's own closest hit on the same rays: occluded implies dst < tMax, and at tMax = +inf the two say the same."""
    hits = ctx.trace_rays(capi.make_rays(segs["origin"], segs["dir"]), no_cull=no_cull)
    closer = hits["dst"] < segs["tMax"]
    bad = np.flatnonzero(occ & ~closer)
    assert len(bad) == 0, f"{what}: occluded but rtTraceRays dst >= tMax for {len(bad)} segments, first {segs[bad[0]]} dst {hits['dst'][bad[0]]}"
    inf = np.isposinf(segs["tMax"])
    assert_occlusion_equal(occ[inf], hits["kind"][inf] != capi.RT_HIT_NONE, f"{what}: tMax = +inf vs rtTraceRays kind")


def check_scene(sc, options_list=({},), sets=None, flags=(False, True), against_trace_rays=True):
    """Every segment set, both flags, against the oracle, for each option set (model skipping on and off unless given)."""
    sets = sets or segment_sets(sc)
    ref_mgr = T.open_mgr(ORACLE_LIB, sc)
    ref = {(name, nc): ref_mgr.context.trace_occlusion(s, no_cull=nc) for name, s in sets.items() for nc in flags}
    ref_mgr.OnDestroy()
    for opts in options_list:
        for skip in ((opts["modelSkip"],) if "modelSkip" in opts else (1, 0)):
            mgr = T.open_mgr(CUDA_LIB, sc, dict(opts, modelSkip=skip))
            for (name, nc), want in ref.items():
                what = f"{sc.name} {opts} modelSkip={skip} {name} no_cull={nc}"
                got = mgr.context.trace_occlusion(sets[name], no_cull=nc)
                assert got.dtype == np.bool_ and got.shape == (len(sets[name]),)
                assert_occlusion_equal(got, want, what, sets[name])
                if against_trace_rays:
                    assert_consistent_with_trace_rays(mgr.context, sets[name], got, nc, what)
            mgr.OnDestroy()
    return ref


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
    check_scene(T._matrices_disagree(scenes.instanced_knots(24, 16, 3, 1, instances=12)))
    check_scene(T._singular(scenes.instanced_knots(24, 16, 3, 1, instances=12)), ({"tlas": 1},))


def test_unity_fixture():
    from test_round2_abi import load_fixture
    check_scene(load_fixture(24, 16))


@pytest.mark.parametrize("name", ["spheres", "tlas", "knot"])
def test_directions_of_every_length(name):
    """In-scene origins with unit directions scaled by 1e-23 .. 3e19 (T.DIRECTION_SCALES), each scale with every tMax set: directions
    outside |dir| in [2^-10, 2^10] take the linear loop, and tMax is measured in multiples of the direction as dst is."""
    sc = {"spheres": lambda: scenes.random_soup(24, 16, 3, 1, triangles=300, spheres=200),
          "tlas": lambda: scenes.instanced_knots(24, 16, 3, 1, instances=150),
          "knot": lambda: scenes.knot_room(24, 16, 3, 1, nu=40, nv=8, glass=True)}[name]()
    base = T.ray_sets(sc, seed=31, n=max(RAYS // 8, 8))["inside"]
    unit = base["dir"] / np.linalg.norm(base["dir"], axis=1, keepdims=True)
    rays = np.concatenate([capi.make_rays(base["origin"], unit.astype(np.float64) * s) for s in T.DIRECTION_SCALES])
    ref = T.open_mgr(ORACLE_LIB, sc)
    closest = ref.context.trace_rays(rays)
    ref.OnDestroy()
    check_scene(sc, ({},), sets=tmax_sets(rays, closest, seed=31))


@pytest.mark.parametrize("accelerator", [False, True], ids=["linear", "accelerator"])
def test_a_sphere_hit_at_exactly_tmax_does_not_count(accelerator):
    """Hazard of the sphere accelerator: its tie rule (equal dst, lower index) starts from index INT_MAX, so seeded with tMax it would
    keep a sphere at exactly dst = tMax, which the reference's strict < rejects.  Segments that end exactly on a sphere's surface are
    not occluded; one ulp longer, they are — through the linear loop (few spheres) and through the accelerator (many)."""
    sc = scenes.random_soup(24, 16, 3, 1, triangles=30, spheres=400 if accelerator else 40)
    centres = sc.spheres["centre"].astype(np.float64)
    rng = np.random.RandomState(37)
    lo, hi = centres.min(axis=0), centres.max(axis=0)
    k = max(RAYS // 2, 48)
    o = rng.uniform(lo, hi, (k, 3))
    rays = capi.make_rays(o, centres[rng.randint(len(centres), size=k)] - o)      # aimed at sphere centres: mostly sphere hits
    ref = T.open_mgr(ORACLE_LIB, sc)
    closest = ref.context.trace_rays(rays)
    ref.OnDestroy()
    on_sphere = closest["kind"] == capi.RT_HIT_SPHERE
    assert on_sphere.mean() > 0.5
    sets = tmax_sets(rays, closest, seed=37)
    ref = check_scene(sc, ({}, {"countStats": 1}), sets={k_: sets[k_] for k_ in ("dst", "below", "above", "inf")})
    for nc in (False, True):
        assert not ref[("dst", nc)][on_sphere].any()
        assert ref[("above", nc)][on_sphere].all()


@pytest.mark.parametrize("name", ["knot", "spheres"])
def test_counters_equal_the_oracle_early_exit(name):
    """With countStats the box / triangle / sphere tests are those of the walk in the reference's order up to the first hit (linear
    spheres here: the accelerator's sphere counters are its own)."""
    sc = scenes.knot_room(24, 16, 3, 1, nu=40, nv=8, glass=True) if name == "knot" else scenes.random_soup(24, 16, 3, 1, triangles=300, spheres=40)
    sets = segment_sets(sc, seed=3)
    full = {}
    for lib in (ORACLE_LIB, CUDA_LIB):
        mgr = T.open_mgr(lib, sc, {"countStats": 1})
        ctx = mgr.context
        ctx.reset_stats()
        got = []
        for s in sets.values():
            for nc in (False, True):
                ctx.trace_occlusion(s, no_cull=nc)
                got.append(ctx.stats())
        if lib == ORACLE_LIB:
            want = got
        else:
            for a, b in zip(got, want):
                assert all(a[k] == b[k] for k in T.COUNTS), (a, b)
                assert a["dispatches"] == 0 and a["kernelMs"] == 0
        ctx.reset_stats()
        ctx.trace_rays(capi.make_rays(sets["inf"]["origin"], sets["inf"]["dir"]))
        full[lib] = ctx.stats()
        mgr.OnDestroy()
    # the early exit does less work than the closest hit on the same rays
    occ_inf = want[0]
    assert occ_inf["triTests"] + occ_inf["boxTests"] < full[ORACLE_LIB]["triTests"] + full[ORACLE_LIB]["boxTests"]


def test_query_before_any_resize_and_after_the_scene_changed():
    sc = scenes.instanced_knots(24, 16, 3, 1, instances=12)
    sc.spheres = scenes.cornell_spheres().spheres[6:8].copy()
    sets = segment_sets(sc, seed=5)
    segs = np.concatenate([sets["above"], sets["fraction"]])
    out = {}
    for lib in (ORACLE_LIB, CUDA_LIB):
        mgr = T.open_mgr(lib, sc, enable=False)          # no OnEnable: no rtResize, no dispatch
        first = mgr.trace_occlusion(segs)
        mgr.OnEnable()
        mgr.RenderFrame()
        l2w, w2l = scenes.trs(position=(0.2, 1.5, 0.0), euler_deg=(10, 20, 30), scale=(0.3, 0.3, 0.3))
        mgr.set_model_transform(4, l2w, w2l)
        sph = sc.spheres.copy()
        sph["centre"][0] = (0.1, 1.6, 0.2)
        mgr.set_spheres(sph)
        second = mgr.trace_occlusion(segs)
        out[lib] = (first, second)
        mgr.OnDestroy()
    assert_occlusion_equal(out[CUDA_LIB][0], out[ORACLE_LIB][0], "before rtResize")
    assert_occlusion_equal(out[CUDA_LIB][1], out[ORACLE_LIB][1], "after ModelInfo / Spheres changed")
    assert not np.array_equal(out[CUDA_LIB][0], out[CUDA_LIB][1]), "the second query did not see the new scene"


@pytest.mark.parametrize("name", ["knot", "soup"])
def test_queries_between_frames_change_nothing_the_frames_show(name):
    sc = (scenes.instanced_knots(32, 24, 4, 2, instances=150) if name == "knot" else
          scenes.random_soup(32, 24, 4, 1, triangles=600, spheres=300))
    far = T.ray_sets(sc, seed=7)["far"]
    segs = segments(far, np.random.RandomState(7).uniform(0.0, 2.0, len(far)))
    images = []
    for with_queries in (False, True):
        mgr = T.open_mgr(CUDA_LIB, sc, {"countStats": 1})
        ctx = mgr.context
        ctx.reset_stats()
        for _ in range(3):
            mgr.RenderFrame()
            if with_queries:
                before = ctx.stats()
                ctx.trace_occlusion(segs)
                after = ctx.stats()
                assert after["dispatches"] == before["dispatches"] and after["kernelMs"] == before["kernelMs"]
                assert after["rays"] == before["rays"] + len(segs)
        images.append((mgr.raytraceFrameTex, mgr.accumulatedResult, ctx.stats(), ctx.pixel_stats()))
        mgr.OnDestroy()
    assert_bit_equal(images[1][0], images[0][0], "FrameRender with queries in between")
    assert_bit_equal(images[1][1], images[0][1], "AccumulatedRender with queries in between")
    assert images[1][3].tobytes() == images[0][3].tobytes(), "PixelStats with queries in between"
    assert images[1][2]["dispatches"] == images[0][2]["dispatches"] == 3


def test_empty_batch_and_every_error_code():
    sc = scenes.knot_room(16, 12, 3, 1, nu=30, nv=6)
    for lib in (ORACLE_LIB, CUDA_LIB):
        mgr = T.open_mgr(lib, sc)
        ctx, L, h = mgr.context, mgr.context._L, mgr.context.handle
        s = segments(T.ray_sets(sc, n=8)["inside"], np.full(8, np.inf, np.float32))
        occ = np.zeros(len(s), dtype=np.uint8)
        st = ctx.stats()
        assert L.rtTraceOcclusion(h, None, 0, None, 0) == capi.RT_OK and ctx.stats()["rays"] == st["rays"]
        assert len(ctx.trace_occlusion(np.zeros(0, dtype=capi.SEGMENT_DTYPE))) == 0
        assert L.rtTraceOcclusion(None, s.ctypes.data, len(s), occ.ctypes.data, 0) == capi.RT_E_INVALID
        assert L.rtTraceOcclusion(h, s.ctypes.data, -1, occ.ctypes.data, 0) == capi.RT_E_INVALID
        assert L.rtTraceOcclusion(h, None, len(s), occ.ctypes.data, 0) == capi.RT_E_INVALID
        assert L.rtTraceOcclusion(h, s.ctypes.data, len(s), None, 0) == capi.RT_E_INVALID
        for fl in (2, -1, 3):
            assert L.rtTraceOcclusion(h, s.ctypes.data, len(s), occ.ctypes.data, fl) == capi.RT_E_INVALID
        ctx.set_int("modelCount", 99)
        assert L.rtTraceOcclusion(h, s.ctypes.data, len(s), occ.ctypes.data, 0) == capi.RT_E_STATE
        ctx.set_int("modelCount", 2)
        models = np.zeros(2, dtype=capi.MODEL_DTYPE)
        models[1]["nodeOffset"] = 10 ** 7
        ctx.set_buffer("ModelInfo", models)
        assert L.rtTraceOcclusion(h, s.ctypes.data, len(s), occ.ctypes.data, 0) == capi.RT_E_STATE
        ctx.set_buffer("Nodes", np.zeros(0, dtype=capi.NODE_DTYPE))
        assert L.rtTraceOcclusion(h, s.ctypes.data, len(s), occ.ctypes.data, 0) == capi.RT_E_STATE
        assert L.rtTraceOcclusionDevice(None, None, None, 0, 0) == capi.RT_E_INVALID
        mgr.OnDestroy()
    from test_round2_abi import chain_bvh, one_model_scene
    for lib in (ORACLE_LIB, CUDA_LIB):
        mgr = T.open_mgr(lib, one_model_scene(16, 12))
        tris, nodes = chain_bvh(64)
        mgr.context.set_buffer("Triangles", tris)
        mgr.context.set_buffer("Nodes", nodes)
        with pytest.raises(capi.RtError) as e:
            mgr.context.trace_occlusion(capi.make_segments(np.zeros((1, 3)), np.ones((1, 3)), np.inf))
        assert e.value.code == capi.RT_E_STATE and "too deep" in str(e.value), lib
        mgr.OnDestroy()


def test_device_pointer_form_on_the_context_stream_and_a_caller_stream():
    torch = pytest.importorskip("torch")
    sc = scenes.instanced_knots(24, 16, 3, 1, instances=150)
    segs = np.concatenate(list(segment_sets(sc, seed=11).values()))
    mgr = T.open_mgr(CUDA_LIB, sc)
    ctx = mgr.context
    want = ctx.trace_occlusion(segs)
    raw = torch.zeros(len(segs) * 28 + 4, dtype=torch.uint8)
    raw[4:] = torch.from_numpy(segs.view(np.uint8).copy())
    d_raw = raw.cuda()
    for stream in (None, torch.cuda.Stream()):
        d_occ = torch.full((len(segs) + 1,), 0x5a, dtype=torch.uint8, device="cuda")
        if stream is not None:
            ctx.set_stream(stream.cuda_stream)
        ctx.trace_occlusion_device(d_raw.data_ptr() + 4, d_occ.data_ptr() + 1, len(segs))      # 4-byte aligned segments, any byte out
        ctx.synchronize()
        got = d_occ.cpu().numpy()
        assert got[0] == 0x5a and set(np.unique(got[1:])) <= {0, 1}
        assert_occlusion_equal(got[1:].astype(bool), want, f"device form, stream {stream}")
    ctx.set_stream(0)
    with pytest.raises(capi.RtError) as e:
        ctx.trace_occlusion_device(d_raw.data_ptr() + 2, d_occ.data_ptr(), len(segs))
    assert e.value.code == capi.RT_E_INVALID
    mgr.OnDestroy()
    o = capi.RtLib(ORACLE_LIB).create(0)
    assert o._L.rtTraceOcclusionDevice(o.handle, None, None, 0, 0) == capi.RT_E_STATE


def test_four_million_segments_on_the_871k_triangle_cluster():
    sc = scenes.knot_cluster(64, 36, 4, 1)
    rng = np.random.RandomState(13)
    n = (4 << 20) + 12345                 # the host form's batches of RT_TRACE_CHUNK_RAYS, with a partial last one
    lo, hi = (-2.7, 0.05, -2.9), (2.7, 3.95, 2.7)
    a, b = rng.uniform(lo, hi, (n, 3)), rng.uniform(lo, hi, (n, 3))
    segs = capi.make_segments(a, b - a, np.float32(1.0 - 2.0 ** -10))        # line of sight between two in-scene points
    mgr = T.open_mgr(CUDA_LIB, sc)
    got = mgr.context.trace_occlusion(segs)
    mgr.OnDestroy()
    sub = rng.choice(n, 200_000, replace=False)
    ref = T.open_mgr(ORACLE_LIB, sc)
    want = ref.context.trace_occlusion(segs[sub])
    ref.OnDestroy()
    assert_occlusion_equal(got[sub], want, "4M segments, seeded 200k subset")
    assert 0.05 < got.mean() < 0.95


def test_manager_trace_occlusion_equals_the_context():
    sc = scenes.knot_room(24, 16, 3, 1, nu=40, nv=8, glass=True)
    segs = segment_sets(sc, seed=41, n=max(RAYS // 4, 16))["fraction"]
    mgr = T.open_mgr(CUDA_LIB, sc)
    for nc in (False, True):
        assert_occlusion_equal(mgr.trace_occlusion(segs, no_cull=nc), mgr.context.trace_occlusion(segs, no_cull=nc), f"manager no_cull={nc}")
    mgr.OnDestroy()
