"""rtTracePaths on the H100 (`-m gpu`): the radiance along caller-supplied rays equals the oracle's Shader::Trace sample loop bit for
bit, rgb and final RNG state.  A pixel of rtDispatch, rebuilt sample by sample from the oracle's camera rays (orCameraSample) through
rtTracePaths(samples = 1), equals the dispatch's FrameRender with every kernel; arbitrary rays (the rtTraceRays ray sets, every
direction length) with random states, sample counts, bounce limits and sky; chaining; what the call reads and leaves alone; its
counters; its refusals; the device form.  The same bodies run in the CPU suite against the SIMT interpreter build
(tests/test_simt_trace_paths.py)."""
import ctypes as C

import numpy as np
import pytest

from conftest import CUDA_LIB, ORACLE_LIB, assert_bit_equal
from ray_tracing_b200 import capi, scenes
import test_gpu_trace_rays as T

pytestmark = pytest.mark.gpu

FRAME = (24, 16)                # frame of the pixel rebuilds (the interpreter twin uses a smaller one)
RAYS = 160                      # rays per set of the arbitrary-ray tests
KERNELS = (0, 1, 2)             # "kernel" of the dispatch a rebuild is compared with


def camera_samples(octx, w, h, states=None) -> np.ndarray:
    """orCameraSample of every pixel of a w x h frame (row-major, row 0 = bottom) on an oracle context: the camera ray and the state
    after its four jitter draws, starting from `states` (n uint32) or from each pixel's own seed."""
    L = octx._L
    L.orCameraSamples.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    ys, xs = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
    xy = np.ascontiguousarray(np.stack([xs.ravel(), ys.ravel()], axis=1).astype(np.int32))
    out = np.zeros(len(xy), dtype=capi.PATH_RAY_DTYPE)
    st = None if states is None else np.ascontiguousarray(states, dtype=np.uint32)
    assert L.orCameraSamples(octx.handle, xy.ctypes.data, len(xy), None if st is None else st.ctypes.data, out.ctypes.data) == capi.RT_OK
    return out


def rebuild_frame(ctx, octx, w, h, R):
    """A frame of R samples per pixel rebuilt through ctx.trace_paths(samples = 1): each sample's camera ray from the oracle, fed the
    state the previous sample returned; the rgb summed in float32 in order and divided by R, as HL:578-581 do."""
    total = np.zeros((w * h, 3), dtype=np.float32)
    states = None
    for _ in range(R):
        out = ctx.trace_paths(camera_samples(octx, w, h, states), 1)
        total = (total + out["rgb"]).astype(np.float32)
        states = out["rngState"]
    return (total / np.float32(R)).astype(np.float32).reshape(h, w, 3)


def open_frame(lib, sc, R, options=None):
    """A manager of the scene at FRAME with NumRaysPerPixel = R, after one RenderFrame (Frame = 0)."""
    sc.settings = dict(sc.settings, numRaysPerPixel=R)
    mgr = T.open_mgr(lib, sc, options)
    mgr.RenderFrame()
    return mgr


def check_camera_rebuild(make, options_list=({},), kernels=None, rays_per_pixel=(1, 3)):
    for R in rays_per_pixel:
        sc = make()
        sc.width, sc.height = FRAME
        w, h = FRAME
        ref = open_frame(ORACLE_LIB, sc, R)
        want = ref.raytraceFrameTex[..., :3]
        assert_bit_equal(rebuild_frame(ref.context, ref.context, w, h, R), want, f"{sc.name} R={R}: oracle rtTracePaths vs its FrameRender")
        for opts in options_list:
            for kernel in kernels or KERNELS:
                for skip in ((opts["modelSkip"],) if "modelSkip" in opts else (1, 0)):
                    o = dict(opts, kernel=kernel, modelSkip=skip)
                    mgr = open_frame(CUDA_LIB, sc, R, o)
                    what = f"{sc.name} R={R} {o}"
                    assert_bit_equal(mgr.raytraceFrameTex[..., :3], want, f"{what}: dispatch vs oracle")
                    assert_bit_equal(rebuild_frame(mgr.context, ref.context, w, h, R), want, f"{what}: rtTracePaths rebuild")
                    mgr.OnDestroy()
        ref.OnDestroy()


def _soup_with_sky_and_defocus():
    sc = scenes.random_soup(24, 16, 4, 1, triangles=400, spheres=60)
    sc.settings = dict(sc.settings, useSky=True, defocusStrength=40.0, focusDistance=6.0)
    return sc


def test_camera_rebuild_cornell_spheres():
    check_camera_rebuild(lambda: scenes.cornell_spheres(24, 16, 4, 1))


def test_camera_rebuild_knot_room_with_glass():
    check_camera_rebuild(lambda: scenes.knot_room(24, 16, 6, 1, nu=40, nv=8, glass=True))


def test_camera_rebuild_soup_with_sky_defocus_and_spheres():
    check_camera_rebuild(_soup_with_sky_and_defocus)


@pytest.mark.parametrize("tlas", [-1, 0, 1])
def test_camera_rebuild_above_128_models_with_the_tlas(tlas):
    check_camera_rebuild(lambda: scenes.instanced_knots(24, 16, 4, 1, instances=150), ({"tlas": tlas},))


def test_camera_rebuild_ten_thousand_spheres_with_the_accelerator():
    check_camera_rebuild(lambda: scenes.random_soup(24, 16, 4, 1, triangles=300, spheres=10000))


def test_camera_rebuild_unity_fixture():
    from test_round2_abi import load_fixture
    check_camera_rebuild(lambda: load_fixture(24, 16))


# ---- arbitrary rays ---------------------------------------------------------------------------------------------------------------
def path_rays(sc, seed=0, n=None):
    """Every ray of the rtTraceRays ray sets (pick rays, in-scene origins, just inside meshes, far origins, direction lengths
    1e-23 .. 3e19, NaN / inf / zero directions) with random RNG states."""
    rays = np.concatenate(list(T.ray_sets(sc, seed=seed, n=n or RAYS).values()))
    states = np.random.RandomState(seed + 1).randint(0, 2 ** 32, size=len(rays), dtype=np.uint64).astype(np.uint32)
    return capi.make_path_rays(rays["origin"], rays["dir"], states)


def assert_radiance_equal(a, b, what):
    assert_bit_equal(np.ascontiguousarray(a["rgb"]), np.ascontiguousarray(b["rgb"]), f"{what}: rgb")
    bad = np.flatnonzero(a["rngState"] != b["rngState"])
    assert len(bad) == 0, f"{what}: rngState differs for {len(bad)} rays, first {bad[0]}: {a[bad[0]]} vs {b[bad[0]]}"


def check_rays(sc, rays, options_list=({},), samples=(1, 3, 16), bounces=(0, 4, 12), sky=(0, 1)):
    cases = [(s, m, u) for s in samples for m in bounces for u in sky]
    ref_mgr = T.open_mgr(ORACLE_LIB, sc)
    ref = {}
    for s, m, u in cases:
        ref_mgr.context.set_int("MaxBounceCount", m)
        ref_mgr.context.set_int("UseSky", u)
        ref[(s, m, u)] = ref_mgr.context.trace_paths(rays, s)
    ref_mgr.OnDestroy()
    for opts in options_list:
        for skip in ((opts["modelSkip"],) if "modelSkip" in opts else (1, 0)):
            mgr = T.open_mgr(CUDA_LIB, sc, dict(opts, modelSkip=skip))
            for (s, m, u), want in ref.items():
                mgr.context.set_int("MaxBounceCount", m)
                mgr.context.set_int("UseSky", u)
                got = mgr.context.trace_paths(rays, s)
                assert got.dtype == capi.PATH_RADIANCE_DTYPE and got.shape == (len(rays),)
                assert_radiance_equal(got, want, f"{sc.name} {opts} modelSkip={skip} samples={s} MaxBounceCount={m} UseSky={u}")
            mgr.OnDestroy()
    return ref


def test_arbitrary_rays_knot_room_with_glass():
    sc = scenes.knot_room(24, 16, 4, 1, nu=40, nv=8, glass=True)
    ref = check_rays(sc, path_rays(sc, seed=1))
    lit = ref[(3, 4, 1)]["rgb"]
    assert np.isfinite(lit).any() and (lit[np.isfinite(lit)] > 0).any()


def test_arbitrary_rays_soup_with_spheres():
    sc = scenes.random_soup(24, 16, 4, 1, triangles=300, spheres=200)
    check_rays(sc, path_rays(sc, seed=2), samples=(1, 16), bounces=(0, 12))


def test_arbitrary_rays_above_128_models():
    sc = scenes.instanced_knots(24, 16, 4, 1, instances=150)
    check_rays(sc, path_rays(sc, seed=3), ({"tlas": 1},), samples=(1, 3), bounces=(4,))


def test_arbitrary_rays_ten_thousand_spheres_with_the_accelerator():
    sc = scenes.random_soup(24, 16, 4, 1, triangles=300, spheres=10000)
    check_rays(sc, path_rays(sc, seed=4), ({}, {"extInstantiation": 1}), samples=(3,), bounces=(12,), sky=(1,))


def test_directions_of_every_length():
    """In-scene origins with unit directions scaled by 1e-23 .. 3e19: the first segment takes the linear loop outside
    |dir| in [2^-10, 2^10], and its hit point starts the next segment, which the per-segment gate tests again."""
    sc = scenes.knot_room(24, 16, 4, 1, nu=40, nv=8, glass=True)
    sc.spheres = scenes.random_soup(8, 8, 1, 1, triangles=3, spheres=80).spheres
    base = T.ray_sets(sc, seed=31, n=max(RAYS // 8, 8))["inside"]
    unit = base["dir"] / np.linalg.norm(base["dir"], axis=1, keepdims=True)
    o = np.concatenate([base["origin"]] * len(T.DIRECTION_SCALES))
    d = np.concatenate([unit.astype(np.float64) * s for s in T.DIRECTION_SCALES])
    rays = capi.make_path_rays(o, d, np.arange(len(o), dtype=np.uint32) * np.uint32(2654435761))
    check_rays(sc, rays, samples=(3,), bounces=(6,), sky=(1,))


# ---- chaining ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S", [2, 5])
def test_chained_single_samples_equal_one_call(S):
    sc = scenes.knot_room(24, 16, 6, 1, nu=40, nv=8, glass=True)
    rays = path_rays(sc, seed=5, n=max(RAYS // 4, 16))
    for lib in (ORACLE_LIB, CUDA_LIB):
        mgr = T.open_mgr(lib, sc)
        ctx = mgr.context
        ctx.set_int("UseSky", 1)
        one = ctx.trace_paths(rays, S)
        r = rays.copy()
        total = np.zeros((len(r), 3), dtype=np.float32)
        for _ in range(S):
            out = ctx.trace_paths(r, 1)
            total = (total + out["rgb"]).astype(np.float32)
            r["rngState"] = out["rngState"]
        chained = np.zeros(len(r), dtype=capi.PATH_RADIANCE_DTYPE)
        chained["rgb"] = (total / np.float32(S)).astype(np.float32)
        chained["rngState"] = r["rngState"]
        assert_radiance_equal(chained, one, f"{lib}: {S} chained calls vs samples={S}")
        mgr.OnDestroy()


def test_a_ray_that_misses_consumes_no_draws():
    sc = scenes.knot_room(24, 16, 4, 1, nu=40, nv=8)
    rng = np.random.RandomState(6)
    n = 64
    o = np.tile([[0.0, 1e4, 0.0]], (n, 1))
    d = np.abs(rng.normal(size=(n, 3))) * [0.2, 1.0, 0.2]                 # upwards, away from the room
    rays = capi.make_path_rays(o, d, rng.randint(0, 2 ** 32, size=n, dtype=np.uint64))
    for lib in (ORACLE_LIB, CUDA_LIB):
        mgr = T.open_mgr(lib, sc)
        for sky in (0, 1):
            mgr.context.set_int("UseSky", sky)
            out = mgr.context.trace_paths(rays, 7)
            assert (out["rngState"] == rays["rngState"]).all(), lib
            assert (out["rgb"] == 0).all() != bool(sky), lib
        mgr.OnDestroy()


# ---- isolation and counters -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["knot", "soup"])
def test_queries_between_frames_change_nothing_the_frames_show(name):
    sc = (scenes.instanced_knots(32, 24, 4, 2, instances=150) if name == "knot" else
          scenes.random_soup(32, 24, 4, 1, triangles=600, spheres=300))
    rays = path_rays(sc, seed=7, n=max(RAYS // 4, 16))
    images = []
    for with_queries in (False, True):
        mgr = T.open_mgr(CUDA_LIB, sc, {"countStats": 1})
        ctx = mgr.context
        ctx.reset_stats()
        for _ in range(3):
            mgr.RenderFrame()
            if with_queries:
                before, frame = ctx.stats(), mgr.raytraceFrameTex
                ctx.trace_paths(rays, 2)
                after = ctx.stats()
                assert after["dispatches"] == before["dispatches"] and after["kernelMs"] == before["kernelMs"]
                assert after["rays"] > before["rays"]
                assert_bit_equal(mgr.raytraceFrameTex, frame, "FrameRender right after a query")
        images.append((mgr.raytraceFrameTex, mgr.accumulatedResult, ctx.stats(), ctx.pixel_stats()))
        mgr.OnDestroy()
    assert_bit_equal(images[1][0], images[0][0], "FrameRender with queries in between")
    assert_bit_equal(images[1][1], images[0][1], "AccumulatedRender with queries in between")
    assert images[1][3].tobytes() == images[0][3].tobytes(), "PixelStats with queries in between"
    assert images[1][2]["dispatches"] == images[0][2]["dispatches"] == 3


def test_camera_frame_seed_and_samples_per_pixel_do_not_change_a_query():
    sc = scenes.knot_room(24, 16, 4, 1, nu=40, nv=8, glass=True)
    rays = path_rays(sc, seed=8, n=max(RAYS // 4, 16))
    for lib in (ORACLE_LIB, CUDA_LIB):
        mgr = T.open_mgr(lib, sc)
        ctx = mgr.context
        want = ctx.trace_paths(rays, 3)
        ctx.set_int("Frame", 17)
        ctx.set_int("renderSeed", 999)
        ctx.set_int("NumRaysPerPixel", 7)
        ctx.set_matrix("CamLocalToWorldMatrix", np.eye(4, dtype=np.float32) * 2.0)
        assert_radiance_equal(ctx.trace_paths(rays, 3), want, f"{lib}: after Frame / renderSeed / camera / NumRaysPerPixel changed")
        mgr.OnDestroy()


@pytest.mark.parametrize("name", ["knot", "spheres"])
def test_rays_grow_by_the_segments_and_counters_equal_the_oracle(name):
    sc = scenes.knot_room(24, 16, 6, 1, nu=40, nv=8, glass=True) if name == "knot" else scenes.random_soup(24, 16, 6, 1, triangles=300, spheres=40)
    rays = path_rays(sc, seed=9, n=max(RAYS // 4, 16))
    stats = {}
    for lib in (ORACLE_LIB, CUDA_LIB):
        for count in (0, 1):
            mgr = T.open_mgr(lib, sc, {"countStats": count})
            ctx = mgr.context
            ctx.reset_stats()
            ctx.trace_paths(rays, 4)
            stats[(lib, count)] = ctx.stats()
            mgr.OnDestroy()
    want = stats[(ORACLE_LIB, 1)]
    assert want["rays"] > 4 * len(rays) // 2          # segments, not rays: most paths bounce
    assert stats[(CUDA_LIB, 0)]["rays"] == want["rays"]
    got = stats[(CUDA_LIB, 1)]
    assert all(got[k] == want[k] for k in T.COUNTS), (got, want)
    assert got["dispatches"] == 0 and got["kernelMs"] == 0


def test_query_before_any_resize_and_after_the_scene_changed():
    sc = scenes.instanced_knots(24, 16, 4, 1, instances=12)
    sc.spheres = scenes.cornell_spheres().spheres[6:8].copy()
    rays = path_rays(sc, seed=10, n=max(RAYS // 4, 16))
    out = {}
    for lib in (ORACLE_LIB, CUDA_LIB):
        mgr = T.open_mgr(lib, sc, enable=False)          # no OnEnable: no rtResize, no dispatch
        first = mgr.trace_paths(rays, 2)
        mgr.OnEnable()
        mgr.RenderFrame()
        l2w, w2l = scenes.trs(position=(0.2, 1.5, 0.0), euler_deg=(10, 20, 30), scale=(0.3, 0.3, 0.3))
        mgr.set_model_transform(4, l2w, w2l)
        sph = sc.spheres.copy()
        sph["centre"][0] = (0.1, 1.6, 0.2)
        mgr.set_spheres(sph)
        second = mgr.trace_paths(rays, 2)
        out[lib] = (first, second)
        mgr.OnDestroy()
    assert_radiance_equal(out[CUDA_LIB][0], out[ORACLE_LIB][0], "before rtResize")
    assert_radiance_equal(out[CUDA_LIB][1], out[ORACLE_LIB][1], "after ModelInfo / Spheres changed")
    assert out[CUDA_LIB][0].tobytes() != out[CUDA_LIB][1].tobytes(), "the second query did not see the new scene"


# ---- refusals ---------------------------------------------------------------------------------------------------------------------
def test_empty_batch_and_every_error_code():
    sc = scenes.knot_room(16, 12, 3, 1, nu=30, nv=6)
    for lib in (ORACLE_LIB, CUDA_LIB):
        mgr = T.open_mgr(lib, sc)
        ctx, L, h = mgr.context, mgr.context._L, mgr.context.handle
        r = path_rays(sc, n=8)[:8].copy()
        out = np.zeros(len(r), dtype=capi.PATH_RADIANCE_DTYPE)
        st = ctx.stats()
        assert L.rtTracePaths(h, None, 0, 1, None) == capi.RT_OK and ctx.stats()["rays"] == st["rays"]
        assert len(ctx.trace_paths(np.zeros(0, dtype=capi.PATH_RAY_DTYPE), 1)) == 0
        assert L.rtTracePaths(None, r.ctypes.data, len(r), 1, out.ctypes.data) == capi.RT_E_INVALID
        assert L.rtTracePaths(h, r.ctypes.data, -1, 1, out.ctypes.data) == capi.RT_E_INVALID
        assert L.rtTracePaths(h, None, len(r), 1, out.ctypes.data) == capi.RT_E_INVALID
        assert L.rtTracePaths(h, r.ctypes.data, len(r), 1, None) == capi.RT_E_INVALID
        for s in (0, -1, capi.RT_MAX_BATCH_SAMPLES + 1):
            assert L.rtTracePaths(h, r.ctypes.data, len(r), s, out.ctypes.data) == capi.RT_E_INVALID, s
        for m in (-1, 201):
            ctx.set_int("MaxBounceCount", m)
            assert L.rtTracePaths(h, r.ctypes.data, len(r), 1, out.ctypes.data) == capi.RT_E_STATE, m
            assert L.rtTracePaths(h, r.ctypes.data, 0, 1, out.ctypes.data) == capi.RT_OK
        ctx.set_int("MaxBounceCount", 200)
        assert L.rtTracePaths(h, r.ctypes.data, len(r), 1, out.ctypes.data) == capi.RT_OK
        ctx.set_int("MaxBounceCount", 0)
        assert L.rtTracePaths(h, r.ctypes.data, len(r), 1, out.ctypes.data) == capi.RT_OK
        ctx.set_int("modelCount", 99)
        assert L.rtTracePaths(h, r.ctypes.data, len(r), 1, out.ctypes.data) == capi.RT_E_STATE
        ctx.set_int("modelCount", 2)
        models = np.zeros(2, dtype=capi.MODEL_DTYPE)
        models[1]["nodeOffset"] = 10 ** 7
        ctx.set_buffer("ModelInfo", models)
        assert L.rtTracePaths(h, r.ctypes.data, len(r), 1, out.ctypes.data) == capi.RT_E_STATE
        ctx.set_buffer("Nodes", np.zeros(0, dtype=capi.NODE_DTYPE))
        assert L.rtTracePaths(h, r.ctypes.data, len(r), 1, out.ctypes.data) == capi.RT_E_STATE
        assert L.rtTracePathsDevice(None, None, None, 0, 1) == capi.RT_E_INVALID
        if lib == CUDA_LIB:                              # (the oracle has no device form: RT_E_STATE)
            assert L.rtTracePathsDevice(h, None, None, 0, 0) == capi.RT_E_INVALID
            assert L.rtTracePathsDevice(h, None, None, 0, 1) == capi.RT_OK
        mgr.OnDestroy()
    from test_round2_abi import chain_bvh, one_model_scene
    for lib in (ORACLE_LIB, CUDA_LIB):
        mgr = T.open_mgr(lib, one_model_scene(16, 12))
        tris, nodes = chain_bvh(64)
        mgr.context.set_buffer("Triangles", tris)
        mgr.context.set_buffer("Nodes", nodes)
        with pytest.raises(capi.RtError) as e:
            mgr.context.trace_paths(capi.make_path_rays(np.zeros((1, 3)), np.ones((1, 3)), 1), 1)
        assert e.value.code == capi.RT_E_STATE and "too deep" in str(e.value), lib
        mgr.OnDestroy()


def test_cpp_manager_equals_the_python_context():
    sc = scenes.knot_room(24, 16, 4, 1, nu=40, nv=8, glass=True)
    rays = path_rays(sc, seed=41, n=max(RAYS // 4, 16))
    for lib in (ORACLE_LIB, CUDA_LIB):
        mgr = T.open_mgr(lib, sc)
        assert_radiance_equal(mgr.trace_paths(rays, 3), mgr.context.trace_paths(rays, 3), f"{lib}: RayComputeManager.TracePaths vs the context")
        mgr.OnDestroy()


# ---- GPU only ---------------------------------------------------------------------------------------------------------------------
def test_device_pointer_form_on_the_context_stream_and_a_caller_stream():
    torch = pytest.importorskip("torch")
    sc = scenes.instanced_knots(24, 16, 4, 1, instances=150)
    rays = path_rays(sc, seed=11)
    mgr = T.open_mgr(CUDA_LIB, sc)
    ctx = mgr.context
    want = ctx.trace_paths(rays, 3)
    raw = torch.zeros(len(rays) * 28 + 4, dtype=torch.uint8)
    raw[4:] = torch.from_numpy(rays.view(np.uint8).copy())
    d_raw = raw.cuda()
    for stream in (None, torch.cuda.Stream()):
        d_out = torch.full((len(rays) * 16 + 16,), 0x5a, dtype=torch.uint8, device="cuda")
        if stream is not None:
            ctx.set_stream(stream.cuda_stream)
        ctx.trace_paths_device(d_raw.data_ptr() + 4, d_out.data_ptr(), len(rays), 3)       # 4-byte aligned rays
        ctx.synchronize()
        got = d_out.cpu().numpy()
        assert (got[len(rays) * 16:] == 0x5a).all()
        assert_radiance_equal(got[: len(rays) * 16].view(capi.PATH_RADIANCE_DTYPE), want, f"device form, stream {stream}")
    ctx.set_stream(0)
    for rp, op in ((d_raw.data_ptr() + 2, d_out.data_ptr()), (d_raw.data_ptr() + 4, d_out.data_ptr() + 4)):
        with pytest.raises(capi.RtError) as e:
            ctx.trace_paths_device(rp, op, len(rays), 1)
        assert e.value.code == capi.RT_E_INVALID
    mgr.OnDestroy()
    o = capi.RtLib(ORACLE_LIB).create(0)
    assert o._L.rtTracePathsDevice(o.handle, None, None, 0, 1) == capi.RT_E_STATE


def test_two_million_camera_paths_on_the_871k_triangle_cluster():
    """1920 x 1080 camera rays and post-jitter states (two batches of the host form, the second partial) at MaxBounceCount 12 against
    a seeded 20k-ray oracle sample."""
    sc = scenes.knot_cluster(1920, 1080, 12, 1)
    ref = T.open_mgr(ORACLE_LIB, sc)
    rays = camera_samples(ref.context, 1920, 1080)
    mgr = T.open_mgr(CUDA_LIB, sc)
    got = mgr.context.trace_paths(rays, 1)
    mgr.OnDestroy()
    sub = np.random.RandomState(13).choice(len(rays), 20_000, replace=False)
    want = ref.context.trace_paths(rays[sub], 1)
    ref.OnDestroy()
    assert_radiance_equal(got[sub], want, "2M camera paths, seeded 20k subset")
    assert (got["rngState"] != rays["rngState"]).mean() > 0.5
