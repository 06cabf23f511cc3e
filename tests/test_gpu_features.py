"""rtDispatchFeatures / rtCameraRays on the H100 (`-m gpu`): the first-hit feature images (albedo, dst, normal, object id, and the two
accumulators) and the camera's own rays equal the oracle's bit for bit — across scenes, options, frames and seeds; closing the loop on
the product alone (rtTracePaths on rtCameraRays rebuilds a 1-sample frame, rtTraceRays on them rebuilds FeatureFrame); accumulation,
resets, resize, partial dispatch and row bands; what the call reads and leaves alone; the materials; every refusal.  The same bodies
run in the CPU suite against the SIMT interpreter build (tests/test_simt_features.py)."""
import numpy as np
import pytest

from conftest import CUDA_LIB, ORACLE_LIB, assert_bit_equal
import ray_tracing_b200 as rt
from ray_tracing_b200 import capi, scenes
import test_gpu_trace_paths as G
import test_gpu_trace_rays as T

pytestmark = pytest.mark.gpu

FRAME = (40, 24)                # size of the images (the interpreter twin uses a smaller one)
IMAGES = capi.FEATURE_IMAGES


def open_ctx(lib, sc, options=None, size=None):
    """A manager of the scene at `size` after OnEnable (scene uploaded, Frame = 1), and its context."""
    sc.width, sc.height = size or FRAME
    mgr = T.open_mgr(lib, sc, options)
    return mgr, mgr.context


def images(ctx):
    return {name: ctx.readback(name) for name in IMAGES}


def assert_features_equal(a, b, what):
    for f in ("albedo", "dst", "normal"):
        assert_bit_equal(np.ascontiguousarray(a[f]), np.ascontiguousarray(b[f]), f"{what}: FeatureFrame.{f}")
    bad = np.argwhere(a["object"] != b["object"])
    assert len(bad) == 0, f"{what}: object differs for {len(bad)} pixels, first {bad[0].tolist()}: {a[tuple(bad[0])]} vs {b[tuple(bad[0])]}"


def assert_images_equal(a, b, what):
    assert_features_equal(a["FeatureFrame"], b["FeatureFrame"], what)
    for name in IMAGES[1:]:
        assert_bit_equal(a[name], b[name], f"{what}: {name}")


def assert_rays_equal(a, b, what):
    for f in ("origin", "dir"):
        assert_bit_equal(np.ascontiguousarray(a[f]), np.ascontiguousarray(b[f]), f"{what}: {f}")
    assert (a["rngState"] == b["rngState"]).all(), f"{what}: rngState"


def run_features(ctx, frames=(1, 2)):
    for f in frames:
        ctx.set_int("Frame", f)
        ctx.dispatch_features()
    return images(ctx)


def check_scene(make, options_list=({},), frames=(1, 2), size=None):
    """FeatureFrame and both accumulators after feature dispatches of `frames`, against the oracle, for each option set (model skipping
    on and off unless given)."""
    mgr, octx = open_ctx(ORACLE_LIB, make(), size=size)
    want = run_features(octx, frames)
    mgr.OnDestroy()
    for opts in options_list:
        for skip in ((opts["modelSkip"],) if "modelSkip" in opts else (1, 0)):
            o = dict(opts, modelSkip=skip)
            mgr, ctx = open_ctx(CUDA_LIB, make(), o, size=size)
            assert_images_equal(run_features(ctx, frames), want, f"{make().name} {o}")
            mgr.OnDestroy()
    return want


def checker_soup():
    """The soup with sky, defocus, diverge and spheres over a checkered floor."""
    sc = scenes.random_soup(24, 16, 4, 1, triangles=400, spheres=60)
    sc.spheres["radius"] *= 6                                  # large enough to show in a small image
    sc.meshes.append(scenes.quad_mesh((-14, -9, -14), (-14, -9, 14), (14, -9, 14), (14, -9, -14)))
    sc.models.append(scenes.ModelDesc(len(sc.meshes) - 1, np.eye(4), np.eye(4),
                                      scenes.material(diffuse=(0.9, 0.1, 0.1), emission=(0.1, 0.1, 0.9), flag=scenes.MAT_CHECKER)))
    sc.settings = dict(sc.settings, useSky=True, defocusStrength=40.0, divergeStrength=2.5, focusDistance=6.0)
    return sc


# ---- 1. the camera's own rays -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["cornell", "soup"])
def test_camera_rays_equal_the_oracles_camera_sample(name):
    make = (lambda: scenes.cornell_spheres(24, 16, 4, 1)) if name == "cornell" else checker_soup
    w, h = FRAME
    for size in (FRAME, (1, h), (w, 1), (1, 1)):              # one pixel wide / high: uv = 0 / 0 (NaN), as the reference computes it
        omgr, octx = open_ctx(ORACLE_LIB, make(), size=size)
        mgr, ctx = open_ctx(CUDA_LIB, make(), size=size)
        for frame, seed in ((1, 12345), (7, 12345), (-1, 12345), (7, -77)):
            for c in (octx, ctx):
                c.set_int("Frame", frame)
                c.set_int("renderSeed", seed)
            want = G.camera_samples(octx, *size).reshape(size[1], size[0])
            what = f"{name} {size} Frame={frame} renderSeed={seed}"
            assert_rays_equal(octx.camera_rays(), want, f"{what}: the oracle's rtCameraRays vs orCameraSample")
            assert_rays_equal(ctx.camera_rays(), want, what)
        ctx.set_tile(1, 3, 2)                                  # a query about the camera: tiles do not apply
        assert_rays_equal(ctx.camera_rays(), want, f"{name} {size}: with rtSetTile")
        assert_rays_equal(mgr.camera_rays(), mgr.context.camera_rays(), f"{name} {size}: the manager's CameraRays (Frame 1)")
        mgr.OnDestroy()
        omgr.OnDestroy()


# ---- 2. closing the loop on the product alone ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["cornell", "knot", "soup"])
def test_paths_and_hits_of_the_camera_rays_rebuild_the_frame_and_the_features(name):
    make = {"cornell": lambda: scenes.cornell_spheres(24, 16, 4, 1), "knot": lambda: scenes.knot_room(24, 16, 6, 1, nu=40, nv=8, glass=True),
            "soup": checker_soup}[name]
    for kernel in (0, 1, 2):
        mgr, ctx = open_ctx(CUDA_LIB, make(), {"kernel": kernel})
        ctx.set_int("Frame", 3)
        ctx.set_int("NumRaysPerPixel", 1)
        rays = ctx.camera_rays()
        ctx.dispatch_full()
        ctx.dispatch_features()
        frame = ctx.readback("FrameRender")
        assert_bit_equal(ctx.trace_paths(rays.reshape(-1), 1)["rgb"].reshape(frame.shape[0], frame.shape[1], 3), frame[..., :3],
                         f"{name} kernel {kernel}: rtTracePaths(rtCameraRays) vs FrameRender")
        hits = ctx.trace_rays(rays["origin"].reshape(-1, 3), rays["dir"].reshape(-1, 3)).reshape(rays.shape)
        feat = ctx.readback("FeatureFrame")
        assert_bit_equal(hits["dst"], feat["dst"], f"{name}: rtTraceRays dst vs FeatureFrame")
        assert_bit_equal(np.ascontiguousarray(hits["normal"]), np.ascontiguousarray(feat["normal"]), f"{name}: rtTraceRays normal vs FeatureFrame")
        obj = np.where(hits["kind"] == capi.RT_HIT_SPHERE, -2 - hits["index"], hits["index"])
        assert (obj == feat["object"]).all(), f"{name}: object ids"
        assert (hits["kind"] != capi.RT_HIT_NONE).any()
        mgr.OnDestroy()


# ---- 3. the images against the oracle -----------------------------------------------------------------------------------------------
def test_cornell_spheres():
    want = check_scene(lambda: scenes.cornell_spheres(24, 16, 4, 1), ({}, {"extInstantiation": 1}, {"countStats": 1}))
    assert (want["FeatureFrame"]["object"] <= -2).all()


def test_knot_room_with_glass():
    want = check_scene(lambda: scenes.knot_room(24, 16, 6, 1, nu=40, nv=8, glass=True), ({}, {"countStats": 1}))
    f = want["FeatureFrame"]
    assert ((f["albedo"] == 1).all(axis=-1) & (f["object"] >= 0)).any(), "no glass pixel in the image"


def test_checker_soup_with_sky_defocus_and_spheres():
    want = check_scene(checker_soup, ({}, {"extInstantiation": 1}))
    obj = want["FeatureFrame"]["object"]
    assert (obj == -1).any() and (obj <= -2).any() and (obj >= 0).any()


@pytest.mark.parametrize("tlas", [-1, 0, 1])
def test_152_instanced_knots_with_the_tlas(tlas):
    check_scene(lambda: scenes.instanced_knots(24, 16, 4, 1, instances=150), ({"tlas": tlas},))


def test_ten_thousand_spheres_with_the_accelerator():
    check_scene(lambda: scenes.random_soup(24, 16, 4, 1, triangles=300, spheres=10000), ({}, {"countStats": 1}))


def test_unity_fixture():
    from test_round2_abi import load_fixture
    check_scene(lambda: load_fixture(24, 16))


# ---- 4. accumulation, resets, resize, partial dispatch, bands -------------------------------------------------------------------------
def test_accumulation_resets_and_resize():
    for lib in (ORACLE_LIB, CUDA_LIB):
        mgr, ctx = open_ctx(lib, checker_soup())
        h, w = ctx.height, ctx.width
        alb = np.zeros((h, w, 4), np.float32)
        nrm = np.zeros((h, w, 4), np.float32)
        for frame in range(1, 6):
            ctx.set_int("Frame", frame)
            ctx.dispatch_features()
            f = ctx.readback("FeatureFrame")
            hit = (f["object"] != -1)[..., None]
            alb = np.where(hit, (alb + np.concatenate([f["albedo"], np.ones((h, w, 1), np.float32)], axis=-1)).astype(np.float32), alb)
            nrm = np.where(hit, (nrm + np.concatenate([f["normal"], np.where(hit, f["dst"][..., None], 0).astype(np.float32)], axis=-1)).astype(np.float32), nrm)
        got = images(ctx)
        assert_bit_equal(got["AccumulatedAlbedo"], alb, f"{lib}: AccumulatedAlbedo = the float sums in frame order")
        assert_bit_equal(got["AccumulatedNormal"], nrm, f"{lib}: AccumulatedNormal = the float sums in frame order")
        miss = got["FeatureFrame"]["object"] == -1
        assert miss.any() and np.isposinf(got["FeatureFrame"]["dst"][miss]).all() and (got["FeatureFrame"]["normal"][miss] == 0).all()
        assert got["AccumulatedAlbedo"][..., 3].max() == 5

        ctx.set_bool("accumulate", False)                      # FeatureFrame only
        ctx.set_int("Frame", 9)
        ctx.dispatch_features()
        after = images(ctx)
        assert after["FeatureFrame"].tobytes() != got["FeatureFrame"].tobytes()
        assert_bit_equal(after["AccumulatedAlbedo"], got["AccumulatedAlbedo"], f"{lib}: accumulate = 0")
        assert_bit_equal(after["AccumulatedNormal"], got["AccumulatedNormal"], f"{lib}: accumulate = 0")

        ctx.dispatch(capi.RT_KERNEL_RESET_ACCUMULATED, 2, 1)   # ResetAccumulated over 16 x 8 pixels, then over the image
        part = images(ctx)
        assert (part["AccumulatedAlbedo"][:8, :16] == 0).all() and (part["AccumulatedNormal"][:8, :16] == 0).all()
        assert_bit_equal(part["AccumulatedAlbedo"][8:], got["AccumulatedAlbedo"][8:], f"{lib}: partial reset")
        ctx.dispatch_full(capi.RT_KERNEL_RESET_ACCUMULATED)
        reset = images(ctx)
        assert (reset["AccumulatedAlbedo"] == 0).all() and (reset["AccumulatedNormal"] == 0).all()
        assert reset["FeatureFrame"].tobytes() == after["FeatureFrame"].tobytes(), f"{lib}: ResetAccumulated leaves FeatureFrame"

        ctx.set_bool("accumulate", True)
        ctx.dispatch_features()
        ctx.resize(w + 8, h)                                   # a new size zeroes all three
        ctx.set_ints("Resolution", [w + 8, h])
        for name, img in images(ctx).items():
            assert img.shape[:2] == (h, w + 8) and not np.frombuffer(img.tobytes(), np.uint8).any(), f"{lib}: {name} after a resize"
        mgr.OnDestroy()


def test_partial_dispatch_and_three_rank_bands_reassemble_the_image():
    make = lambda: scenes.knot_room(24, 16, 6, 1, nu=40, nv=8, glass=True)
    mgr, octx = open_ctx(ORACLE_LIB, make())
    whole = run_features(octx, (1, 2))
    mgr.OnDestroy()
    h, w = whole["FeatureFrame"].shape
    for lib in (ORACLE_LIB, CUDA_LIB):
        mgr, ctx = open_ctx(lib, make())
        ctx.set_int("Frame", 1)
        ctx.dispatch_features(2, 1)                            # 16 x 8 pixels
        got = images(ctx)
        assert_features_equal(got["FeatureFrame"][:8, :16], run_one(make, 1)["FeatureFrame"][:8, :16], f"{lib}: partial dispatch")
        outside = np.ones((h, w), bool)
        outside[:8, :16] = False
        for name in IMAGES:
            assert not np.frombuffer(got[name][outside].tobytes(), np.uint8).any(), f"{lib}: {name} outside a partial dispatch"
        ctx.dispatch_features(gz=0)
        assert images(ctx)["FeatureFrame"].tobytes() == got["FeatureFrame"].tobytes()
        mgr.OnDestroy()

        parts = []
        for rank in range(3):
            mgr, ctx = open_ctx(lib, make())
            ctx.set_tile(rank, 3, 2)
            parts.append(run_features(ctx, (1, 2)))
            mgr.OnDestroy()
        rows = (np.arange(h) // 2) % 3
        for rank, p in enumerate(parts):
            for name in IMAGES:
                assert not np.frombuffer(p[name][rows != rank].tobytes(), np.uint8).any(), f"{lib}: rank {rank} wrote {name} outside its bands"
        joined = {name: parts[0][name].copy() for name in IMAGES}
        for name in IMAGES:
            for rank in (1, 2):
                joined[name][rows == rank] = parts[rank][name][rows == rank]
        assert_images_equal(joined, whole, f"{lib}: three ranks reassembled")


def run_one(make, frame):
    mgr, octx = open_ctx(ORACLE_LIB, make())
    out = run_features(octx, (frame,))
    mgr.OnDestroy()
    return out


# ---- 5. isolation and counters --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["knot", "soup"])
def test_feature_dispatches_between_frames_change_nothing_the_frames_show(name):
    make = (lambda: scenes.instanced_knots(32, 24, 4, 2, instances=150)) if name == "knot" else (lambda: scenes.random_soup(32, 24, 4, 1, triangles=600, spheres=300))
    results = []
    for with_features in (False, True):
        mgr, ctx = open_ctx(CUDA_LIB, make(), {"countStats": 1})
        ctx.reset_stats()
        for _ in range(3):
            if with_features:
                mgr.RenderFeatures()
            mgr.RenderFrame()
            if with_features:
                before, frame, accum, pix = ctx.stats(), mgr.raytraceFrameTex, mgr.accumulatedResult, ctx.pixel_stats()
                frames_before = mgr.numAccumulatedFrames
                mgr.RenderFeatures()
                after = ctx.stats()
                assert after["dispatches"] == before["dispatches"] and after["kernelMs"] == before["kernelMs"]
                assert after["rays"] == before["rays"] + ctx.width * ctx.height
                assert mgr.numAccumulatedFrames == frames_before
                assert_bit_equal(mgr.raytraceFrameTex, frame, "FrameRender right after a feature dispatch")
                assert_bit_equal(mgr.accumulatedResult, accum, "AccumulatedRender right after a feature dispatch")
                assert ctx.pixel_stats().tobytes() == pix.tobytes(), "PixelStats right after a feature dispatch"
        results.append((mgr.raytraceFrameTex, mgr.accumulatedResult, ctx.stats()))
        mgr.OnDestroy()
    assert_bit_equal(results[1][0], results[0][0], "FrameRender with feature dispatches in between")
    assert_bit_equal(results[1][1], results[0][1], "AccumulatedRender with feature dispatches in between")
    assert results[1][2]["dispatches"] == results[0][2]["dispatches"] == 3


def test_samples_per_pixel_bounce_limit_and_sky_do_not_change_a_feature():
    for lib in (ORACLE_LIB, CUDA_LIB):
        mgr, ctx = open_ctx(lib, checker_soup())
        ctx.dispatch_features()
        want = ctx.readback("FeatureFrame")
        ctx.set_int("NumRaysPerPixel", 7)
        ctx.set_int("MaxBounceCount", 500)
        ctx.set_int("UseSky", 0)
        ctx.set_float("SunIntensity", 99.0)
        ctx.dispatch_features()
        assert_features_equal(ctx.readback("FeatureFrame"), want, f"{lib}: after NumRaysPerPixel / MaxBounceCount / sky changed")
        mgr.OnDestroy()


@pytest.mark.parametrize("name", ["knot", "spheres"])
def test_rays_grow_by_the_pixels_and_counters_equal_the_oracle(name):
    make = (lambda: scenes.knot_room(24, 16, 6, 1, nu=40, nv=8, glass=True)) if name == "knot" else (lambda: scenes.random_soup(24, 16, 6, 1, triangles=300, spheres=40))
    stats = {}
    for lib in (ORACLE_LIB, CUDA_LIB):
        for count in (0, 1):
            mgr, ctx = open_ctx(lib, make(), {"countStats": count})
            ctx.reset_stats()
            ctx.dispatch_features()
            ctx.dispatch_features(2, 1)
            stats[(lib, count)] = ctx.stats()
            mgr.OnDestroy()
    want = stats[(ORACLE_LIB, 1)]
    assert want["rays"] == FRAME[0] * FRAME[1] + 16 * 8
    assert stats[(CUDA_LIB, 0)]["rays"] == want["rays"]
    got = stats[(CUDA_LIB, 1)]
    assert all(got[k] == want[k] for k in T.COUNTS), (got, want)
    assert got["dispatches"] == 0 and got["kernelMs"] == 0


# ---- 6. materials -------------------------------------------------------------------------------------------------------------------
def material_scene():
    """A wall of quads facing the camera, one material each: a checker board (cells of 2/3: many boundaries), glass, an emitter, NaN in
    specularCol, a quad facing away (culled: the quad behind it shows), and a quad in the plane where a sphere starts (equal dst)."""
    mats = [scenes.material(diffuse=(0.9, 0.2, 0.1), emission=(0.1, 0.2, 0.9), flag=scenes.MAT_CHECKER),
            scenes.material(flag=scenes.MAT_GLASS, ior=1.5, diffuse=(0.3, 0.3, 0.3)),
            scenes.material(diffuse=(0.2, 0.7, 0.2), emission=(1, 0.5, 0.25), emissionStrength=8.0),
            scenes.material(diffuse=(0.5, 0.5, 0.5), specular=(np.nan, np.inf, 1.0)),
            scenes.material(diffuse=(0.1, 0.1, 0.8)),
            scenes.material(diffuse=(0.8, 0.8, 0.1))]
    meshes, models = [], []

    def quad(x0, x1, z, mat, flip=False):
        p = [(x0, -1, z), (x0, 1, z), (x1, 1, z), (x1, -1, z)]
        meshes.append(scenes.quad_mesh(*(p[::-1] if flip else p)))
        models.append(scenes.ModelDesc(len(meshes) - 1, np.eye(4), np.eye(4), mat))

    for k in range(4):
        quad(-3 + 1.5 * k, -1.5 + 1.5 * k, 4.0, mats[k])
    quad(-3, 3, 3.5, mats[4], flip=True)                       # faces away from the camera: culled, the wall behind it shows
    quad(-3, 3, 6.0, mats[5])                                  # behind everything: never the winner where the wall is
    sph = np.zeros(2, dtype=capi.SPHERE_DTYPE)
    sph[0] = scenes._sphere((0.0, 2.0, 5.0), 1.0, scenes.material(flag=scenes.MAT_GLASS, ior=1.3))      # glass sphere above the wall
    sph[1] = scenes._sphere((0.0, -2.0, 5.0), 1.0, scenes.material(diffuse=(0.4, 0.1, 0.6)))
    cam, _ = scenes.trs(position=(0.0, 0.0, -2.0))
    return scenes.Scene(name="materials", width=40, height=24, spheres=sph, meshes=meshes, models=models, cam_local_to_world=cam, fov=70.0,
                        settings=dict(divergeStrength=0.0))


def test_materials_checker_glass_emitter_culled_and_nan():
    want = check_scene(material_scene, ({}, {"countStats": 1}), frames=(1,), size=(80, 48))
    f = want["FeatureFrame"]
    by_model = lambda m: f["albedo"][f["object"] == m]
    checker = by_model(0)
    assert len(np.unique(checker.round(3), axis=0)) == 2, "both checker colours"
    assert (by_model(1) == 1).all() and len(by_model(1)) > 0, "a glass mesh is white"
    assert (f["albedo"][f["object"] == -2] == 1).all() and (f["object"] == -2).any(), "a glass sphere is white"
    assert_bit_equal(by_model(2), np.broadcast_to(np.float32([0.2, 0.7, 0.2]), by_model(2).shape).copy(), "an emitter shows its diffuse colour")
    nan = by_model(3)
    assert len(nan) and np.isnan(nan[:, :2]).all() and (nan[:, 2] == 0.5).all(), "NaN where specularCol - col is not finite"
    assert not (f["object"] == 4).any(), "a back face of an opaque model is culled"
    assert (f["object"] == -3).any()


def test_a_sphere_and_a_model_at_equal_dst_the_sphere_wins():
    """An axis-aligned ray from the camera's origin meets a sphere's pole and a quad through it at the same float dst."""
    sc = material_scene()
    sc.spheres = sc.spheres[1:].copy()
    sc.spheres["centre"][0] = (0.0, 0.0, 5.0)                  # its near pole at z = 4: in the plane of the wall
    sc.settings = dict(sc.settings, divergeStrength=0.0, defocusStrength=0.0)
    for lib in (ORACLE_LIB, CUDA_LIB):
        mgr, ctx = open_ctx(lib, sc, size=(41, 25))            # odd size: the centre pixel looks straight along +z
        ctx.dispatch_features()
        f = ctx.readback("FeatureFrame")[12, 20]
        ray = ctx.camera_rays()[12, 20]
        hits = ctx.trace_rays(ray["origin"][None], ray["dir"][None])
        assert f["dst"] == 6.0 and f["object"] == -2, (lib, f)
        assert hits["kind"][0] == capi.RT_HIT_SPHERE and hits["dst"][0] == f["dst"]
        ctx.set_buffer("Spheres", np.zeros(0, dtype=capi.SPHERE_DTYPE))      # without the sphere the wall is hit at the same dst
        alone = ctx.trace_rays(np.float32([[0, 0, -2]]), np.float32([[0, 0, 1]]))
        assert alone["dst"][0] == 6.0 and alone["kind"][0] == capi.RT_HIT_MODEL, (lib, alone)
        mgr.OnDestroy()


# ---- 7. refusals and states -----------------------------------------------------------------------------------------------------------
def test_every_refusal_and_state():
    sc = scenes.knot_room(16, 12, 3, 1, nu=30, nv=6)
    for lib in (ORACLE_LIB, CUDA_LIB):
        mgr = T.open_mgr(lib, sc, enable=False)                # no OnEnable: no rtResize
        ctx, L, h = mgr.context, mgr.context._L, mgr.context.handle
        buf = np.zeros(16 * 12, dtype=capi.PATH_RAY_DTYPE)
        assert L.rtDispatchFeatures(h, 2, 2, 1) == capi.RT_E_STATE
        assert L.rtCameraRays(h, buf.ctypes.data, buf.nbytes) == capi.RT_E_STATE
        mgr.OnEnable()
        for name in IMAGES:                                    # before the first feature dispatch
            with pytest.raises(capi.RtError) as e:
                ctx.readback(name)
            assert e.value.code == capi.RT_E_STATE, (lib, name)
        assert L.rtDispatchFeatures(None, 2, 2, 1) == capi.RT_E_INVALID
        assert L.rtDispatchFeatures(h, -1, 2, 1) == capi.RT_E_INVALID
        assert L.rtCameraRays(None, buf.ctypes.data, buf.nbytes) == capi.RT_E_INVALID
        assert L.rtCameraRays(h, None, buf.nbytes) == capi.RT_E_INVALID
        assert L.rtCameraRays(h, buf.ctypes.data, buf.nbytes - 28) == capi.RT_E_INVALID
        assert L.rtCameraRaysDevice(None, None, 0) == capi.RT_E_INVALID
        assert L.rtCameraRays(h, buf.ctypes.data, buf.nbytes) == capi.RT_OK
        ctx.set_ints("Resolution", [8, 12])
        assert L.rtDispatchFeatures(h, 2, 2, 1) == capi.RT_E_STATE
        assert L.rtCameraRays(h, buf.ctypes.data, buf.nbytes) == capi.RT_E_STATE
        ctx.set_ints("Resolution", [16, 12])
        assert L.rtDispatchFeatures(h, 0, 0, 1) == capi.RT_OK   # covers nothing, allocates the images
        for name in IMAGES:
            assert not np.frombuffer(ctx.readback(name).tobytes(), np.uint8).any()
            out = np.zeros(16 * 12 * 9, np.float32)
            assert L.rtReadback(h, name.encode(), out.ctypes.data, out.nbytes) == capi.RT_E_INVALID
        ctx.set_int("modelCount", 99)
        assert L.rtDispatchFeatures(h, 2, 2, 1) == capi.RT_E_STATE
        assert L.rtCameraRays(h, buf.ctypes.data, buf.nbytes) == capi.RT_OK          # needs no scene
        ctx.set_int("modelCount", len(sc.models))
        assert L.rtDispatchFeatures(h, 2, 2, 1) == capi.RT_OK
        mgr.OnDestroy()


def test_cpp_manager_equals_the_raw_context():
    make = lambda: scenes.knot_room(24, 16, 4, 1, nu=40, nv=8, glass=True)
    for lib in (ORACLE_LIB, CUDA_LIB):
        mgr, _ = open_ctx(lib, make())
        for _ in range(2):
            mgr.RenderFeatures()
            mgr.RenderFrame()
        via_mgr = {"FeatureFrame": mgr.feature_frame, "AccumulatedAlbedo": mgr.accumulated_albedo, "AccumulatedNormal": mgr.accumulated_normal}
        rays = mgr.camera_rays()
        assert mgr.numAccumulatedFrames == 3
        mgr.ResetAccumulatedRender()
        assert (mgr.accumulated_albedo == 0).all() and (mgr.accumulated_normal == 0).all()
        mgr.OnDestroy()
        mgr, ctx = open_ctx(lib, make())
        assert_images_equal(via_mgr, run_features(ctx, (1, 2)), f"{lib}: RenderFeatures vs rtDispatchFeatures")
        ctx.set_int("Frame", 3)
        assert_rays_equal(rays, ctx.camera_rays(), f"{lib}: CameraRays vs rtCameraRays")
        mgr.OnDestroy()


# ---- 8. GPU only ------------------------------------------------------------------------------------------------------------------------
def test_group_context_is_refused():
    torch = pytest.importorskip("torch")
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    check_group_refusal(CUDA_LIB, [0, 1])


def check_group_refusal(lib, devices):
    sc = scenes.knot_room(16, 12, 3, 1, nu=30, nv=6)
    mgr = rt.RayComputeManager(lib, devices=devices)
    scenes.apply(sc, mgr)
    mgr.OnEnable()
    ctx = mgr.context
    with pytest.raises(capi.RtError) as e:
        ctx.dispatch_features()
    assert e.value.code == capi.RT_E_STATE and "group" in str(e.value)
    for name in IMAGES:
        with pytest.raises(capi.RtError) as e:
            ctx.readback(name)
        assert e.value.code == capi.RT_E_STATE
    assert ctx.camera_rays().shape == (12, 16)                 # the camera query works on the group's context
    mgr.OnDestroy()


def test_device_pointer_forms_on_the_context_stream_and_a_caller_stream():
    torch = pytest.importorskip("torch")
    mgr, ctx = open_ctx(CUDA_LIB, checker_soup())
    w, h = ctx.width, ctx.height
    ctx.set_int("Frame", 4)
    want = ctx.camera_rays()
    n = w * h * 28
    for stream in (None, torch.cuda.Stream()):
        d = torch.full((n + 4 + 16,), 0x5a, dtype=torch.uint8, device="cuda")
        if stream is not None:
            ctx.set_stream(stream.cuda_stream)
        ctx.camera_rays_device(d.data_ptr() + 4, n)            # 4-byte aligned
        ctx.dispatch_features()
        ctx.synchronize()
        got = d.cpu().numpy()
        assert (got[:4] == 0x5a).all() and (got[4 + n:] == 0x5a).all()
        assert_rays_equal(got[4:4 + n].view(capi.PATH_RAY_DTYPE).reshape(h, w), want, f"device form, stream {stream}")
        for name in IMAGES:
            ptr, nbytes = ctx.device_pointer(name)
            assert ptr and nbytes == w * h * (32 if name == "FeatureFrame" else 16)
    ctx.set_stream(0)
    with pytest.raises(capi.RtError) as e:
        ctx.camera_rays_device(d.data_ptr() + 2, n)
    assert e.value.code == capi.RT_E_INVALID
    with pytest.raises(capi.RtError) as e:
        ctx.camera_rays_device(d.data_ptr() + 4, n - 28)
    assert e.value.code == capi.RT_E_INVALID
    mgr.OnDestroy()
    o = capi.RtLib(ORACLE_LIB).create(0)
    assert o._L.rtCameraRaysDevice(o.handle, None, 0) == capi.RT_E_STATE


def test_4k_features_on_the_871k_triangle_cluster_against_a_sparse_oracle_sample():
    """3840 x 2160 feature rays against the oracle on ten seeded rows (38,400 pixels): bands of one row with the row as the rank make
    the oracle trace that row alone."""
    sc = scenes.knot_cluster(3840, 2160, 12, 1)
    mgr, ctx = open_ctx(CUDA_LIB, sc, size=(3840, 2160))
    ctx.dispatch_features()
    got = ctx.readback("FeatureFrame")
    mgr.OnDestroy()
    ys = np.sort(np.random.RandomState(21).choice(2160, 10, replace=False))
    omgr, octx = open_ctx(ORACLE_LIB, sc, size=(3840, 2160))
    for y in ys:
        octx.set_tile(int(y), 2160, 1)
        octx.dispatch_features()
    want = octx.readback("FeatureFrame")
    omgr.OnDestroy()
    assert_features_equal(got[ys], want[ys], "4K cluster, ten rows")
    assert (got["object"][ys] >= 0).all() and len(np.unique(got["object"][ys])) > 1      # the cluster stands in a closed room
