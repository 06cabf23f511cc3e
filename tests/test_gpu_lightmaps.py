"""rtBakeLightmap on the H100 (`-m gpu`): cosine-weighted path-traced lighting at surface texels equals the oracle's restatement bit for
bit, `rejected` and the counters included, on the seven scenes of the probe and cube-map tests with model skipping on and off,
MaxBounceCount 0 and 4 and sample counts around the chunk and tree edges, for vertex texels of the scene's meshes, random points and
normals, adversarial normals and far / NaN positions; a texel rebuilt sample by sample (orLightmapRays -> rtTracePaths(samples = 1) ->
the numpy chunk sums, padded tree and division of tests/test_gpu_cubemaps.py) equals the call; the hook's directions are a
cosine-weighted hemisphere; a furnace, the sky alone against float64, and the reference's own diffuse bounce; seeds and texel indices,
internal launches and host batches, isolation, n = 0 and every refusal, the device form, both managers.  The same bodies run in the CPU
suite against the SIMT interpreter build (tests/test_simt_lightmaps.py)."""
import ctypes as C

import numpy as np
import pytest

from conftest import CUDA_LIB, ORACLE_LIB, assert_bit_equal
from ray_tracing_b200 import capi, manager, scenes
import test_gpu_cubemaps as CM
import test_gpu_probes as P
import test_gpu_trace_paths as G
import test_gpu_trace_rays as T

pytestmark = pytest.mark.gpu

SAMPLES = (1, 31, 32, 33, 1025)                         # around a chunk (32) and a padded tree of 33 chunks
BOUNCES = (0, 4)
RANDOM = 3                                              # random points with random normals per set
VERTICES = 4                                            # vertex texels of the scene's meshes per set
SKY_SAMPLES = 4096                                      # the sky-alone integral and the direction statistics
BOUNCE_SAMPLES, BOUNCE_REF = 4096, 1 << 18              # the bake and the reference's diffuse bounce, per texel
U = 2.0 ** -24                                          # binary32 unit roundoff


# ---- helpers ----------------------------------------------------------------------------------------------------------------------
def surface_points(positions, normals):
    pts = np.zeros(len(positions), dtype=capi.SURFACE_POINT_DTYPE)
    pts["position"], pts["normal"] = np.asarray(positions, dtype=np.float32), np.asarray(normals, dtype=np.float32)
    return pts


ADVERSARIAL = np.array([(0, 0, 1), (0, 0, -1), (1, 0, -0.0), (1e-4, 0, -1), (0.0006, -0.0008, 0), (600, 0, 800), (0, 0, 0),
                        (1e-40, 0, 0), (np.nan, 0, 1), (np.inf, 0, 0), (0, -np.inf, 0)], dtype=np.float32)


def texel_set(sc, seed):
    """Vertex texels of the scene's models, random points (rtTraceRays' "inside" origins) with random normals of random length, the
    adversarial normals at one in-scene point (+-z, (1, 0, -0), nearly -z, lengths 1e-3 and 1e3, zero, denormal, NaN, +-inf), and a far
    and a NaN position, which fail the gate."""
    rng = np.random.RandomState(seed)
    parts = []
    if sc.models:
        vt = np.concatenate([manager.vertex_texels(sc.meshes[m.mesh].vertices, sc.meshes[m.mesh].normals, m.local_to_world)
                             for m in sc.models[:3]])
        parts.append(vt[rng.choice(len(vt), VERTICES, replace=False)])
    pos = P.probe_positions(sc, seed=seed, n=RANDOM + 1, special=False)
    nrm = rng.standard_normal((RANDOM, 3)) * rng.uniform(0.1, 10.0, (RANDOM, 1))
    parts.append(surface_points(pos[:RANDOM], nrm))
    parts.append(surface_points(np.repeat(pos[RANDOM:], len(ADVERSARIAL), axis=0), ADVERSARIAL))
    parts.append(surface_points([[1e5, 1e5, -1e5], [np.nan, 0.0, 0.0]], [[0, 1, 0], [0, 1, 0]]))
    return np.ascontiguousarray(np.concatenate(parts))


def lightmap_rays(octx, points, samples, seed):
    """orLightmapRays: every sample's start (o, d, H(H(seed + p) + k)) as n * samples PATH_RAY_DTYPE records."""
    L = octx._L
    L.orLightmapRays.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_uint32, C.c_void_p]
    pts = capi.as_surface_points(points)
    out = np.zeros(len(pts) * samples, dtype=capi.PATH_RAY_DTYPE)
    assert L.orLightmapRays(octx.handle, pts.ctypes.data, len(pts), samples, seed, out.ctypes.data) == capi.RT_OK
    return out


def oracle_texels(octx, points, samples, seed, first, count):
    """orLightmapTexels: texels first .. first + count - 1 of the call, from the oracle."""
    L = octx._L
    L.orLightmapTexels.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_uint32, C.c_int, C.c_int, C.c_void_p]
    pts = capi.as_surface_points(points)
    out = np.zeros(count, dtype=capi.CUBE_TEXEL_DTYPE)
    assert L.orLightmapTexels(octx.handle, pts.ctypes.data, len(pts), samples, seed, first, count, out.ctypes.data) == capi.RT_OK
    return out


def unit64(v):
    v = np.asarray(v, dtype=np.float64)
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


def bake(ctx, points, samples, seed, stats=False):
    ctx.reset_stats()
    out = ctx.bake_lightmap(points, samples, seed)
    return (out, ctx.stats()) if stats else out


def check_oracle(sc, points, options_list=({},), samples=None, bounces=None, seed=7, sky=None):
    """rtBakeLightmap against the oracle for every (samples, MaxBounceCount), each option set with modelSkip 1 and 0 and a counting
    run: texel bits, rejected, RtStats.rays and, counting, the box / triangle / sphere counters."""
    runs = [(s, m) for s in (samples or SAMPLES) for m in (bounces or BOUNCES)]
    ref_mgr = T.open_mgr(ORACLE_LIB, sc)
    if sky is not None:
        ref_mgr.context.set_int("UseSky", sky)
    ref = {}
    for s, m in runs:
        ref_mgr.context.set_int("MaxBounceCount", m)
        ref[(s, m)] = bake(ref_mgr.context, points, s, seed, stats=True)
    ref_mgr.OnDestroy()
    for opts in list(options_list) + [{"countStats": 1}]:
        for skip in ((opts["modelSkip"],) if "modelSkip" in opts else (1, 0)):
            mgr = T.open_mgr(CUDA_LIB, sc, dict(opts, modelSkip=skip))
            if sky is not None:
                mgr.context.set_int("UseSky", sky)
            for (s, m), (want, wst) in ref.items():
                mgr.context.set_int("MaxBounceCount", m)
                got, gst = bake(mgr.context, points, s, seed, stats=True)
                what = f"{sc.name} {opts} modelSkip={skip} samples={s} MaxBounceCount={m}"
                assert got.shape == (len(points),) and got.dtype == capi.CUBE_TEXEL_DTYPE
                CM.assert_texels_equal(got, want, what)
                keys = (P.COUNTS(sc) if opts.get("countStats") else ("rays",))
                assert all(gst[k] == wst[k] for k in keys), (what, gst, wst)
                assert gst["dispatches"] == 0 and gst["kernelMs"] == 0
            mgr.OnDestroy()
    return ref


def richest(ref):
    return ref[max(ref, key=lambda k: (k[1], k[0]))][0]


# ---- against the oracle -----------------------------------------------------------------------------------------------------------
def test_oracle_cornell_spheres():
    sc = scenes.cornell_spheres(24, 16, 4, 1)
    pts = texel_set(sc, 1)
    ref = check_oracle(sc, pts)
    assert (richest(ref)["rgb"][:RANDOM] > 0).any(axis=1).all()        # every random texel gathers some light


def test_oracle_knot_room_with_glass():
    sc = scenes.knot_room(24, 16, 4, 1, nu=40, nv=8, glass=True)
    check_oracle(sc, texel_set(sc, 2), sky=1)


def test_oracle_soup_with_sky_and_spheres():
    sc = G._soup_with_sky_and_defocus()
    check_oracle(sc, texel_set(sc, 3))


@pytest.mark.parametrize("tlas", [-1, 0, 1])
def test_oracle_above_128_models_with_the_tlas(tlas):
    sc = scenes.instanced_knots(24, 16, 4, 1, instances=150)
    check_oracle(sc, texel_set(sc, 4), ({"tlas": tlas},))


def test_oracle_ten_thousand_spheres_with_the_accelerator():
    sc = scenes.random_soup(24, 16, 4, 1, triangles=300, spheres=10000)
    check_oracle(sc, texel_set(sc, 5), ({}, {"extInstantiation": 1}), sky=1)


def test_oracle_unity_fixture():
    from test_round2_abi import load_fixture
    sc = load_fixture(24, 16)
    check_oracle(sc, texel_set(sc, 6))


def test_oracle_nan_sun_rejects_samples():
    """Every path that reaches the sky is NaN: those samples are counted in `rejected`, count as black, and every texel stays finite."""
    sc = scenes.random_soup(24, 16, max_bounces=3, rays_per_pixel=1, triangles=600, spheres=8)
    sc.settings["sunIntensity"] = float("nan")
    ref = check_oracle(sc, texel_set(sc, 8), sky=1)
    got = richest(ref)
    assert got["rejected"].sum() > 0 and np.isfinite(got["rgb"]).all()


# ---- the rebuild through rtTracePaths and the directions --------------------------------------------------------------------------
@pytest.mark.parametrize("samples", [33, 1025])
def test_rebuild_through_trace_paths(samples):
    """orLightmapRays -> this build's rtTracePaths(samples = 1) -> numpy: the chunk sums in k order, the padded tree and the division
    give rtBakeLightmap's bits, with and without a NaN sun; the hook's origins are the points lifted by 0.001 along the unit normal."""
    sc = scenes.knot_room(24, 16, 4, 1, nu=40, nv=8, glass=True)
    sc.settings = dict(sc.settings, useSky=True)
    pts = texel_set(sc, 9)
    ref = T.open_mgr(ORACLE_LIB, sc)
    mgr = T.open_mgr(CUDA_LIB, sc)
    for sun in (10.0, float("nan")):
        mgr.context.set_float("SunIntensity", sun)
        rays = lightmap_rays(ref.context, pts, samples, 21)
        want = CM.mean32(mgr.context.trace_paths(rays, 1)["rgb"], len(pts), samples)
        got = mgr.context.bake_lightmap(pts, samples, 21)
        assert_bit_equal(got["rgb"], want[0], f"SunIntensity={sun}: rgb")
        assert np.array_equal(got["rejected"], want[1]), f"SunIntensity={sun}: rejected"
        assert (want[1] > 0).any() == (sun != sun)
    f = np.float32
    m = pts["normal"][:RANDOM + VERTICES]
    n = (m * (f(1) / np.sqrt(((m[:, 0] * m[:, 0] + m[:, 1] * m[:, 1]) + m[:, 2] * m[:, 2]).astype(f)))[:, None]).astype(f)
    o = (pts["position"][:RANDOM + VERTICES] + (n * f(0.001)).astype(f)).astype(f)
    got_o = rays["origin"].reshape(len(pts), samples, 3)[:RANDOM + VERTICES]
    assert_bit_equal(np.ascontiguousarray(got_o), np.repeat(o[:, None], samples, axis=1), "the hook's origins")
    ref.OnDestroy()
    mgr.OnDestroy()


def test_directions_are_a_cosine_weighted_hemisphere():
    """The hook's directions about nine normals (axes, both signs of z at x = 0, the -0 case, nearly -z, a random one): all in the
    hemisphere and of unit length; at 4,096 samples the mean of cos(theta) is 2/3 and the fraction inside a cone of half-angle theta is
    sin^2(theta) (uniform would give 1/2 and 1 - cos(theta); a mirrored hemisphere fails the first check)."""
    normals = np.array([(0, 0, 1), (0, 0, -1), (1, 0, -0.0), (0, 1, 0), (0, -1, 0), (-1, 0, 0), (1e-4, 0, -1), (0.3, -0.5, 0.8),
                        (-2.0, 7.0, 0.5)], dtype=np.float32)
    pts = surface_points(np.zeros_like(normals), normals)
    o = capi.RtLib(ORACLE_LIB).create(0)
    rays = lightmap_rays(o, pts, SKY_SAMPLES, 5)
    o.destroy()
    d = rays["dir"].reshape(len(pts), SKY_SAMPLES, 3).astype(np.float64)
    n = unit64(normals)
    cos = np.einsum("pkc,pc->pk", d, n)
    assert (cos >= -1e-6).all(), cos.min()
    assert np.abs(np.linalg.norm(d, axis=-1) - 1.0).max() < 4e-7
    assert (np.abs(cos.mean(axis=1) - 2.0 / 3.0) < 1e-3).all(), cos.mean(axis=1)
    for deg in (30.0, 60.0):
        inside = (cos >= np.cos(np.radians(deg))).mean(axis=1)
        assert (np.abs(inside - np.sin(np.radians(deg)) ** 2) < 1e-2).all(), (deg, inside)


# ---- physics ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("samples", [1, 33, 1024])
def test_furnace_inside_a_closed_emitter(samples):
    """Texels inside a closed sphere of black emitters with emission 0.5: every sample is 0.5, so rgb is 0.5 exactly."""
    sc = scenes.Scene("furnace", 16, 12, cam_local_to_world=np.eye(4), settings=dict(useSky=False, maxBounceCount=4))
    mat = scenes.material(diffuse=(0, 0, 0), emission=(0.5, 0.5, 0.5), emissionStrength=1.0, specularProbability=0.0)
    sc.spheres = np.stack([scenes._sphere((1.0, 2.0, 3.0), 2.0, mat)])
    pts = surface_points([[1.0, 2.0, 3.0], [1.5, 1.2, 3.4], [1.0, 0.1, 3.0]], [[0, 1, 0], [0.3, -2.0, 0.1], [0, 1, 0]])
    mgr = T.open_mgr(CUDA_LIB, sc)
    got = mgr.context.bake_lightmap(pts, samples, 8)
    mgr.OnDestroy()
    assert (got["rejected"] == 0).all()
    assert (got["rgb"] == np.float32(0.5)).all(), got["rgb"]


SKY_NORMALS = np.array([(0, 1, 0), (0, -1, 0), (1, 0, 0), (0.3, -0.5, 0.8)], dtype=np.float32)


def sky_integral64(normal, grid=1024):
    """E / pi of the sun-less sky about `normal` in float64: the mean of the sky over a midpoint grid of the cosine-weighted map."""
    n = unit64(normal)
    t = np.array([1.0, 0.0, 0.0]) if abs(n[0]) < 0.9 else np.array([0.0, 1.0, 0.0])
    T_ = unit64(np.cross(t, n))
    B_ = np.cross(n, T_)
    u, v = np.meshgrid((np.arange(grid) + 0.5) / grid, (np.arange(grid) + 0.5) / grid, indexing="ij")
    u, v = u.reshape(-1), v.reshape(-1)
    r = np.sqrt(u)
    d = (r * np.cos(2 * np.pi * v))[:, None] * T_ + (r * np.sin(2 * np.pi * v))[:, None] * B_ + np.sqrt(1 - u)[:, None] * n
    return P.sky64(d, np.zeros(3), 500.0, 0.0).mean(axis=0)


@pytest.mark.parametrize("samples", [1, 33, SKY_SAMPLES])
def test_sky_alone_against_float64(samples):
    """No geometry, the sky on and the sun off, four normals: each texel is the float64 mean of the restated sky over its own sample
    directions (the hook's binary32 ones) within the sums' rounding plus 64 ulps of the sky per sample; at 4,096 samples it is within
    1 % of the float64 hemisphere integral."""
    sc = scenes.Scene("sky", 16, 12, cam_local_to_world=np.eye(4), settings=dict(useSky=True, maxBounceCount=4, sunIntensity=0.0),
                      sun_forward=(-0.3, -0.8, -0.52))
    pts = surface_points([[0.0, 0.0, 0.0], [3.0, -1.0, 2.0], [0.0, 5.0, 0.0], [-1.0, 0.0, 1.0]], SKY_NORMALS)
    ref = T.open_mgr(ORACLE_LIB, sc)
    rays = lightmap_rays(ref.context, pts, samples, 3)
    ref.OnDestroy()
    d = rays["dir"].astype(np.float64)
    L64 = P.sky64(d, np.zeros(3), 500.0, 0.0).reshape(-1, samples, 3)
    want = L64.mean(axis=1)
    mag = np.abs(L64).sum(axis=1) / samples
    depth = max(0, int(np.ceil(np.log2(-(-samples // capi.RT_PROBE_CHUNK)))))
    tol = mag * ((capi.RT_PROBE_CHUNK + depth + 2) * U + 64 * U)
    mgr = T.open_mgr(CUDA_LIB, sc)
    got = mgr.context.bake_lightmap(pts, samples, 3)
    mgr.OnDestroy()
    assert (got["rejected"] == 0).all()
    err = np.abs(got["rgb"].astype(np.float64) - want)
    assert (err <= tol).all(), (err.max(), (err / tol).max())
    if samples == SKY_SAMPLES:
        exact = np.stack([sky_integral64(nm) for nm in SKY_NORMALS])
        rel = np.abs(got["rgb"].astype(np.float64) - exact) / exact
        assert (rel < 0.01).all(), rel


def test_against_the_reference_diffuse_bounce():
    """Five floor and wall vertices of the knot room: the bake agrees within 5 combined standard errors with the mean of rtTracePaths
    samples that start at o along normalize(n + a random unit vector) (HL:524-525), each on its own random state.  The bake's standard
    error is taken from its own samples' spread (orLightmapRays -> rtTracePaths), an upper bound for its R2 directions."""
    sc = scenes.knot_room(24, 16, 4, 1, nu=40, nv=8)
    room = sc.meshes[1]
    vt = manager.vertex_texels(room.vertices, room.normals, np.eye(4))
    pts = vt[[0, 5, 9, 13, 17]]                                  # floor, ceiling-adjacent floor row, back, left and right walls
    rng = np.random.RandomState(23)
    mgr = T.open_mgr(CUDA_LIB, sc)
    got = mgr.context.bake_lightmap(pts, BOUNCE_SAMPLES, 31)
    ref = T.open_mgr(ORACLE_LIB, sc)
    own = mgr.context.trace_paths(lightmap_rays(ref.context, pts, BOUNCE_SAMPLES, 31), 1)["rgb"].reshape(len(pts), BOUNCE_SAMPLES, 3)
    ref.OnDestroy()
    se_bake = own.astype(np.float64).std(axis=1) / np.sqrt(BOUNCE_SAMPLES)
    f = np.float32
    for i, p in enumerate(pts):
        n = p["normal"].astype(f)
        o = (p["position"] + (n * f(0.001)).astype(f)).astype(f)
        r = unit64(rng.standard_normal((BOUNCE_REF, 3)))
        rays = np.zeros(BOUNCE_REF, dtype=capi.PATH_RAY_DTYPE)
        rays["origin"] = o
        rays["dir"] = unit64(n.astype(np.float64) + r).astype(f)
        rays["rngState"] = rng.randint(0, 2 ** 32, BOUNCE_REF, dtype=np.uint64).astype(np.uint32)
        L = mgr.context.trace_paths(rays, 1)["rgb"].astype(np.float64)
        se = np.sqrt(L.var(axis=0) / BOUNCE_REF + se_bake[i] ** 2)
        diff = np.abs(got["rgb"][i].astype(np.float64) - L.mean(axis=0))
        assert (diff <= 5 * se + 1e-6).all(), (i, got["rgb"][i], L.mean(axis=0), se)
        assert (L.mean(axis=0) > 0).all()
    mgr.OnDestroy()


# ---- call behaviour ---------------------------------------------------------------------------------------------------------------
def test_seed_and_texel_index_enter_only_as_seed_plus_p():
    """Texel p of a call at seed s is the one-texel call at seed s + p; the same call again is the same; another seed gives other paths."""
    sc = scenes.cornell_spheres(24, 16, 4, 1)
    pts = texel_set(sc, 10)
    mgr = T.open_mgr(CUDA_LIB, sc)
    ctx = mgr.context
    s = 40
    full = ctx.bake_lightmap(pts, s, 0xFFFFFFF0)
    for p in range(len(pts)):
        CM.assert_texels_equal(ctx.bake_lightmap(pts[p:p + 1], s, (0xFFFFFFF0 + p) & 0xFFFFFFFF), full[p:p + 1], f"texel {p} at seed + p")
    CM.assert_texels_equal(ctx.bake_lightmap(pts, s, 0xFFFFFFF0), full, "the same call again")
    assert not np.array_equal(ctx.bake_lightmap(pts, s, 1)["rgb"], full["rgb"])
    mgr.OnDestroy()


def test_bakes_between_frames_change_nothing_the_frames_show():
    sc = scenes.instanced_knots(32, 24, 4, 2, instances=150)
    pts = texel_set(sc, 11)
    images = []
    for with_bakes in (False, True):
        mgr = T.open_mgr(CUDA_LIB, sc, {"countStats": 1})
        ctx = mgr.context
        ctx.reset_stats()
        for _ in range(3):
            mgr.RenderFrame()
            if with_bakes:
                before, frame = ctx.stats(), mgr.raytraceFrameTex
                ctx.bake_lightmap(pts, 33, 5)
                after = ctx.stats()
                assert after["dispatches"] == before["dispatches"] and after["kernelMs"] == before["kernelMs"]
                assert after["rays"] > before["rays"]
                assert_bit_equal(mgr.raytraceFrameTex, frame, "FrameRender right after a bake")
        images.append((mgr.raytraceFrameTex, mgr.accumulatedResult, ctx.stats(), ctx.pixel_stats()))
        mgr.OnDestroy()
    assert_bit_equal(images[1][0], images[0][0], "FrameRender with bakes in between")
    assert_bit_equal(images[1][1], images[0][1], "AccumulatedRender with bakes in between")
    assert images[1][3].tobytes() == images[0][3].tobytes(), "PixelStats with bakes in between"
    assert images[1][2]["dispatches"] == images[0][2]["dispatches"] == 3


def test_camera_frame_seed_and_samples_per_pixel_do_not_change_a_bake():
    sc = scenes.knot_room(24, 16, 4, 1, nu=40, nv=8, glass=True)
    pts = texel_set(sc, 12)
    for lib in (ORACLE_LIB, CUDA_LIB):
        mgr = T.open_mgr(lib, sc, enable=False)          # no OnEnable: no rtResize, no dispatch
        ctx = mgr.context
        want = mgr.bake_lightmap(pts, 33, 3)
        ctx.set_int("Frame", 17)
        ctx.set_int("renderSeed", 999)
        ctx.set_int("NumRaysPerPixel", 7)
        ctx.set_matrix("CamLocalToWorldMatrix", np.eye(4, dtype=np.float32) * 2.0)
        CM.assert_texels_equal(ctx.bake_lightmap(pts, 33, 3), want, f"{lib}: after Frame / renderSeed / camera / NumRaysPerPixel changed")
        mgr.OnDestroy()


def test_empty_call_and_every_error_code():
    sc = scenes.knot_room(16, 12, 3, 1, nu=30, nv=6)
    for lib in (ORACLE_LIB, CUDA_LIB):
        mgr = T.open_mgr(lib, sc)
        ctx, L, h = mgr.context, mgr.context._L, mgr.context.handle
        pts = texel_set(sc, 0)[:4].copy()
        out = np.zeros(len(pts), dtype=capi.CUBE_TEXEL_DTYPE)
        st = ctx.stats()
        assert L.rtBakeLightmap(h, None, 0, 1, 0, None) == capi.RT_OK and ctx.stats()["rays"] == st["rays"]
        assert ctx.bake_lightmap(np.zeros((0, 6)), 4).shape == (0,)
        assert L.rtBakeLightmap(None, pts.ctypes.data, len(pts), 1, 0, out.ctypes.data) == capi.RT_E_INVALID
        assert L.rtBakeLightmap(h, pts.ctypes.data, -1, 1, 0, out.ctypes.data) == capi.RT_E_INVALID
        assert L.rtBakeLightmap(h, None, len(pts), 1, 0, out.ctypes.data) == capi.RT_E_INVALID
        assert L.rtBakeLightmap(h, pts.ctypes.data, len(pts), 1, 0, None) == capi.RT_E_INVALID
        for s in (0, -1, capi.RT_MAX_BATCH_SAMPLES + 1):
            assert L.rtBakeLightmap(h, pts.ctypes.data, len(pts), s, 0, out.ctypes.data) == capi.RT_E_INVALID, s
            assert L.rtBakeLightmap(h, pts.ctypes.data, 0, s, 0, out.ctypes.data) == capi.RT_E_INVALID, s
        for m in (-1, 201):
            ctx.set_int("MaxBounceCount", m)
            assert L.rtBakeLightmap(h, pts.ctypes.data, len(pts), 1, 0, out.ctypes.data) == capi.RT_E_STATE, m
            assert L.rtBakeLightmap(h, pts.ctypes.data, 0, 1, 0, out.ctypes.data) == capi.RT_OK
        ctx.set_int("MaxBounceCount", 200)
        assert L.rtBakeLightmap(h, pts.ctypes.data, len(pts), 1, 0, out.ctypes.data) == capi.RT_OK
        ctx.set_int("MaxBounceCount", 0)
        assert L.rtBakeLightmap(h, pts.ctypes.data, len(pts), 1, 0, out.ctypes.data) == capi.RT_OK
        ctx.set_int("modelCount", 99)
        assert L.rtBakeLightmap(h, pts.ctypes.data, len(pts), 1, 0, out.ctypes.data) == capi.RT_E_STATE
        ctx.set_int("modelCount", 2)
        models = np.zeros(2, dtype=capi.MODEL_DTYPE)
        models[1]["nodeOffset"] = 10 ** 7
        ctx.set_buffer("ModelInfo", models)
        assert L.rtBakeLightmap(h, pts.ctypes.data, len(pts), 1, 0, out.ctypes.data) == capi.RT_E_STATE
        ctx.set_buffer("Nodes", np.zeros(0, dtype=capi.NODE_DTYPE))
        assert L.rtBakeLightmap(h, pts.ctypes.data, len(pts), 1, 0, out.ctypes.data) == capi.RT_E_STATE
        assert L.rtBakeLightmapDevice(None, None, None, 0, 1, 0) == capi.RT_E_INVALID
        if lib == CUDA_LIB:                              # (the oracle has no device form: RT_E_STATE)
            assert L.rtBakeLightmapDevice(h, None, None, 0, 0, 0) == capi.RT_E_INVALID
            assert L.rtBakeLightmapDevice(h, None, None, -1, 1, 0) == capi.RT_E_INVALID
            assert L.rtBakeLightmapDevice(h, None, None, 1, 1, 0) == capi.RT_E_INVALID
            assert L.rtBakeLightmapDevice(h, None, None, 0, 1, 0) == capi.RT_OK
        mgr.OnDestroy()
    from test_round2_abi import chain_bvh, one_model_scene
    for lib in (ORACLE_LIB, CUDA_LIB):
        mgr = T.open_mgr(lib, one_model_scene(16, 12))
        tris, nodes = chain_bvh(64)
        mgr.context.set_buffer("Triangles", tris)
        mgr.context.set_buffer("Nodes", nodes)
        with pytest.raises(capi.RtError) as e:
            mgr.context.bake_lightmap(surface_points([[0, 0, 0]], [[0, 1, 0]]), 1)
        assert e.value.code == capi.RT_E_STATE and "too deep" in str(e.value), lib
        mgr.OnDestroy()


def test_cpp_manager_equals_the_python_context():
    sc = scenes.knot_room(24, 16, 4, 1, nu=40, nv=8, glass=True)
    pts = texel_set(sc, 13)
    for lib in (ORACLE_LIB, CUDA_LIB):
        mgr = T.open_mgr(lib, sc)
        CM.assert_texels_equal(mgr.bake_lightmap(pts, 33, 9), mgr.context.bake_lightmap(pts, 33, 9),
                               f"{lib}: RayComputeManager.BakeLightmap vs the context")
        mgr.OnDestroy()


def test_vertex_texels_are_the_transformed_vertices_and_shading_normals():
    """vertex_texels: (M [v, 1]).xyz and normalize(M3x3 n) (HL:367, not the inverse transpose), against float64."""
    sc = scenes.knot_room(24, 16, 4, 1, nu=40, nv=8)
    m = sc.models[0]
    mesh = sc.meshes[m.mesh]
    vt = manager.vertex_texels(mesh.vertices, mesh.normals, m.local_to_world)
    assert vt.dtype == capi.SURFACE_POINT_DTYPE and len(vt) == len(mesh.vertices)
    M = np.asarray(m.local_to_world, dtype=np.float32).astype(np.float64)
    pos = mesh.vertices.astype(np.float64) @ M[:3, :3].T + M[:3, 3]
    nrm = unit64(mesh.normals.astype(np.float64) @ M[:3, :3].T)
    assert np.abs(vt["position"] - pos).max() < 1e-5 * max(1.0, np.abs(pos).max())
    assert np.abs(vt["normal"] - nrm).max() < 1e-6


# ---- GPU only ---------------------------------------------------------------------------------------------------------------------
def test_texel_indices_across_internal_launches():
    """32,800 samples are 1,025 chunks, so a launch holds floor(7 * 2^20 / 1025) = 7,161 texels: 7,171 texels take two launches.  The
    host and device forms equal each other, and the oracle's texels on both sides of the boundary (and the first and last) equal the
    call."""
    torch = pytest.importorskip("torch")
    samples = 32 * 1025
    per = capi.RT_CUBE_SCRATCH_CHUNKS // (samples // capi.RT_PROBE_CHUNK)
    assert per == 7161
    sc = scenes.cornell_spheres(24, 16, 4, 1)
    rng = np.random.RandomState(14)
    base = texel_set(sc, 14)
    pts = base[rng.randint(0, RANDOM, per + 10)]
    pts["normal"] += rng.uniform(-0.3, 0.3, (len(pts), 3)).astype(np.float32)
    mgr = T.open_mgr(CUDA_LIB, sc)
    got = mgr.context.bake_lightmap(pts, samples, 77)
    d_pts = torch.from_numpy(pts.view(np.uint8).copy()).cuda()
    d_out = torch.zeros(len(pts) * 16, dtype=torch.uint8, device="cuda")
    mgr.context.bake_lightmap_device(d_pts.data_ptr(), d_out.data_ptr(), len(pts), samples, 77)
    mgr.context.synchronize()
    dev = d_out.cpu().numpy().view(capi.CUBE_TEXEL_DTYPE)
    mgr.OnDestroy()
    CM.assert_texels_equal(dev, got, "device form vs host form across launches")
    ref = T.open_mgr(ORACLE_LIB, sc)
    for t in (0, per - 1, per, len(pts) - 1):
        CM.assert_texels_equal(got[t: t + 1], oracle_texels(ref.context, pts, samples, 77, t, 1), f"texel {t}")
    ref.OnDestroy()


def test_more_texels_than_one_host_batch():
    """RT_TRACE_CHUNK_RAYS + 5 texels at 3 samples: the host form's two batches equal one device-form launch over all texels, and the
    oracle's texels at the batch boundary."""
    torch = pytest.importorskip("torch")
    n = capi.RT_TRACE_CHUNK_RAYS + 5
    sc = scenes.cornell_spheres(24, 16, 4, 1)
    rng = np.random.RandomState(15)
    base = texel_set(sc, 15)[:RANDOM]
    pts = base[rng.randint(0, RANDOM, n)]
    pts["normal"] = rng.standard_normal((n, 3)).astype(np.float32)
    mgr = T.open_mgr(CUDA_LIB, sc)
    got = mgr.context.bake_lightmap(pts, 3, 99)
    d_pts = torch.from_numpy(pts.view(np.uint8).copy()).cuda()
    d_out = torch.zeros(n * 16, dtype=torch.uint8, device="cuda")
    mgr.context.bake_lightmap_device(d_pts.data_ptr(), d_out.data_ptr(), n, 3, 99)
    mgr.context.synchronize()
    CM.assert_texels_equal(d_out.cpu().numpy().view(capi.CUBE_TEXEL_DTYPE), got, "host batches vs one device call")
    mgr.OnDestroy()
    ref = T.open_mgr(ORACLE_LIB, sc)
    b = capi.RT_TRACE_CHUNK_RAYS
    CM.assert_texels_equal(got[b - 2: b + 2], oracle_texels(ref.context, pts, 3, 99, b - 2, 4), "the batch boundary")
    ref.OnDestroy()


def test_device_form_on_the_context_stream_and_a_caller_stream():
    torch = pytest.importorskip("torch")
    sc = scenes.instanced_knots(24, 16, 4, 1, instances=150)
    pts = texel_set(sc, 16)
    n = len(pts)
    mgr = T.open_mgr(CUDA_LIB, sc)
    ctx = mgr.context
    want = ctx.bake_lightmap(pts, 100, 4)
    raw = torch.zeros(n * 24 + 4, dtype=torch.uint8)
    raw[4:] = torch.from_numpy(pts.view(np.uint8).reshape(-1).copy())
    d_raw = raw.cuda()
    for stream in (None, torch.cuda.Stream()):
        d_out = torch.full((n * 16 + 16,), 0x5a, dtype=torch.uint8, device="cuda")
        if stream is not None:
            ctx.set_stream(stream.cuda_stream)
        ctx.bake_lightmap_device(d_raw.data_ptr() + 4, d_out.data_ptr(), n, 100, 4)       # 4-byte aligned points
        ctx.synchronize()
        got = d_out.cpu().numpy()
        assert (got[n * 16:] == 0x5a).all()
        CM.assert_texels_equal(got[: n * 16].view(capi.CUBE_TEXEL_DTYPE), want, f"device form, stream {stream}")
    ctx.set_stream(0)
    for pp, op in ((d_raw.data_ptr() + 2, d_out.data_ptr()), (d_raw.data_ptr() + 4, d_out.data_ptr() + 4)):
        with pytest.raises(capi.RtError) as e:
            ctx.bake_lightmap_device(pp, op, n, 1)
        assert e.value.code == capi.RT_E_INVALID
    mgr.OnDestroy()
    o = capi.RtLib(ORACLE_LIB).create(0)
    assert o._L.rtBakeLightmapDevice(o.handle, None, None, 0, 1, 0) == capi.RT_E_STATE


def test_vertex_texels_of_the_871k_triangle_cluster():
    """A slice of the cluster's vertex texels at 64 samples and MaxBounceCount 12 against the oracle's texels for a seeded subset."""
    sc = scenes.knot_cluster(64, 36, 12, 1)
    m = sc.models[0]
    mesh = sc.meshes[m.mesh]
    pts = manager.vertex_texels(mesh.vertices, mesh.normals, m.local_to_world)[::97][:4096]
    mgr = T.open_mgr(CUDA_LIB, sc)
    got = mgr.context.bake_lightmap(pts, 64, 1234)
    mgr.OnDestroy()
    ref = T.open_mgr(ORACLE_LIB, sc)
    for t in np.random.RandomState(17).choice(len(got), 16, replace=False):
        CM.assert_texels_equal(got[t: t + 1], oracle_texels(ref.context, pts, 64, 1234, int(t), 1), f"texel {t}")
    ref.OnDestroy()
    assert (got["rgb"][:, 0] > 0).mean() > 0.5
