"""rtBakeProbes on the H100 (`-m gpu`): the L2 spherical harmonics of path-traced radiance at probe positions equal the oracle's
restatement bit for bit, `rejected` and the counters included, on seven scenes with model skipping on and off, MaxBounceCount 0 and 4,
and sample counts around the chunk and tree edges; a probe rebuilt sample by sample (orProbeRays -> rtTracePaths(samples = 1) -> a
numpy restatement of the basis, the chunk sums, the padded tree and the scale) equals the call; probe indices across internal
launches; 4,096 probes on the 871k-triangle cluster; isolation, seeds, n = 0 and every refusal, the device form, both managers; and
two analytic checks against float64 (a sky alone, the inside of an emissive sphere).  The same bodies run in the CPU suite against the
SIMT interpreter build (tests/test_simt_probes.py)."""
import ctypes as C

import numpy as np
import pytest

from conftest import CUDA_LIB, ORACLE_LIB, assert_bit_equal
from ray_tracing_b200 import capi, scenes
import test_gpu_trace_paths as G
import test_gpu_trace_rays as T

pytestmark = pytest.mark.gpu

PROBES = 6                                              # in-scene probes per set (plus a far and a NaN position)
SAMPLES = (1, 31, 32, 33, 1024, 1025, 32 * 33)          # around a chunk (32), a warp's 32 chunks and the padded tree
BOUNCES = (0, 4)
U = 2.0 ** -24                                          # binary32 unit roundoff


# ---- helpers ----------------------------------------------------------------------------------------------------------------------
def probe_positions(sc, seed=0, n=None, special=True):
    """n points between the camera and the scene's surfaces (rtTraceRays' "inside" origins), then a far and a NaN position."""
    pts = T.ray_sets(sc, seed=seed, n=n or PROBES)["inside"]["origin"][: n or PROBES].astype(np.float32)
    if special:
        pts = np.concatenate([pts, np.array([[1e5, 1e5, -1e5], [np.nan, 0.0, 0.0]], dtype=np.float32)])
    return np.ascontiguousarray(pts)


def probe_rays(octx, positions, samples, seed):
    """orProbeRays: every sample's start (position, d_k, H(H(seed + p) + k)) as n * samples PATH_RAY_DTYPE records."""
    L = octx._L
    L.orProbeRays.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_uint32, C.c_void_p]
    pos = np.ascontiguousarray(positions, dtype=np.float32).reshape(-1, 3)
    out = np.zeros(len(pos) * samples, dtype=capi.PATH_RAY_DTYPE)
    assert L.orProbeRays(octx.handle, pos.ctypes.data, len(pos), samples, seed, out.ctypes.data) == capi.RT_OK
    return out


def basis32(d):
    """The header's nine basis functions in binary32, one operation at a time: (..., 9)."""
    f = np.float32
    x, y, z = d[..., 0].astype(f), d[..., 1].astype(f), d[..., 2].astype(f)
    return np.stack([np.full_like(x, f(0.282094792)), f(0.488602512) * y, f(0.488602512) * z, f(0.488602512) * x,
                     f(1.09254843) * (x * y), f(1.09254843) * (y * z), f(0.315391565) * ((f(3) * (z * z)) - f(1)),
                     f(1.09254843) * (x * z), f(0.546274215) * ((x * x) - (y * y))], axis=-1)


def project32(rays, radiance, n, samples):
    """The header's projection restated in numpy binary32 from the samples' directions and radiances: (sh (n, 3, 9), rejected (n,))."""
    f = np.float32
    chunk = capi.RT_PROBE_CHUNK
    chunks = -(-samples // chunk)
    d = rays["dir"].reshape(n, samples, 3)
    L = radiance.reshape(n, samples, 3).astype(f)
    ok = np.isfinite(L).all(axis=-1)
    terms = np.where(ok[..., None, None], L[..., :, None] * basis32(d)[..., None, :], f(0))     # (n, S, 3, 9)
    pad = np.zeros((n, chunks * chunk, 3, 9), dtype=f)                                           # +0 adds nothing to a sum from +0
    pad[:, :samples] = terms
    pad = pad.reshape(n, chunks, chunk, 3, 9)
    sums = np.zeros((n, chunks, 3, 9), dtype=f)
    for j in range(chunk):                                                                       # k order within a chunk
        sums = (sums + pad[:, :, j]).astype(f)
    width = 1
    while width < chunks:
        width *= 2
    tree = np.zeros((n, width, 3, 9), dtype=f)
    tree[:, :chunks] = sums
    while tree.shape[1] > 1:                                                                     # adjacent pairs, level by level
        tree = (tree[:, 0::2] + tree[:, 1::2]).astype(f)
    scale = f(12.566371) / f(samples)
    return (tree[:, 0] * scale).astype(f), (~ok).sum(axis=1).astype(np.uint32)


def assert_probes_equal(a, b, what):
    assert_bit_equal(np.ascontiguousarray(a[0]), np.ascontiguousarray(b[0]), f"{what}: sh")
    bad = np.flatnonzero(a[1] != b[1])
    assert len(bad) == 0, f"{what}: rejected differs for {len(bad)} probes, first {bad[0]}: {a[1][bad[0]]} vs {b[1][bad[0]]}"


def bake(ctx, positions, samples, seed, stats=False):
    ctx.reset_stats()
    out = ctx.bake_probes(positions, samples, seed)
    return (out, ctx.stats()) if stats else out


def COUNTS(sc):
    """The counters a counting run shares with the oracle: with the sphere accelerator (more than 64 spheres) the sphere counters are
    the accelerator's own, as in rtTraceRays."""
    return tuple(k for k in T.COUNTS if k != "sphereTests" or len(sc.spheres) <= 64)


def check_oracle(sc, positions, options_list=({},), samples=None, bounces=None, seed=7, sky=None):
    """rtBakeProbes against the oracle for every (samples, MaxBounceCount), each option set with modelSkip 1 and 0 and a counting
    run: SH bits, rejected, RtStats.rays and, counting, the box / triangle / sphere counters (COUNTS)."""
    cases = [(s, m) for s in (samples or SAMPLES) for m in (bounces or BOUNCES)]
    ref_mgr = T.open_mgr(ORACLE_LIB, sc)
    if sky is not None:
        ref_mgr.context.set_int("UseSky", sky)
    ref = {}
    for s, m in cases:
        ref_mgr.context.set_int("MaxBounceCount", m)
        ref[(s, m)] = bake(ref_mgr.context, positions, s, seed, stats=True)
    ref_mgr.OnDestroy()
    for opts in list(options_list) + [{"countStats": 1}]:
        for skip in ((opts["modelSkip"],) if "modelSkip" in opts else (1, 0)):
            mgr = T.open_mgr(CUDA_LIB, sc, dict(opts, modelSkip=skip))
            if sky is not None:
                mgr.context.set_int("UseSky", sky)
            for (s, m), (want, wst) in ref.items():
                mgr.context.set_int("MaxBounceCount", m)
                got, gst = bake(mgr.context, positions, s, seed, stats=True)
                what = f"{sc.name} {opts} modelSkip={skip} samples={s} MaxBounceCount={m}"
                assert got[0].shape == (len(positions), 3, 9) and got[0].dtype == np.float32 and got[1].dtype == np.uint32
                assert_probes_equal(got, want, what)
                keys = (COUNTS(sc) if opts.get("countStats") else ("rays",))
                assert all(gst[k] == wst[k] for k in keys), (what, gst, wst)
                assert gst["dispatches"] == 0 and gst["kernelMs"] == 0
            mgr.OnDestroy()
    return ref


# ---- against the oracle -----------------------------------------------------------------------------------------------------------
def test_oracle_cornell_spheres():
    sc = scenes.cornell_spheres(24, 16, 4, 1)
    ref = check_oracle(sc, probe_positions(sc, seed=1))
    lit = ref[(SAMPLES[-1], 4)][0][0][:PROBES, :, 0]
    assert (lit > 0).all()                               # every in-scene probe sees the light


def test_oracle_knot_room_with_glass():
    sc = scenes.knot_room(24, 16, 4, 1, nu=40, nv=8, glass=True)
    check_oracle(sc, probe_positions(sc, seed=2), sky=1)


def test_oracle_soup_with_sky_and_spheres():
    sc = G._soup_with_sky_and_defocus()
    check_oracle(sc, probe_positions(sc, seed=3))


@pytest.mark.parametrize("tlas", [-1, 0, 1])
def test_oracle_above_128_models_with_the_tlas(tlas):
    sc = scenes.instanced_knots(24, 16, 4, 1, instances=150)
    check_oracle(sc, probe_positions(sc, seed=4), ({"tlas": tlas},))


def test_oracle_ten_thousand_spheres_with_the_accelerator():
    sc = scenes.random_soup(24, 16, 4, 1, triangles=300, spheres=10000)
    check_oracle(sc, probe_positions(sc, seed=5), ({}, {"extInstantiation": 1}), sky=1)


def test_oracle_unity_fixture():
    from test_round2_abi import load_fixture
    sc = load_fixture(24, 16)
    check_oracle(sc, probe_positions(sc, seed=6))


def test_oracle_nan_sun_rejects_samples():
    """The NaN scene of test_gpu_adaptive.py::test_nan_pixels_against_the_oracle: every path that reaches the sky is NaN; those
    samples are counted in `rejected` and the probe stays finite."""
    sc = scenes.random_soup(24, 16, max_bounces=3, rays_per_pixel=1, triangles=600, spheres=8)
    sc.settings["sunIntensity"] = float("nan")
    ref = check_oracle(sc, probe_positions(sc, seed=8), sky=1)
    sh, rejected = ref[(SAMPLES[-1], 4)][0]
    assert (rejected[:PROBES] > 0).all() and np.isfinite(sh[:PROBES]).all()


# ---- the rebuild through rtTracePaths ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("samples", [33, 1025])
def test_rebuild_through_trace_paths(samples):
    """orProbeRays -> this build's rtTracePaths(samples = 1) -> numpy: the basis, the chunk sums in k order, the padded tree and the
    scale give rtBakeProbes' bits; the NaN-sun sky makes some samples non-finite, which both leave out."""
    sc = scenes.knot_room(24, 16, 4, 1, nu=40, nv=8, glass=True)
    sc.settings = dict(sc.settings, useSky=True)
    pos = probe_positions(sc, seed=9, n=4)
    ref = T.open_mgr(ORACLE_LIB, sc)
    mgr = T.open_mgr(CUDA_LIB, sc)
    for sun in (10.0, float("nan")):
        mgr.context.set_float("SunIntensity", sun)
        rays = probe_rays(ref.context, pos, samples, 21)
        want = project32(rays, mgr.context.trace_paths(rays, 1)["rgb"], len(pos), samples)
        assert_probes_equal(mgr.context.bake_probes(pos, samples, 21), want, f"SunIntensity={sun}")
        assert (want[1] > 0).any() == (sun != sun)
    ref.OnDestroy()
    mgr.OnDestroy()


# ---- seeds and probe indices ------------------------------------------------------------------------------------------------------
def test_seed_and_probe_index_enter_only_as_seed_plus_p():
    """Probe p of a call is the one-probe call at seed + p (the state is H(H(seed + p) + k)); another seed gives other paths."""
    sc = scenes.cornell_spheres(24, 16, 4, 1)
    pos = probe_positions(sc, seed=10, n=5, special=False)
    mgr = T.open_mgr(CUDA_LIB, sc)
    ctx = mgr.context
    full = ctx.bake_probes(pos, 40, 0xFFFFFFFE)
    for p in range(len(pos)):
        one = ctx.bake_probes(pos[p: p + 1], 40, (0xFFFFFFFE + p) & 0xFFFFFFFF)      # seed + p wraps modulo 2^32
        assert_probes_equal((one[0][0], one[1][0]), (full[0][p], full[1][p]), f"probe {p}")
    assert_probes_equal(ctx.bake_probes(pos, 40, 0xFFFFFFFE), full, "the same call again")
    other = ctx.bake_probes(pos, 40, 1)
    assert not np.array_equal(other[0], full[0])
    mgr.OnDestroy()


# ---- isolation --------------------------------------------------------------------------------------------------------------------
def test_bakes_between_frames_change_nothing_the_frames_show():
    sc = scenes.instanced_knots(32, 24, 4, 2, instances=150)
    pos = probe_positions(sc, seed=11, n=4)
    images = []
    for with_bakes in (False, True):
        mgr = T.open_mgr(CUDA_LIB, sc, {"countStats": 1})
        ctx = mgr.context
        ctx.reset_stats()
        for _ in range(3):
            mgr.RenderFrame()
            if with_bakes:
                before, frame = ctx.stats(), mgr.raytraceFrameTex
                ctx.bake_probes(pos, 33, 5)
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
    pos = probe_positions(sc, seed=12, n=4)
    for lib in (ORACLE_LIB, CUDA_LIB):
        mgr = T.open_mgr(lib, sc, enable=False)          # no OnEnable: no rtResize, no dispatch
        ctx = mgr.context
        want = mgr.bake_probes(pos, 33, 3)
        ctx.set_int("Frame", 17)
        ctx.set_int("renderSeed", 999)
        ctx.set_int("NumRaysPerPixel", 7)
        ctx.set_matrix("CamLocalToWorldMatrix", np.eye(4, dtype=np.float32) * 2.0)
        assert_probes_equal(ctx.bake_probes(pos, 33, 3), want, f"{lib}: after Frame / renderSeed / camera / NumRaysPerPixel changed")
        mgr.OnDestroy()


# ---- refusals ---------------------------------------------------------------------------------------------------------------------
def test_empty_call_and_every_error_code():
    sc = scenes.knot_room(16, 12, 3, 1, nu=30, nv=6)
    for lib in (ORACLE_LIB, CUDA_LIB):
        mgr = T.open_mgr(lib, sc)
        ctx, L, h = mgr.context, mgr.context._L, mgr.context.handle
        pos = probe_positions(sc, n=3, special=False)
        out = np.zeros(len(pos), dtype=capi.PROBE_SH_DTYPE)
        st = ctx.stats()
        assert L.rtBakeProbes(h, None, 0, 1, 0, None) == capi.RT_OK and ctx.stats()["rays"] == st["rays"]
        sh, rej = ctx.bake_probes(np.zeros((0, 3)), 1)
        assert sh.shape == (0, 3, 9) and rej.shape == (0,)
        assert L.rtBakeProbes(None, pos.ctypes.data, len(pos), 1, 0, out.ctypes.data) == capi.RT_E_INVALID
        assert L.rtBakeProbes(h, pos.ctypes.data, -1, 1, 0, out.ctypes.data) == capi.RT_E_INVALID
        assert L.rtBakeProbes(h, None, len(pos), 1, 0, out.ctypes.data) == capi.RT_E_INVALID
        assert L.rtBakeProbes(h, pos.ctypes.data, len(pos), 1, 0, None) == capi.RT_E_INVALID
        for s in (0, -1, capi.RT_MAX_BATCH_SAMPLES + 1):
            assert L.rtBakeProbes(h, pos.ctypes.data, len(pos), s, 0, out.ctypes.data) == capi.RT_E_INVALID, s
        for m in (-1, 201):
            ctx.set_int("MaxBounceCount", m)
            assert L.rtBakeProbes(h, pos.ctypes.data, len(pos), 1, 0, out.ctypes.data) == capi.RT_E_STATE, m
            assert L.rtBakeProbes(h, pos.ctypes.data, 0, 1, 0, out.ctypes.data) == capi.RT_OK
        ctx.set_int("MaxBounceCount", 200)
        assert L.rtBakeProbes(h, pos.ctypes.data, len(pos), 1, 0, out.ctypes.data) == capi.RT_OK
        ctx.set_int("MaxBounceCount", 0)
        assert L.rtBakeProbes(h, pos.ctypes.data, len(pos), 1, 0, out.ctypes.data) == capi.RT_OK
        ctx.set_int("modelCount", 99)
        assert L.rtBakeProbes(h, pos.ctypes.data, len(pos), 1, 0, out.ctypes.data) == capi.RT_E_STATE
        ctx.set_int("modelCount", 2)
        models = np.zeros(2, dtype=capi.MODEL_DTYPE)
        models[1]["nodeOffset"] = 10 ** 7
        ctx.set_buffer("ModelInfo", models)
        assert L.rtBakeProbes(h, pos.ctypes.data, len(pos), 1, 0, out.ctypes.data) == capi.RT_E_STATE
        ctx.set_buffer("Nodes", np.zeros(0, dtype=capi.NODE_DTYPE))
        assert L.rtBakeProbes(h, pos.ctypes.data, len(pos), 1, 0, out.ctypes.data) == capi.RT_E_STATE
        assert L.rtBakeProbesDevice(None, None, None, 0, 1, 0) == capi.RT_E_INVALID
        if lib == CUDA_LIB:                              # (the oracle has no device form: RT_E_STATE)
            assert L.rtBakeProbesDevice(h, None, None, 0, 0, 0) == capi.RT_E_INVALID
            assert L.rtBakeProbesDevice(h, None, None, -1, 1, 0) == capi.RT_E_INVALID
            assert L.rtBakeProbesDevice(h, None, None, 0, 1, 0) == capi.RT_OK
        mgr.OnDestroy()
    from test_round2_abi import chain_bvh, one_model_scene
    for lib in (ORACLE_LIB, CUDA_LIB):
        mgr = T.open_mgr(lib, one_model_scene(16, 12))
        tris, nodes = chain_bvh(64)
        mgr.context.set_buffer("Triangles", tris)
        mgr.context.set_buffer("Nodes", nodes)
        with pytest.raises(capi.RtError) as e:
            mgr.context.bake_probes(np.zeros((1, 3)), 1)
        assert e.value.code == capi.RT_E_STATE and "too deep" in str(e.value), lib
        mgr.OnDestroy()


def test_cpp_manager_equals_the_python_context():
    sc = scenes.knot_room(24, 16, 4, 1, nu=40, nv=8, glass=True)
    pos = probe_positions(sc, seed=13, n=4)
    for lib in (ORACLE_LIB, CUDA_LIB):
        mgr = T.open_mgr(lib, sc)
        assert_probes_equal(mgr.bake_probes(pos, 33, 9), mgr.context.bake_probes(pos, 33, 9), f"{lib}: RayComputeManager.BakeProbes vs the context")
        mgr.OnDestroy()


# ---- analytic checks (float64) ----------------------------------------------------------------------------------------------------
def rule64(d, values, samples):
    """sum_k values_k * Y_i(d_k) * 4 pi / S in float64 with the header's constants, and the same sum of |terms|: (.., 3, 9) each."""
    x, y, z = d[:, 0], d[:, 1], d[:, 2]
    Y = np.stack([np.full_like(x, np.float32(0.282094792)), np.float32(0.488602512) * y, np.float32(0.488602512) * z,
                  np.float32(0.488602512) * x, np.float32(1.09254843) * x * y, np.float32(1.09254843) * y * z,
                  np.float32(0.315391565) * (3 * z * z - 1), np.float32(1.09254843) * x * z, np.float32(0.546274215) * (x * x - y * y)], axis=-1)
    terms = values[:, :, None] * Y[:, None, :]
    scale = float(np.float32(12.566371)) / samples
    return terms.sum(axis=0) * scale, np.abs(terms).sum(axis=0) * scale, np.abs(Y).sum(axis=0) * scale


def sum_bound(samples):
    """Relative rounding of one coefficient in units of |terms|: Y (<= 4 operations), the product, 32 sequential additions in a chunk,
    the tree's depth and the scale (2)."""
    depth = max(0, int(np.ceil(np.log2(-(-samples // capi.RT_PROBE_CHUNK)))))
    return (4 + 1 + capi.RT_PROBE_CHUNK + depth + 2 + 2) * U


def sky64(d, sun_dir, sun_focus, sun_intensity):
    """GetEnvironmentLight (HL:167-183) in float64: ground / horizon / zenith gradient and the sun."""
    def smoothstep(a, b, v):
        t = np.clip((v - a) / (b - a), 0.0, 1.0)
        return t * t * (3.0 - 2.0 * t)
    ground, horizon, zenith = np.array([0.35, 0.3, 0.35]), np.array([1.0, 1.0, 1.0]), np.array([0.08, 0.37, 0.73])
    ground, horizon, zenith = (np.float32(v).astype(np.float64) for v in (ground, horizon, zenith))
    grad_t = smoothstep(0.0, 0.4, d[:, 1]) ** 0.35
    g2s = smoothstep(-0.01, 0.0, d[:, 1])
    grad = horizon + (zenith - horizon) * grad_t[:, None]
    sun = np.maximum(0.0, d @ sun_dir) ** (1000.0 / sun_focus) * sun_intensity
    return ground + (grad - ground) * g2s[:, None] + (sun[:, None] * np.ones(3)) * (g2s >= 1.0)[:, None]


@pytest.mark.parametrize("samples", [1, 33, 1025, 4096])
def test_sky_alone_against_float64(samples):
    """No geometry, the sky on: every sample is the sky in its direction.  The SH equal the float64 sum of the restated sky over the
    rule's directions (the hook's binary32 ones), within the sums' rounding plus 64 ulps of the sky per sample (about twenty binary32
    operations and two pow, whose error grows with log of its result times the exponent)."""
    sc = scenes.Scene("sky", 16, 12, cam_local_to_world=np.eye(4), settings=dict(useSky=True, maxBounceCount=4),
                      sun_forward=(-0.3, -0.8, -0.52))
    pos = np.array([[0.0, 0.0, 0.0], [3.0, -1.0, 2.0]], dtype=np.float32)
    ref = T.open_mgr(ORACLE_LIB, sc)
    rays = probe_rays(ref.context, pos, samples, 3)
    ref.OnDestroy()
    d = rays["dir"][:samples].astype(np.float64)
    exact = np.stack([np.cos(2 * np.pi * ((np.arange(samples, dtype=np.uint64) * 2654435769) % 2 ** 32) / 2 ** 32),
                      np.sin(2 * np.pi * ((np.arange(samples, dtype=np.uint64) * 2654435769) % 2 ** 32) / 2 ** 32)], axis=1)
    z = 1.0 - (2.0 * np.arange(samples) + 1.0) / samples
    rule = np.concatenate([exact * np.sqrt(1 - z * z)[:, None], z[:, None]], axis=1)
    assert np.abs(d - rule).max() < 64 * U, "the hook's directions are the spherical Fibonacci rule"
    sun_dir = np.float32([0.3, 0.8, 0.52]).astype(np.float64)
    L64 = sky64(d, sun_dir, 500.0, 10.0)
    want, mag, ymag = rule64(d, L64, samples)
    errL = rule64(d, np.abs(L64) * 64 * U, samples)[1]
    mgr = T.open_mgr(CUDA_LIB, sc)
    sh, rejected = mgr.context.bake_probes(pos, samples, 3)
    mgr.OnDestroy()
    assert (rejected == 0).all()
    for p in range(len(pos)):
        err = np.abs(sh[p].astype(np.float64) - want)
        tol = mag * sum_bound(samples) + errL
        assert (err <= tol).all(), (p, err.max(), (err / tol).max())


@pytest.mark.parametrize("samples", [1, 32, 1000])
def test_inside_a_closed_emissive_sphere(samples):
    """A probe inside one emissive sphere with black albedo: every sample is the emission E, so c0 = E * 4 pi * Y0 and the higher
    coefficients are the rule's float64 values, within the sums' rounding."""
    sc = scenes.Scene("emissive sphere", 16, 12, cam_local_to_world=np.eye(4), settings=dict(useSky=False, maxBounceCount=4))
    mat = scenes.material(diffuse=(0, 0, 0), emission=(0.9, 0.5, 0.25), emissionStrength=3.0, specularProbability=0.0)
    sc.spheres = np.stack([scenes._sphere((1.0, 2.0, 3.0), 2.0, mat)])
    pos = np.array([[1.0, 2.0, 3.0], [1.5, 1.2, 3.4]], dtype=np.float32)
    E = (np.float32([0.9, 0.5, 0.25]) * np.float32(3.0)).astype(np.float64)
    ref = T.open_mgr(ORACLE_LIB, sc)
    rays = probe_rays(ref.context, pos, samples, 8)
    ref.OnDestroy()
    d = rays["dir"][:samples].astype(np.float64)
    want, mag, _ = rule64(d, np.tile(E, (samples, 1)), samples)
    assert np.allclose(want[:, 0], E * float(np.float32(12.566371)) * float(np.float32(0.282094792)), rtol=1e-12, atol=0)
    mgr = T.open_mgr(CUDA_LIB, sc)
    sh, rejected = mgr.context.bake_probes(pos, samples, 8)
    mgr.OnDestroy()
    assert (rejected == 0).all()
    for p in range(len(pos)):
        err = np.abs(sh[p].astype(np.float64) - want)
        assert (err <= mag * sum_bound(samples)).all(), (p, err.max())


# ---- GPU only ---------------------------------------------------------------------------------------------------------------------
def test_probe_indices_across_internal_launches():
    """32,800 samples are 1,025 chunks, so a launch holds floor(2^20 / 1025) = 1023 probes: 1,025 probes take two launches.  The
    host and device forms equal each other, and oracle rows on both sides of the boundary (and the first) equal the call."""
    torch = pytest.importorskip("torch")
    samples, n = 32 * 1025, 1025
    per = capi.RT_PROBE_SCRATCH_CHUNKS // (samples // capi.RT_PROBE_CHUNK)
    assert per == 1023
    sc = scenes.cornell_spheres(24, 16, 4, 1)
    base = probe_positions(sc, seed=14, n=32, special=False)
    pos = np.ascontiguousarray(base[np.arange(n) % len(base)])
    mgr = T.open_mgr(CUDA_LIB, sc)
    got = mgr.context.bake_probes(pos, samples, 77)
    d_pos = torch.from_numpy(pos).cuda()
    d_out = torch.zeros(n * 112, dtype=torch.uint8, device="cuda")
    mgr.context.bake_probes_device(d_pos.data_ptr(), d_out.data_ptr(), n, samples, 77)
    mgr.context.synchronize()
    dev = d_out.cpu().numpy().view(capi.PROBE_SH_DTYPE)
    mgr.OnDestroy()
    assert_probes_equal((dev["sh"], dev["rejected"]), got, "device form vs host form across launches")
    ref = T.open_mgr(ORACLE_LIB, sc)
    for p in (0, per - 1, per, n - 1):
        want = ref.context.bake_probes(pos[p: p + 1], samples, 77 + p)
        assert_probes_equal((got[0][p: p + 1], got[1][p: p + 1]), want, f"probe {p}")
    ref.OnDestroy()


def test_device_form_on_the_context_stream_and_a_caller_stream():
    torch = pytest.importorskip("torch")
    sc = scenes.instanced_knots(24, 16, 4, 1, instances=150)
    pos = probe_positions(sc, seed=15, n=40)
    n = len(pos)
    mgr = T.open_mgr(CUDA_LIB, sc)
    ctx = mgr.context
    want = ctx.bake_probes(pos, 100, 4)
    raw = torch.zeros(n * 12 + 4, dtype=torch.uint8)
    raw[4:] = torch.from_numpy(pos.view(np.uint8).reshape(-1).copy())
    d_raw = raw.cuda()
    for stream in (None, torch.cuda.Stream()):
        d_out = torch.full((n * 112 + 16,), 0x5a, dtype=torch.uint8, device="cuda")
        if stream is not None:
            ctx.set_stream(stream.cuda_stream)
        ctx.bake_probes_device(d_raw.data_ptr() + 4, d_out.data_ptr(), n, 100, 4)       # 4-byte aligned positions
        ctx.synchronize()
        got = d_out.cpu().numpy()
        assert (got[n * 112:] == 0x5a).all()
        rec = got[: n * 112].view(capi.PROBE_SH_DTYPE)
        assert_probes_equal((rec["sh"], rec["rejected"]), want, f"device form, stream {stream}")
    ctx.set_stream(0)
    for pp, op in ((d_raw.data_ptr() + 2, d_out.data_ptr()), (d_raw.data_ptr() + 4, d_out.data_ptr() + 4)):
        with pytest.raises(capi.RtError) as e:
            ctx.bake_probes_device(pp, op, n, 1)
        assert e.value.code == capi.RT_E_INVALID
    mgr.OnDestroy()
    o = capi.RtLib(ORACLE_LIB).create(0)
    assert o._L.rtBakeProbesDevice(o.handle, None, None, 0, 1, 0) == capi.RT_E_STATE


def test_four_thousand_probes_on_the_871k_triangle_cluster():
    """4,096 probes at 256 samples and MaxBounceCount 12 against oracle rows for a seeded subset of 24."""
    sc = scenes.knot_cluster(64, 36, 12, 1)
    pos = probe_positions(sc, seed=16, n=4096, special=False)
    mgr = T.open_mgr(CUDA_LIB, sc)
    got = mgr.context.bake_probes(pos, 256, 1234)
    mgr.OnDestroy()
    ref = T.open_mgr(ORACLE_LIB, sc)
    for p in np.random.RandomState(17).choice(len(pos), 24, replace=False):
        want = ref.context.bake_probes(pos[p: p + 1], 256, 1234 + int(p))
        assert_probes_equal((got[0][p: p + 1], got[1][p: p + 1]), want, f"probe {p}")
    ref.OnDestroy()
    assert (got[0][:, :, 0] > 0).mean() > 0.5
