"""rtBakeCubemaps on the H100 (`-m gpu`): HDR cube maps of path-traced radiance at probe positions equal the oracle's restatement bit
for bit, `rejected` and the counters included, on seven scenes with model skipping on and off, MaxBounceCount 0 and 4, and face sizes and
sample counts around the chunk and tree edges; a texel rebuilt sample by sample (orCubemapRays -> rtTracePaths(samples = 1) -> a numpy
restatement of the chunk sums, the padded tree and the division) equals the call, and a numpy restatement of the directions equals the
hook's; the face order and orientation in a room of six coloured walls; anti-aliasing along a straight emissive edge against its float64
coverage; seeds and texel indices; texel indices across internal launches; four probes on the 871k-triangle cluster; isolation, n = 0 and
every refusal, the device form, both managers; a sky alone against float64; write_cubemap_exr.  The same bodies run in the CPU suite
against the SIMT interpreter build (tests/test_simt_cubemaps.py)."""
import ctypes as C

import numpy as np
import pytest

from conftest import CUDA_LIB, ORACLE_LIB, assert_bit_equal
from ray_tracing_b200 import capi, display, scenes
import test_gpu_probes as P
import test_gpu_trace_paths as G
import test_gpu_trace_rays as T

pytestmark = pytest.mark.gpu

PROBES = 3                                              # in-scene probes per set (plus a far and a NaN position)
# (faceSize, samples): every face size with the samples around a chunk (32) and a padded tree of 33 chunks, while N^2 * S stays small
CASES = tuple((N, S) for N in (1, 2, 7, 16) for S in (1, 31, 32, 33, 1025) if N * N * S <= 9000)
BOUNCES = (0, 4)
AA_FACE = 8                                             # the face size of the anti-aliasing test (at 1,024 samples)
U = 2.0 ** -24                                          # binary32 unit roundoff
R2 = (3242174889, 2447445414)                           # 2^32 / g and 2^32 / g^2, g the plastic number
# the face table: d is normalize(vector(a, b)) per face, in the order +X, -X, +Y, -Y, +Z, -Z
FACES = (lambda a, b, o: (o, -b, -a), lambda a, b, o: (-o, -b, a), lambda a, b, o: (a, o, b),
         lambda a, b, o: (a, -o, -b), lambda a, b, o: (a, -b, o), lambda a, b, o: (-a, -b, -o))


# ---- helpers ----------------------------------------------------------------------------------------------------------------------
def cubemap_rays(octx, positions, N, samples, seed):
    """orCubemapRays: every sample's start (position, d, H(H(seed + tau) + k)) as n * 6 * N^2 * samples PATH_RAY_DTYPE records."""
    L = octx._L
    L.orCubemapRays.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_uint32, C.c_void_p]
    pos = np.ascontiguousarray(positions, dtype=np.float32).reshape(-1, 3)
    out = np.zeros(len(pos) * 6 * N * N * samples, dtype=capi.PATH_RAY_DTYPE)
    assert L.orCubemapRays(octx.handle, pos.ctypes.data, len(pos), N, samples, seed, out.ctypes.data) == capi.RT_OK
    return out


def oracle_texels(octx, positions, N, samples, seed, first, count):
    """orCubemapTexels: texels first .. first + count - 1 of the call, from the oracle."""
    L = octx._L
    L.orCubemapTexels.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_uint32, C.c_int, C.c_int, C.c_void_p]
    pos = np.ascontiguousarray(positions, dtype=np.float32).reshape(-1, 3)
    out = np.zeros(count, dtype=capi.CUBE_TEXEL_DTYPE)
    assert L.orCubemapTexels(octx.handle, pos.ctypes.data, len(pos), N, samples, seed, first, count, out.ctypes.data) == capi.RT_OK
    return out


def offsets32(samples):
    """The header's R2 sub-texel offsets in binary32: (u, v), each (samples,)."""
    k = np.arange(samples, dtype=np.uint64)
    return tuple(((k * c + 2 ** 31) % 2 ** 32).astype(np.uint32).astype(np.float32) * np.float32(2.0 ** -32) for c in R2)


def directions32(N, samples):
    """The header's directions restated in numpy binary32, one operation at a time: (6, N, N, samples, 3)."""
    f = np.float32
    u, v = offsets32(samples)
    xs = np.arange(N, dtype=np.float32)
    a = ((((xs[None, :, None] + u[None, None, :]) / f(N)) * f(2)) - f(1)).astype(f)            # (1, x, k)
    b = ((((xs[:, None, None] + v[None, None, :]) / f(N)) * f(2)) - f(1)).astype(f)            # (y, 1, k)
    a, b = np.broadcast_arrays(a, b)
    one = np.ones_like(a)
    out = np.empty((6, N, N, samples, 3), dtype=f)
    for face, vec in enumerate(FACES):
        w = np.stack(vec(a, b, one), axis=-1).astype(f)
        dot = ((w[..., 0] * w[..., 0] + w[..., 1] * w[..., 1]) + w[..., 2] * w[..., 2]).astype(f)
        inv = (f(1) / np.sqrt(dot)).astype(f)
        out[face] = w * inv[..., None]
    return out


def mean32(radiance, texels, samples):
    """The header's sums restated in numpy binary32 from the samples' radiances: (rgb (texels, 3), rejected (texels,))."""
    f = np.float32
    chunk = capi.RT_PROBE_CHUNK
    chunks = -(-samples // chunk)
    L = radiance.reshape(texels, samples, 3).astype(f)
    ok = np.isfinite(L).all(axis=-1)
    pad = np.zeros((texels, chunks * chunk, 3), dtype=f)                                        # +0 adds nothing to a sum from +0
    pad[:, :samples] = np.where(ok[..., None], L, f(0))
    pad = pad.reshape(texels, chunks, chunk, 3)
    sums = np.zeros((texels, chunks, 3), dtype=f)
    for j in range(chunk):                                                                      # k order within a chunk
        sums = (sums + pad[:, :, j]).astype(f)
    width = 1
    while width < chunks:
        width *= 2
    tree = np.zeros((texels, width, 3), dtype=f)
    tree[:, :chunks] = sums
    while tree.shape[1] > 1:                                                                    # adjacent pairs, level by level
        tree = (tree[:, 0::2] + tree[:, 1::2]).astype(f)
    return (tree[:, 0] / f(samples)).astype(f), (~ok).sum(axis=1).astype(np.uint32)


def assert_texels_equal(a, b, what):
    a, b = np.asarray(a).reshape(-1), np.asarray(b).reshape(-1)
    assert_bit_equal(np.ascontiguousarray(a["rgb"]), np.ascontiguousarray(b["rgb"]), f"{what}: rgb")
    bad = np.flatnonzero(a["rejected"] != b["rejected"])
    assert len(bad) == 0, f"{what}: rejected differs for {len(bad)} texels, first {bad[0]}: {a['rejected'][bad[0]]} vs {b['rejected'][bad[0]]}"


def bake(ctx, positions, N, samples, seed, stats=False):
    ctx.reset_stats()
    out = ctx.bake_cubemaps(positions, N, samples, seed)
    return (out, ctx.stats()) if stats else out


def check_oracle(sc, positions, options_list=({},), cases=None, bounces=None, seed=7, sky=None):
    """rtBakeCubemaps against the oracle for every ((faceSize, samples), MaxBounceCount), each option set with modelSkip 1 and 0 and a
    counting run: texel bits, rejected, RtStats.rays and, counting, the box / triangle / sphere counters."""
    runs = [(c, m) for c in (cases or CASES) for m in (bounces or BOUNCES)]
    ref_mgr = T.open_mgr(ORACLE_LIB, sc)
    if sky is not None:
        ref_mgr.context.set_int("UseSky", sky)
    ref = {}
    for (N, s), m in runs:
        ref_mgr.context.set_int("MaxBounceCount", m)
        ref[(N, s, m)] = bake(ref_mgr.context, positions, N, s, seed, stats=True)
    ref_mgr.OnDestroy()
    for opts in list(options_list) + [{"countStats": 1}]:
        for skip in ((opts["modelSkip"],) if "modelSkip" in opts else (1, 0)):
            mgr = T.open_mgr(CUDA_LIB, sc, dict(opts, modelSkip=skip))
            if sky is not None:
                mgr.context.set_int("UseSky", sky)
            for (N, s, m), (want, wst) in ref.items():
                mgr.context.set_int("MaxBounceCount", m)
                got, gst = bake(mgr.context, positions, N, s, seed, stats=True)
                what = f"{sc.name} {opts} modelSkip={skip} faceSize={N} samples={s} MaxBounceCount={m}"
                assert got.shape == (len(positions), 6, N, N) and got.dtype == capi.CUBE_TEXEL_DTYPE
                assert_texels_equal(got, want, what)
                keys = (P.COUNTS(sc) if opts.get("countStats") else ("rays",))
                assert all(gst[k] == wst[k] for k in keys), (what, gst, wst)
                assert gst["dispatches"] == 0 and gst["kernelMs"] == 0
            mgr.OnDestroy()
    return ref


def richest(ref):
    """The result of the largest case of check_oracle's: most bounces, then most texels x samples."""
    return ref[max(ref, key=lambda k: (k[2], k[0] * k[0] * k[1]))][0]


def emissive_quad(p0, p1, p2, p3, emission, strength):
    """A scene of one emissive quad (normal cross(p1 - p0, p2 - p0)), no sky: a miss is black."""
    sc = scenes.Scene("quad", 16, 12, cam_local_to_world=np.eye(4), settings=dict(useSky=False, maxBounceCount=0))
    sc.meshes = [scenes.quad_mesh(p0, p1, p2, p3)]
    m, w = scenes.trs()
    sc.models = [scenes.ModelDesc(0, m, w, scenes.material(diffuse=(0, 0, 0), emission=emission, emissionStrength=strength,
                                                             specularProbability=0.0))]
    return sc


# ---- against the oracle -----------------------------------------------------------------------------------------------------------
def test_oracle_cornell_spheres():
    sc = scenes.cornell_spheres(24, 16, 4, 1)
    ref = check_oracle(sc, P.probe_positions(sc, seed=1, n=PROBES))
    lit = richest(ref)["rgb"][:PROBES]
    assert (lit > 0).any(axis=(1, 2, 3, 4)).all()        # every in-scene probe sees light on some face


def test_oracle_knot_room_with_glass():
    sc = scenes.knot_room(24, 16, 4, 1, nu=40, nv=8, glass=True)
    check_oracle(sc, P.probe_positions(sc, seed=2, n=PROBES), sky=1)


def test_oracle_soup_with_sky_and_spheres():
    sc = G._soup_with_sky_and_defocus()
    check_oracle(sc, P.probe_positions(sc, seed=3, n=PROBES))


@pytest.mark.parametrize("tlas", [-1, 0, 1])
def test_oracle_above_128_models_with_the_tlas(tlas):
    sc = scenes.instanced_knots(24, 16, 4, 1, instances=150)
    check_oracle(sc, P.probe_positions(sc, seed=4, n=PROBES), ({"tlas": tlas},))


def test_oracle_ten_thousand_spheres_with_the_accelerator():
    sc = scenes.random_soup(24, 16, 4, 1, triangles=300, spheres=10000)
    check_oracle(sc, P.probe_positions(sc, seed=5, n=PROBES), ({}, {"extInstantiation": 1}), sky=1)


def test_oracle_unity_fixture():
    from test_round2_abi import load_fixture
    sc = load_fixture(24, 16)
    check_oracle(sc, P.probe_positions(sc, seed=6, n=PROBES))


def test_oracle_nan_sun_rejects_samples():
    """The NaN-sun scene of test_gpu_probes.py: every path that reaches the sky is NaN; those samples are counted in `rejected`, count
    as black, and every in-scene texel stays finite."""
    sc = scenes.random_soup(24, 16, max_bounces=3, rays_per_pixel=1, triangles=600, spheres=8)
    sc.settings["sunIntensity"] = float("nan")
    ref = check_oracle(sc, P.probe_positions(sc, seed=8, n=PROBES), sky=1)
    got = richest(ref)[:PROBES]
    assert got["rejected"].sum() > 0 and np.isfinite(got["rgb"]).all()


# ---- the rebuild through rtTracePaths ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N, samples", [(3, 33), (2, 1025)])
def test_rebuild_through_trace_paths(N, samples):
    """orCubemapRays -> this build's rtTracePaths(samples = 1) -> numpy: the chunk sums in k order, the padded tree and the division
    give rtBakeCubemaps' bits; the NaN-sun sky makes some samples non-finite, which both leave out.  The hook's directions are the
    numpy binary32 restatement of the R2 offsets and the face table, bit for bit."""
    sc = scenes.knot_room(24, 16, 4, 1, nu=40, nv=8, glass=True)
    sc.settings = dict(sc.settings, useSky=True)
    pos = P.probe_positions(sc, seed=9, n=2)
    ref = T.open_mgr(ORACLE_LIB, sc)
    mgr = T.open_mgr(CUDA_LIB, sc)
    texels = len(pos) * 6 * N * N
    for sun in (10.0, float("nan")):
        mgr.context.set_float("SunIntensity", sun)
        rays = cubemap_rays(ref.context, pos, N, samples, 21)
        want = mean32(mgr.context.trace_paths(rays, 1)["rgb"], texels, samples)
        got = mgr.context.bake_cubemaps(pos, N, samples, 21).reshape(-1)
        assert_bit_equal(got["rgb"], want[0], f"SunIntensity={sun}: rgb")
        assert np.array_equal(got["rejected"], want[1]), f"SunIntensity={sun}: rejected"
        assert (want[1] > 0).any() == (sun != sun)
    d = directions32(N, samples)
    assert_bit_equal(rays["dir"].reshape(len(pos), 6, N, N, samples, 3)[0], d, "the hook's directions vs numpy")
    assert_bit_equal(rays["dir"].reshape(len(pos), 6, N, N, samples, 3)[1], d, "the second probe's directions")
    assert np.array_equal(rays["origin"].reshape(len(pos), -1, 3).view(np.uint32),
                          np.repeat(pos[:, None], 6 * N * N * samples, axis=1).view(np.uint32))
    ref.OnDestroy()
    mgr.OnDestroy()


# ---- orientation ------------------------------------------------------------------------------------------------------------------
def test_faces_in_a_room_of_six_coloured_walls():
    """The probe at the centre of a closed room whose walls (+X, -X, +Y, -Y, +Z, -Z, each 1 from the centre) emit six colours, no bounce,
    one sample (the texel centres): every texel of face f is wall f's emission x strength bit for bit.  Texel (0, 0) and (N - 1, N - 1)
    of each face point into the octants the face table gives, checked in float64 from the hook's directions."""
    R = 1000.0
    colours = [(1.0, 0.0, 0.0), (0.0, 1.0, 0.0), (0.0, 0.0, 1.0), (1.0, 1.0, 0.0), (0.0, 1.0, 1.0), (1.0, 0.0, 1.0)]
    strengths = [2.0, 3.0, 5.0, 7.0, 11.0, 13.0]
    axes = [(1, 0, 0), (-1, 0, 0), (0, 1, 0), (0, -1, 0), (0, 0, 1), (0, 0, -1)]
    sph = [scenes._sphere(tuple((R + 1.0) * np.array(ax)), R, scenes.material(diffuse=(0, 0, 0), emission=c, emissionStrength=s,
                                                                                 specularProbability=0.0))
           for ax, c, s in zip(axes, colours, strengths)]
    sc = scenes.Scene("six walls", 16, 12, spheres=np.array(sph, dtype=scenes.SPHERE_DTYPE), cam_local_to_world=np.eye(4),
                      settings=dict(useSky=False, maxBounceCount=0))
    N = 8
    pos = np.zeros((1, 3), dtype=np.float32)
    mgr = T.open_mgr(CUDA_LIB, sc)
    got = mgr.context.bake_cubemaps(pos, N, 1, 5)[0]
    mgr.OnDestroy()
    for f in range(6):
        E = (np.float32(colours[f]) * np.float32(strengths[f])).astype(np.float32)
        assert_bit_equal(got[f]["rgb"], np.broadcast_to(E, (N, N, 3)).copy(), f"face {f}")
        assert (got[f]["rejected"] == 0).all()
    ref = T.open_mgr(ORACLE_LIB, sc)
    d = cubemap_rays(ref.context, pos, N, 1, 5)["dir"].reshape(6, N, N, 3).astype(np.float64)
    ref.OnDestroy()
    # (sign of x, y, z) at texel (0, 0) and at (N - 1, N - 1): a, b = -1 + 1/N and 1 - 1/N through the table
    octants = [((1, 1, 1), (1, -1, -1)), ((-1, 1, -1), (-1, -1, 1)), ((-1, 1, -1), (1, 1, 1)),
               ((-1, -1, 1), (1, -1, -1)), ((-1, 1, 1), (1, -1, 1)), ((1, 1, -1), (-1, -1, -1))]
    for f in range(6):
        assert tuple(np.sign(d[f, 0, 0]).astype(int)) == octants[f][0], (f, d[f, 0, 0])
        assert tuple(np.sign(d[f, N - 1, N - 1]).astype(int)) == octants[f][1], (f, d[f, N - 1, N - 1])
        assert np.argmax(np.abs(d[f]).reshape(-1, 3).sum(axis=0)) == f // 2          # the face's axis dominates
        assert np.allclose(np.linalg.norm(d[f], axis=-1), 1.0, atol=4 * U)


# ---- anti-aliasing ----------------------------------------------------------------------------------------------------------------
def _coverage(lo, hi, edge, below):
    """The fraction of [lo, hi] on the covered side of `edge` (below: the side < edge), float64."""
    t = np.clip((edge - lo) / (hi - lo), 0.0, 1.0)
    return t if below else 1.0 - t


@pytest.mark.parametrize("edge", ["a", "b"])
def test_a_straight_edge_is_anti_aliased(edge):
    """An emissive wall with a straight edge through the inside of a column (line of constant a, on +X) or of a row (constant b, on
    +Y), no bounce, 1,024 samples: each texel is the emission times the fraction of its area the wall covers, within 1/128 of the
    emission (about twice the extreme discrepancy of the 1,024 R2 offsets: 0.0021 in u, 0.0031 in v).  A centre ray per texel with the
    same samples (rtTracePaths) reads 0 or the full emission on the same texels."""
    N, S, E = AA_FACE, 1024, np.float32(4.0)
    Y = 1000.0
    lo = np.arange(N) / N * 2 - 1
    hi = (np.arange(N) + 1) / N * 2 - 1
    i = N // 2 + N // 4                                  # the edge at 40% of column / row i
    e = lo[i] + 0.4 * (hi[i] - lo[i])
    if edge == "a":
        # plane x = 1, covered where z >= -e: on +X (1, -b, -a) that is a <= e
        sc = emissive_quad((1, -Y, -e), (1, -Y, Y), (1, Y, Y), (1, Y, -e), (1, 1, 1), E)
        face = 0
    else:
        # plane y = 1, covered where z >= e: on +Y (a, 1, b) that is b >= e
        sc = emissive_quad((-Y, 1, e), (Y, 1, e), (Y, 1, Y), (-Y, 1, Y), (1, 1, 1), E)
        face = 2
    pos = np.zeros((1, 3), dtype=np.float32)
    mgr = T.open_mgr(CUDA_LIB, sc)
    got = mgr.context.bake_cubemaps(pos, N, S, 3)[0, face]["rgb"].astype(np.float64)
    if edge == "a":
        frac = np.broadcast_to(_coverage(lo, hi, e, True)[None, :], (N, N))
    else:
        frac = np.broadcast_to(_coverage(lo, hi, e, False)[:, None], (N, N))
    want = float(E) * frac
    assert (np.abs(got - want[..., None]) <= float(E) / 128).all(), np.abs(got - want[..., None]).max()
    partial = (frac > 0) & (frac < 1)
    assert partial.sum() == N and np.allclose(frac[partial], 0.4 if edge == "a" else 0.6)
    # the centre-ray route: one direction per texel (sample 0's offset is the centre), all S samples along it
    ref = T.open_mgr(ORACLE_LIB, sc)
    centre = cubemap_rays(ref.context, pos, N, 1, 3).reshape(6, N, N)[face].reshape(-1)
    ref.OnDestroy()
    one = mgr.context.trace_paths(centre, S)["rgb"].reshape(N, N, 3)
    mgr.OnDestroy()
    assert np.isin(one[partial], [0.0, E]).all()
    assert (np.abs(got[partial] - float(E) / 2) < float(E) / 4).all()


# ---- seeds and texel indices ------------------------------------------------------------------------------------------------------
def test_seed_and_texel_index_enter_only_as_seed_plus_tau():
    """Probe 1 of a two-probe call at seed s is the one-probe call at seed s + 6 N^2 (tau counts from the call's first texel); the
    same call again is the same; another seed gives other paths."""
    sc = scenes.cornell_spheres(24, 16, 4, 1)
    pos = P.probe_positions(sc, seed=10, n=2, special=False)
    mgr = T.open_mgr(CUDA_LIB, sc)
    ctx = mgr.context
    N, s = 3, 40
    full = ctx.bake_cubemaps(pos, N, s, 0xFFFFFFF0)
    assert_texels_equal(ctx.bake_cubemaps(pos[:1], N, s, 0xFFFFFFF0)[0], full[0], "probe 0")
    assert_texels_equal(ctx.bake_cubemaps(pos[1:], N, s, (0xFFFFFFF0 + 6 * N * N) & 0xFFFFFFFF)[0], full[1], "probe 1 at seed + 6N^2")
    assert_texels_equal(ctx.bake_cubemaps(pos, N, s, 0xFFFFFFF0), full, "the same call again")
    assert not np.array_equal(ctx.bake_cubemaps(pos, N, s, 1)["rgb"], full["rgb"])
    mgr.OnDestroy()


# ---- isolation --------------------------------------------------------------------------------------------------------------------
def test_bakes_between_frames_change_nothing_the_frames_show():
    sc = scenes.instanced_knots(32, 24, 4, 2, instances=150)
    pos = P.probe_positions(sc, seed=11, n=2)
    images = []
    for with_bakes in (False, True):
        mgr = T.open_mgr(CUDA_LIB, sc, {"countStats": 1})
        ctx = mgr.context
        ctx.reset_stats()
        for _ in range(3):
            mgr.RenderFrame()
            if with_bakes:
                before, frame = ctx.stats(), mgr.raytraceFrameTex
                ctx.bake_cubemaps(pos, 2, 33, 5)
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
    pos = P.probe_positions(sc, seed=12, n=2)
    for lib in (ORACLE_LIB, CUDA_LIB):
        mgr = T.open_mgr(lib, sc, enable=False)          # no OnEnable: no rtResize, no dispatch
        ctx = mgr.context
        want = mgr.bake_cubemaps(pos, 2, 33, 3)
        ctx.set_int("Frame", 17)
        ctx.set_int("renderSeed", 999)
        ctx.set_int("NumRaysPerPixel", 7)
        ctx.set_matrix("CamLocalToWorldMatrix", np.eye(4, dtype=np.float32) * 2.0)
        assert_texels_equal(ctx.bake_cubemaps(pos, 2, 33, 3), want, f"{lib}: after Frame / renderSeed / camera / NumRaysPerPixel changed")
        mgr.OnDestroy()


# ---- refusals ---------------------------------------------------------------------------------------------------------------------
def test_empty_call_and_every_error_code():
    sc = scenes.knot_room(16, 12, 3, 1, nu=30, nv=6)
    for lib in (ORACLE_LIB, CUDA_LIB):
        mgr = T.open_mgr(lib, sc)
        ctx, L, h = mgr.context, mgr.context._L, mgr.context.handle
        pos = P.probe_positions(sc, n=2, special=False)
        out = np.zeros(len(pos) * 6, dtype=capi.CUBE_TEXEL_DTYPE)
        st = ctx.stats()
        assert L.rtBakeCubemaps(h, None, 0, 1, 1, 0, None) == capi.RT_OK and ctx.stats()["rays"] == st["rays"]
        assert ctx.bake_cubemaps(np.zeros((0, 3)), 4, 1).shape == (0, 6, 4, 4)
        assert L.rtBakeCubemaps(None, pos.ctypes.data, len(pos), 1, 1, 0, out.ctypes.data) == capi.RT_E_INVALID
        assert L.rtBakeCubemaps(h, pos.ctypes.data, -1, 1, 1, 0, out.ctypes.data) == capi.RT_E_INVALID
        assert L.rtBakeCubemaps(h, None, len(pos), 1, 1, 0, out.ctypes.data) == capi.RT_E_INVALID
        assert L.rtBakeCubemaps(h, pos.ctypes.data, len(pos), 1, 1, 0, None) == capi.RT_E_INVALID
        for s in (0, -1, capi.RT_MAX_BATCH_SAMPLES + 1):
            assert L.rtBakeCubemaps(h, pos.ctypes.data, len(pos), 1, s, 0, out.ctypes.data) == capi.RT_E_INVALID, s
        for N in (0, -1, capi.RT_CUBE_MAX_FACE + 1):
            assert L.rtBakeCubemaps(h, pos.ctypes.data, len(pos), N, 1, 0, out.ctypes.data) == capi.RT_E_INVALID, N
            assert L.rtBakeCubemaps(h, pos.ctypes.data, 0, N, 1, 0, out.ctypes.data) == capi.RT_E_INVALID, N
        # 2^31 - 1 texels at most: 21,846 probes of 6 x 128^2 are past it (and are refused before anything is read)
        assert L.rtBakeCubemaps(h, pos.ctypes.data, 21846, 128, 1, 0, out.ctypes.data) == capi.RT_E_INVALID
        for m in (-1, 201):
            ctx.set_int("MaxBounceCount", m)
            assert L.rtBakeCubemaps(h, pos.ctypes.data, len(pos), 1, 1, 0, out.ctypes.data) == capi.RT_E_STATE, m
            assert L.rtBakeCubemaps(h, pos.ctypes.data, 0, 1, 1, 0, out.ctypes.data) == capi.RT_OK
        ctx.set_int("MaxBounceCount", 200)
        assert L.rtBakeCubemaps(h, pos.ctypes.data, len(pos), 1, 1, 0, out.ctypes.data) == capi.RT_OK
        ctx.set_int("MaxBounceCount", 0)
        assert L.rtBakeCubemaps(h, pos.ctypes.data, len(pos), 1, 1, 0, out.ctypes.data) == capi.RT_OK
        ctx.set_int("modelCount", 99)
        assert L.rtBakeCubemaps(h, pos.ctypes.data, len(pos), 1, 1, 0, out.ctypes.data) == capi.RT_E_STATE
        ctx.set_int("modelCount", 2)
        models = np.zeros(2, dtype=capi.MODEL_DTYPE)
        models[1]["nodeOffset"] = 10 ** 7
        ctx.set_buffer("ModelInfo", models)
        assert L.rtBakeCubemaps(h, pos.ctypes.data, len(pos), 1, 1, 0, out.ctypes.data) == capi.RT_E_STATE
        ctx.set_buffer("Nodes", np.zeros(0, dtype=capi.NODE_DTYPE))
        assert L.rtBakeCubemaps(h, pos.ctypes.data, len(pos), 1, 1, 0, out.ctypes.data) == capi.RT_E_STATE
        assert L.rtBakeCubemapsDevice(None, None, None, 0, 1, 1, 0) == capi.RT_E_INVALID
        if lib == CUDA_LIB:                              # (the oracle has no device form: RT_E_STATE)
            assert L.rtBakeCubemapsDevice(h, None, None, 0, 1, 0, 0) == capi.RT_E_INVALID
            assert L.rtBakeCubemapsDevice(h, None, None, 0, 0, 1, 0) == capi.RT_E_INVALID
            assert L.rtBakeCubemapsDevice(h, None, None, -1, 1, 1, 0) == capi.RT_E_INVALID
            assert L.rtBakeCubemapsDevice(h, None, None, 0, 1, 1, 0) == capi.RT_OK
        mgr.OnDestroy()
    from test_round2_abi import chain_bvh, one_model_scene
    for lib in (ORACLE_LIB, CUDA_LIB):
        mgr = T.open_mgr(lib, one_model_scene(16, 12))
        tris, nodes = chain_bvh(64)
        mgr.context.set_buffer("Triangles", tris)
        mgr.context.set_buffer("Nodes", nodes)
        with pytest.raises(capi.RtError) as e:
            mgr.context.bake_cubemaps(np.zeros((1, 3)), 1, 1)
        assert e.value.code == capi.RT_E_STATE and "too deep" in str(e.value), lib
        mgr.OnDestroy()


def test_cpp_manager_equals_the_python_context():
    sc = scenes.knot_room(24, 16, 4, 1, nu=40, nv=8, glass=True)
    pos = P.probe_positions(sc, seed=13, n=2)
    for lib in (ORACLE_LIB, CUDA_LIB):
        mgr = T.open_mgr(lib, sc)
        assert_texels_equal(mgr.bake_cubemaps(pos, 3, 33, 9), mgr.context.bake_cubemaps(pos, 3, 33, 9),
                            f"{lib}: RayComputeManager.BakeCubemaps vs the context")
        mgr.OnDestroy()


# ---- against float64 --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N, samples", [(4, 1), (2, 33), (1, 1025)])
def test_sky_alone_against_float64(N, samples):
    """No geometry, the sky on: every sample is the sky in its direction.  Each texel is the float64 mean of the restated sky over its
    own sample directions (the hook's binary32 ones), within the sum's rounding (32 additions in a chunk, the tree's depth, the division)
    plus 64 ulps of the sky per sample (as test_gpu_probes.py::test_sky_alone_against_float64 derives)."""
    sc = scenes.Scene("sky", 16, 12, cam_local_to_world=np.eye(4), settings=dict(useSky=True, maxBounceCount=4),
                      sun_forward=(-0.3, -0.8, -0.52))
    pos = np.array([[0.0, 0.0, 0.0], [3.0, -1.0, 2.0]], dtype=np.float32)
    ref = T.open_mgr(ORACLE_LIB, sc)
    rays = cubemap_rays(ref.context, pos, N, samples, 3)
    ref.OnDestroy()
    d = rays["dir"].astype(np.float64)
    L64 = P.sky64(d, np.float32([0.3, 0.8, 0.52]).astype(np.float64), 500.0, 10.0).reshape(-1, samples, 3)
    want = L64.mean(axis=1)
    mag = np.abs(L64).sum(axis=1) / samples
    depth = max(0, int(np.ceil(np.log2(-(-samples // capi.RT_PROBE_CHUNK)))))
    tol = mag * ((capi.RT_PROBE_CHUNK + depth + 2) * U + 64 * U)
    mgr = T.open_mgr(CUDA_LIB, sc)
    got = mgr.context.bake_cubemaps(pos, N, samples, 3).reshape(-1)
    mgr.OnDestroy()
    assert (got["rejected"] == 0).all()
    err = np.abs(got["rgb"].astype(np.float64) - want)
    assert (err <= tol).all(), (err.max(), (err / tol).max())


# ---- write_cubemap_exr ------------------------------------------------------------------------------------------------------------
def test_write_cubemap_exr_round_trips_the_faces_in_order(tmp_path):
    N = 5
    faces = np.zeros((6, N, N), dtype=capi.CUBE_TEXEL_DTYPE)
    faces["rgb"] = np.random.RandomState(3).standard_normal((6, N, N, 3)).astype(np.float32) * 100
    faces["rgb"][2, 1, 3] = (np.inf, 0.0, -0.0)
    path = str(tmp_path / "probe.exr")
    display.write_cubemap_exr(path, faces)
    img = display.read_exr(path)
    assert img.shape == (N, 6 * N, 4)
    for f in range(6):
        assert_bit_equal(img[:, f * N:(f + 1) * N, :3], faces["rgb"][f], f"face {f}")
    assert (img[..., 3] == 1.0).all()
    display.write_cubemap_exr(path, faces["rgb"])                       # a plain (6, N, N, 3) float array too
    assert display.read_exr(path).tobytes() == img.tobytes()


# ---- GPU only ---------------------------------------------------------------------------------------------------------------------
def test_texel_indices_across_internal_launches():
    """32,800 samples are 1,025 chunks, so a launch holds floor(7 * 2^20 / 1025) = 7,161 texels: two probes of 6 x 35^2 = 7,350
    texels take three launches, split inside probe 0's -Z face and probe 1's +X face.  The host and device forms equal each other, and
    the oracle's texels on both sides of each boundary (and the first and last) equal the call."""
    torch = pytest.importorskip("torch")
    samples, N = 32 * 1025, 35
    per = capi.RT_CUBE_SCRATCH_CHUNKS // (samples // capi.RT_PROBE_CHUNK)
    assert per == 7161
    sc = scenes.cornell_spheres(24, 16, 4, 1)
    pos = P.probe_positions(sc, seed=14, n=2, special=False)
    total = len(pos) * 6 * N * N
    assert per < 6 * N * N < 2 * per < total < 3 * per
    mgr = T.open_mgr(CUDA_LIB, sc)
    got = mgr.context.bake_cubemaps(pos, N, samples, 77).reshape(-1)
    d_pos = torch.from_numpy(pos).cuda()
    d_out = torch.zeros(total * 16, dtype=torch.uint8, device="cuda")
    mgr.context.bake_cubemaps_device(d_pos.data_ptr(), d_out.data_ptr(), len(pos), N, samples, 77)
    mgr.context.synchronize()
    dev = d_out.cpu().numpy().view(capi.CUBE_TEXEL_DTYPE)
    mgr.OnDestroy()
    assert_texels_equal(dev, got, "device form vs host form across launches")
    ref = T.open_mgr(ORACLE_LIB, sc)
    for t in (0, per - 1, per, 2 * per - 1, 2 * per, total - 1):
        assert_texels_equal(got[t: t + 1], oracle_texels(ref.context, pos, N, samples, 77, t, 1), f"texel {t}")
    ref.OnDestroy()


def test_device_form_on_the_context_stream_and_a_caller_stream():
    torch = pytest.importorskip("torch")
    sc = scenes.instanced_knots(24, 16, 4, 1, instances=150)
    pos = P.probe_positions(sc, seed=15, n=6)
    n, N = len(pos), 4
    texels = n * 6 * N * N
    mgr = T.open_mgr(CUDA_LIB, sc)
    ctx = mgr.context
    want = ctx.bake_cubemaps(pos, N, 100, 4)
    raw = torch.zeros(n * 12 + 4, dtype=torch.uint8)
    raw[4:] = torch.from_numpy(pos.view(np.uint8).reshape(-1).copy())
    d_raw = raw.cuda()
    for stream in (None, torch.cuda.Stream()):
        d_out = torch.full((texels * 16 + 16,), 0x5a, dtype=torch.uint8, device="cuda")
        if stream is not None:
            ctx.set_stream(stream.cuda_stream)
        ctx.bake_cubemaps_device(d_raw.data_ptr() + 4, d_out.data_ptr(), n, N, 100, 4)       # 4-byte aligned positions
        ctx.synchronize()
        got = d_out.cpu().numpy()
        assert (got[texels * 16:] == 0x5a).all()
        assert_texels_equal(got[: texels * 16].view(capi.CUBE_TEXEL_DTYPE), want, f"device form, stream {stream}")
    ctx.set_stream(0)
    for pp, op in ((d_raw.data_ptr() + 2, d_out.data_ptr()), (d_raw.data_ptr() + 4, d_out.data_ptr() + 4)):
        with pytest.raises(capi.RtError) as e:
            ctx.bake_cubemaps_device(pp, op, n, N, 1)
        assert e.value.code == capi.RT_E_INVALID
    mgr.OnDestroy()
    o = capi.RtLib(ORACLE_LIB).create(0)
    assert o._L.rtBakeCubemapsDevice(o.handle, None, None, 0, 1, 1, 0) == capi.RT_E_STATE


def test_four_probes_on_the_871k_triangle_cluster():
    """Four probes at faceSize 64, 64 samples and MaxBounceCount 12 against the oracle's texels for a seeded subset of 24."""
    sc = scenes.knot_cluster(64, 36, 12, 1)
    pos = P.probe_positions(sc, seed=16, n=4, special=False)
    mgr = T.open_mgr(CUDA_LIB, sc)
    got = mgr.context.bake_cubemaps(pos, 64, 64, 1234).reshape(-1)
    mgr.OnDestroy()
    ref = T.open_mgr(ORACLE_LIB, sc)
    for t in np.random.RandomState(17).choice(len(got), 24, replace=False):
        assert_texels_equal(got[t: t + 1], oracle_texels(ref.context, pos, 64, 64, 1234, int(t), 1), f"texel {t}")
    ref.OnDestroy()
    assert ((got["rgb"][:, 0] > 0).reshape(len(pos), -1).mean(axis=1) > 0.05).all()     # every probe sees lit surfaces
