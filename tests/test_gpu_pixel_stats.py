"""Per-pixel traversal counters ("PixelStats") and their heat map (rtReadbackPixelStats / rtDisplayPixelStats) on the H100
(`-m gpu`): every kernel's counting launch attributes each pixel's rays, box, triangle and sphere tests exactly as the CPU oracle
counts them, the image sums to the RtStats totals, and counting leaves the rendered images unchanged.  The same bodies run in the
CPU suite against the SIMT interpreter build (tests/test_simt_pixel_stats.py)."""
import ctypes as C

import numpy as np
import pytest

from conftest import CUDA_LIB, ORACLE_LIB, assert_bit_equal
import ray_tracing_b200 as rt
from ray_tracing_b200 import capi, scenes

pytestmark = pytest.mark.gpu

FIELDS = ("rays", "boxTests", "triTests", "sphereTests", "sphereBoxTests")


def run(lib, sc, frames=1, options=None, tile=None):
    """Render `frames` frames through the host manager with "countStats" = 1 (unless options say otherwise);
    returns (frame, accumulated, RtStats dict, PixelStats image or None)."""
    mgr = rt.RayComputeManager(lib)
    scenes.apply(sc, mgr)
    ctx = mgr.context
    opts = {"countStats": 1}
    opts.update(options or {})
    for k, v in opts.items():
        ctx.set_option(k, v)
    if tile:
        ctx.set_tile(*tile)
    mgr.OnEnable()
    ctx.reset_stats()
    for _ in range(frames):
        mgr.RenderFrame()
    pix = mgr.pixel_stats() if opts["countStats"] else None
    out = (mgr.raytraceFrameTex, mgr.accumulatedResult, ctx.stats(), pix)
    mgr.OnDestroy()
    return out


def assert_sums_match(pix, st, what=""):
    for k in FIELDS:
        assert int(pix[k].astype(np.uint64).sum()) == st[k], f"{what}: sum of PixelStats.{k} = {int(pix[k].astype(np.uint64).sum())}, RtStats.{k} = {st[k]}"


def assert_pixels_equal(got, ref, fields=FIELDS, what=""):
    for k in fields:
        bad = np.argwhere(got[k] != ref[k])
        assert len(bad) == 0, f"{what}: PixelStats.{k} differs at {len(bad)} pixels, first (y, x) = {bad[0].tolist()}: {got[k][tuple(bad[0])]} vs {ref[k][tuple(bad[0])]}"


def check_against_oracle(sc, frames=1, options_list=({},), fields=FIELDS):
    """The counting launch of every option set: images equal to the oracle's and to a plain launch, PixelStats equal to the
    oracle's (fields), and the image sums equal to RtStats."""
    fo, ao, so, po = run(ORACLE_LIB, sc, frames)
    assert_sums_match(po, so, "oracle")
    for opts in options_list:
        fg, ag, sg, pg = run(CUDA_LIB, sc, frames, opts)
        assert_bit_equal(fg, fo, f"{sc.name} {opts} FrameRender")
        assert_bit_equal(ag, ao, f"{sc.name} {opts} AccumulatedRender")
        fp, ap, _, _ = run(CUDA_LIB, sc, frames, dict(opts, countStats=0))
        assert_bit_equal(fg, fp, f"{sc.name} {opts}: counting launch vs plain launch, FrameRender")
        assert_bit_equal(ag, ap, f"{sc.name} {opts}: counting launch vs plain launch, AccumulatedRender")
        assert_pixels_equal(pg, po, fields, f"{sc.name} {opts}")
        assert_sums_match(pg, sg, f"{sc.name} {opts}")
    return po


@pytest.mark.parametrize("kernel", [0, 1, 2])
def test_spheres_and_meshes_per_pixel_equal_the_oracle(kernel):
    po = check_against_oracle(scenes.cornell_spheres(40, 30, 4, 2), frames=2, options_list=({"kernel": kernel},))
    assert po["sphereTests"].min() > 0
    po = check_against_oracle(scenes.knot_room(40, 24, 4, 2, nu=60, nv=8), options_list=({"kernel": kernel},))
    assert po["boxTests"].min() > 0 and po["triTests"].max() > 0


def test_sample_chunks_per_pixel_equal_the_oracle():
    """Kernel 1 with a pixel's samples in 2 and 3 chunks taken by different lanes: their shares add up to the pixel's counts."""
    check_against_oracle(scenes.knot_room(40, 24, 4, 6, nu=60, nv=8), options_list=({"kernel": 1, "sampleChunks": 2}, {"kernel": 1, "sampleChunks": 3}))


def test_pool_rays_carried_across_phases_per_pixel_equal_the_oracle():
    """Kernel 2: a ray is counted by the lane that pops it and may stay in flight across shade phases (tailLanes)."""
    sc = scenes.knot_room(48, 27, max_bounces=6, rays_per_pixel=2, nu=80, nv=8, glass=True)
    check_against_oracle(sc, options_list=tuple({"kernel": 2, "poolSlots": s, "tailLanes": t} for s in (32, 96) for t in (0, 31)))


@pytest.mark.parametrize("kernel", [0, 1, 2])
def test_sphere_accelerator_in_the_extension_instantiation(kernel):
    """80 spheres (above 64: the accelerator) in the <EXT> launch.  Rays and mesh tests per pixel equal the oracle's linear scan; the
    accelerator makes fewer sphere tests (at most one per sphere per ray) plus sphereBoxTests, summed exactly into RtStats."""
    sc = scenes.random_soup(32, 24, max_bounces=4, rays_per_pixel=2, triangles=2000, spheres=80)
    fo, ao, so, po = run(ORACLE_LIB, sc)
    fg, ag, sg, pg = run(CUDA_LIB, sc, options={"kernel": kernel, "extInstantiation": 1})
    assert_bit_equal(ag, ao, f"kernel {kernel}")
    assert_pixels_equal(pg, po, ("rays", "boxTests", "triTests"), f"kernel {kernel}")
    assert_sums_match(pg, sg, f"kernel {kernel}")
    assert np.all(pg["sphereTests"] <= po["sphereTests"]) and sg["sphereBoxTests"] > 0
    assert np.all(pg["sphereBoxTests"][pg["rays"] > 0] > 0)


def test_glass_mesh_and_unity_fixture_per_pixel_equal_the_oracle():
    sc = scenes.knot_room(40, 24, max_bounces=8, rays_per_pixel=2, nu=60, nv=8, glass=True)
    sc.models[1].material["flag"] = scenes.MAT_CHECKER
    check_against_oracle(sc, options_list=({"kernel": 0}, {"kernel": 1}, {"kernel": 2}))
    from test_round2_abi import load_fixture
    check_against_oracle(load_fixture(48, 27), options_list=({"kernel": 1}, {"kernel": 2}))


def test_accumulation_reset_resize_and_partial_dispatch():
    sc = scenes.knot_room(40, 24, 4, 2, nu=60, nv=8)
    lib = capi.RtLib(CUDA_LIB)
    mgr = rt.RayComputeManager(CUDA_LIB)
    scenes.apply(sc, mgr)
    ctx = mgr.context
    ctx.set_option("countStats", 1)
    mgr.OnEnable()
    ctx.reset_stats()
    ctx.dispatch_full()
    one = ctx.pixel_stats()
    assert one["rays"].min() >= 2
    ctx.dispatch_full()                                     # same Frame, nothing else changed: the same counts again
    two = ctx.pixel_stats()
    for k in FIELDS:
        assert np.array_equal(two[k], 2 * one[k]), k
    ctx.reset_stats()
    assert all(not ctx.pixel_stats()[k].any() for k in FIELDS)
    ctx.dispatch(capi.RT_KERNEL_RAYTRACE, 2, 1)             # pixels x < 16, y < 8 only
    part = ctx.pixel_stats()
    assert np.array_equal(part["rays"][:8, :16], one["rays"][:8, :16]) and not part["rays"][8:].any() and not part["rays"][:, 16:].any()
    ctx.dispatch_full()
    assert np.array_equal(ctx.pixel_stats()["rays"][8:], one["rays"][8:])
    ctx.resize(32, 16)
    ctx.set_ints("Resolution", [32, 16])
    assert ctx.pixel_stats().shape == (16, 32) and not ctx.pixel_stats()["rays"].any()
    mgr.OnDestroy()
    del lib


def test_sparse_pixels_of_a_large_scene_against_the_oracle():
    """A 640x360, 6-bounce, 4-spp mesh frame: 1024 seeded pixels of the GPU's PixelStats against orRenderPixelStats."""
    sc = scenes.knot_room(640, 360, max_bounces=6, rays_per_pixel=4, nu=400, nv=24, glass=True)
    _, _, sg, pg = run(CUDA_LIB, sc)
    assert_sums_match(pg, sg, "640x360")
    rng = np.random.RandomState(5)
    n = 1024
    xy = np.stack([rng.randint(0, sc.width, n), rng.randint(0, sc.height, n)], axis=1).astype(np.int32)
    mgr = rt.RayComputeManager(ORACLE_LIB)
    scenes.apply(sc, mgr)
    mgr.OnEnable()
    out = np.zeros(n, dtype=capi.PIXEL_STATS_DTYPE)
    assert C.CDLL(ORACLE_LIB).orRenderPixelStats(C.c_void_p(mgr.context.handle.value), xy.ctypes.data_as(C.c_void_p), n, out.ctypes.data_as(C.c_void_p)) == 0
    mgr.OnDestroy()
    got = pg[xy[:, 1], xy[:, 0]]
    for k in FIELDS:
        assert np.array_equal(got[k], out[k]), k


# ---- the heat map -----------------------------------------------------------------------------------------------------------------

def encode_reference(pix, vis_mode, scale):
    """The encode pinned in include/rt_b200.h, restated in numpy float32 (every operation rounds to binary32, RNE)."""
    rays = pix["rays"]
    if vis_mode == 4:
        v = rays.astype(np.float32)
    else:
        count = pix["boxTests"] if vis_mode == 1 else pix["triTests"] if vis_mode == 2 else (pix["sphereTests"] + pix["sphereBoxTests"]).astype(np.uint32)
        with np.errstate(divide="ignore", invalid="ignore"):
            v = count.astype(np.float32) / rays.astype(np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        t = v / np.float32(scale)
        g = np.trunc(np.where(t > 1, 0, t) * np.float32(255) + np.float32(0.5)).astype(np.uint8)
    out = np.empty(rays.shape + (4,), dtype=np.uint8)
    out[..., 0] = np.where(t > 1, 255, g); out[..., 1] = np.where(t > 1, 0, g); out[..., 2] = out[..., 1]; out[..., 3] = 255
    out[rays == 0] = (0, 0, 0, 255)
    return out


def _scales(pix):
    """Several scales per mode, among them values that put pixels exactly at the threshold (t == 1) and just beside it."""
    with np.errstate(divide="ignore", invalid="ignore"):
        box = pix["boxTests"].astype(np.float32) / pix["rays"].astype(np.float32)
    at = float(np.nanmax(box[pix["rays"] > 0]))
    return {1: [at, float(np.nextafter(np.float32(at), np.float32(0))), 1.0, 7.5, 1e6],
            2: [1.0, 3.0, 17.25, 1e3], 3: [0.5, 9.0, 100.0], 4: [float(pix["rays"].max()), 1.0, 2.0, 3.999]}


def test_display_equals_the_oracle_and_the_restated_encode():
    sc = scenes.random_soup(32, 24, max_bounces=3, rays_per_pixel=2, triangles=1500, spheres=12)
    ctxs = []
    for lib in (ORACLE_LIB, CUDA_LIB):
        mgr = rt.RayComputeManager(lib)
        scenes.apply(sc, mgr)
        mgr.context.set_option("countStats", 1)
        mgr.OnEnable()
        mgr.context.reset_stats()
        mgr.context.dispatch(capi.RT_KERNEL_RAYTRACE, 3, 3)     # a partial dispatch: untouched pixels (rays == 0) are black
        ctxs.append(mgr)
    po, pg = ctxs[0].pixel_stats(), ctxs[1].pixel_stats()
    assert_pixels_equal(pg, po)
    assert (po["rays"] == 0).any()
    for mode, scales in _scales(po).items():
        for s in scales:
            want = encode_reference(po, mode, s)
            got_o, got_g = ctxs[0].debug_view(mode, s), ctxs[1].debug_view(mode, s)
            assert np.array_equal(got_o, want), (mode, s)
            assert np.array_equal(got_g, want), (mode, s)
    # the threshold itself: the largest box tests / ray at scale = that value is white, one ulp below it is red
    at = _scales(po)[1][0]
    top = (po["rays"] > 0) & (po["boxTests"].astype(np.float32) / np.maximum(po["rays"], 1).astype(np.float32) == np.float32(at))
    assert np.all(ctxs[1].debug_view(1, at)[top] == (255, 255, 255, 255))
    assert np.all(ctxs[1].debug_view(1, _scales(po)[1][1])[top] == (255, 0, 0, 255))
    for m in ctxs:
        m.OnDestroy()


def test_error_codes():
    for lib in (ORACLE_LIB, CUDA_LIB):
        L = capi.RtLib(lib)
        ctx = L.create()
        sc = scenes.cornell_spheres(16, 8, 2, 1)
        buf8 = np.zeros(16 * 8 * 4, dtype=np.uint8)
        stats = np.zeros(16 * 8, dtype=capi.PIXEL_STATS_DTYPE)

        def code(fn):
            try:
                fn()
            except capi.RtError as e:
                return e.code
            return 0
        ctx.resize(16, 8)
        assert ctx._L.rtReadbackPixelStats(ctx.handle, stats.ctypes.data_as(C.c_void_p), stats.nbytes) == capi.RT_E_STATE
        assert ctx._L.rtDisplayPixelStats(ctx.handle, 1, 1.0, buf8.ctypes.data_as(C.c_void_p), buf8.nbytes) == capi.RT_E_STATE
        mgr = rt.RayComputeManager(lib)
        scenes.apply(sc, mgr)
        mgr.context.set_option("countStats", 1)
        mgr.OnEnable()
        m = mgr.context
        assert code(lambda: m.pixel_stats()) == capi.RT_E_STATE      # no counting dispatch yet
        mgr.RenderFrame()
        for mode, scale in ((0, 1.0), (5, 1.0), (-1, 1.0), (1, 0.0), (1, -1.0), (1, float("inf")), (1, float("nan"))):
            assert code(lambda: m.display_pixel_stats(mode, scale)) == capi.RT_E_INVALID, (lib, mode, scale)
        assert m._L.rtDisplayPixelStats(m.handle, 1, 1.0, buf8.ctypes.data_as(C.c_void_p), buf8.nbytes - 4) == capi.RT_E_INVALID
        assert m._L.rtReadbackPixelStats(m.handle, stats.ctypes.data_as(C.c_void_p), stats.nbytes + 20) == capi.RT_E_INVALID
        assert m._L.rtReadbackPixelStats(m.handle, stats.ctypes.data_as(C.c_void_p), stats.nbytes) == 0
        # the uniforms of the reference's debug view stay accepted and change nothing
        m.set_int("visMode", 3); m.set_float("debugVisScale", 2.0); m.set_vector("debugParams", (1, 2, 3, 4))
        mgr.OnDestroy()
        ctx.destroy()
