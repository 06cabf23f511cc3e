"""rtDispatchFrames on the H100 (`-m gpu`): n accumulated frames in one launch equal, bit for bit, n rtDispatch calls with "Frame"
stepped by one — FrameRender, AccumulatedRender, RtStats and PixelStats — and the oracle's images.  The same bodies run in the CPU
suite against the SIMT interpreter build (tests/test_simt_frames.py)."""
import numpy as np
import pytest

from conftest import CUDA_LIB, ORACLE_LIB, assert_bit_equal
import ray_tracing_b200 as rt
from ray_tracing_b200 import capi, scenes

pytestmark = pytest.mark.gpu

COUNTS = ("rays", "boxTests", "triTests", "sphereTests", "sphereBoxTests")


def _open(lib, sc, options=None, tile=None, devices=None, frame=None):
    mgr = rt.RayComputeManager(lib, devices=devices) if devices else rt.RayComputeManager(lib)
    scenes.apply(sc, mgr)
    ctx = mgr.context
    for k, v in (options or {}).items():
        ctx.set_option(k, v)
    if tile:
        ctx.set_tile(*tile)
    mgr.OnEnable()                      # uniforms set, AccumulatedRender zeroed, Frame = 1
    if frame is not None:
        ctx.set_int("Frame", frame)
    ctx.reset_stats()
    return mgr, ctx


def _result(mgr, ctx, counting):
    st = ctx.stats()
    out = dict(frame=mgr.raytraceFrameTex, accum=mgr.accumulatedResult, stats=st,
               pix=mgr.pixel_stats() if counting else None)
    mgr.OnDestroy()
    return out


def render_both(lib, sc, n, options=None, tile=None, groups=None, frame=None, before=0, devices=None):
    """(batch, sequence): rtDispatchFrames(n) and n rtDispatch calls with Frame = F .. F + n - 1 then Frame = F, each on a fresh context
    after `before` single dispatches at Frame = F - before .. F - 1 (an accumulation that is already non-zero)."""
    counting = bool((options or {}).get("countStats"))
    out = []
    for batched in (True, False):
        mgr, ctx = _open(lib, sc, options, tile, devices, frame)
        F = ctx_frame = frame if frame is not None else 1
        g = groups or ((sc.width + 7) // 8, (sc.height + 7) // 8, 1)
        for k in range(before):
            ctx.set_int("Frame", _wrap(F - before + k))
            ctx.dispatch(capi.RT_KERNEL_RAYTRACE, *g)
        ctx.set_int("Frame", F)
        if batched:
            ctx.dispatch_frames(n, *g)
        else:
            for k in range(n):
                ctx.set_int("Frame", _wrap(F + k))
                ctx.dispatch(capi.RT_KERNEL_RAYTRACE, *g)
            ctx.set_int("Frame", ctx_frame)
        out.append(_result(mgr, ctx, counting))
    return out


def _wrap(f):
    """Frame + k modulo 2^32, as the int the uniform holds."""
    f &= 0xffffffff
    return f - (1 << 32) if f >= (1 << 31) else f


def assert_same(b, s, what, stats=True):
    assert_bit_equal(b["frame"], s["frame"], f"{what}: FrameRender")
    assert_bit_equal(b["accum"], s["accum"], f"{what}: AccumulatedRender")
    if stats:
        for k in COUNTS + ("dispatches",):
            assert b["stats"][k] == s["stats"][k], f"{what}: RtStats.{k} {b['stats'][k]} vs {s['stats'][k]}"
    if b["pix"] is not None:
        for k in COUNTS:
            assert np.array_equal(b["pix"][k], s["pix"][k]), f"{what}: PixelStats.{k}"


def check(sc, n, options_list=({},), oracle=True, **kw):
    """For every option set: the batch equals the library's own n dispatches; and (oracle) the images equal the oracle's batch."""
    ref = render_both(ORACLE_LIB, sc, n, **kw)[0] if oracle else None
    for opts in options_list:
        b, s = render_both(CUDA_LIB, sc, n, options=opts, **kw)
        assert_same(b, s, f"{sc.name} n={n} {opts}")
        if ref is not None:
            assert_bit_equal(b["accum"], ref["accum"], f"{sc.name} n={n} {opts}: AccumulatedRender vs the oracle")
            assert_bit_equal(b["frame"], ref["frame"], f"{sc.name} n={n} {opts}: FrameRender vs the oracle")
    return ref


@pytest.mark.parametrize("kernel", [-1, 0, 1, 2])
def test_batch_equals_dispatches_per_kernel(kernel):
    check(scenes.cornell_spheres(24, 16, 3, 2), 3, ({"kernel": kernel},))
    check(scenes.knot_room(24, 16, 3, 2, nu=30, nv=6), 4, ({"kernel": kernel},))


def test_pool_sizes_and_tail_lanes():
    sc = scenes.knot_room(32, 16, max_bounces=5, rays_per_pixel=2, nu=40, nv=8, glass=True)
    check(sc, 3, tuple({"kernel": 2, "poolSlots": s, "tailLanes": t} for s in (32, 64, 96) for t in (0, 31)))


@pytest.mark.parametrize("kernel", [1, 2])
def test_extension_instantiation_sphere_accelerator_and_tlas(kernel):
    check(scenes.knot_room(24, 16, 3, 2, nu=30, nv=6), 3, ({"kernel": kernel, "extInstantiation": 1}, {"kernel": kernel, "tlas": 1}))
    check(scenes.random_soup(24, 16, max_bounces=3, rays_per_pixel=2, triangles=600, spheres=80), 3, ({"kernel": kernel},))


@pytest.mark.parametrize("kernel", [0, 1, 2])
def test_count_stats_and_pixel_stats_equal_the_dispatches(kernel):
    check(scenes.knot_room(24, 16, 3, 2, nu=30, nv=6), 3, ({"kernel": kernel, "countStats": 1},))
    check(scenes.random_soup(24, 16, max_bounces=3, rays_per_pixel=1, triangles=600, spheres=80), 2, ({"kernel": kernel, "countStats": 1},), oracle=False)


def test_glass_sky_and_defocus():
    sc = scenes.knot_room(24, 16, max_bounces=6, rays_per_pixel=2, nu=30, nv=6, glass=True)
    sc.settings.update(useSky=True, defocusStrength=40.0)
    check(sc, 3, ({"kernel": 0}, {"kernel": 1}, {"kernel": 2}))


@pytest.mark.parametrize("spp", [0, 1, 3])
def test_samples_per_pixel_and_a_non_zero_accumulation(spp):
    sc = scenes.knot_room(24, 16, 3, spp, nu=30, nv=6)
    check(sc, 3, ({}, {"kernel": 1}, {"kernel": 2}), before=2, frame=5)


def test_partial_dispatch_and_row_band_ranks():
    sc = scenes.knot_room(40, 24, 3, 2, nu=30, nv=6)
    check(sc, 3, ({"kernel": 1}, {"kernel": 2}), groups=(3, 2, 1))
    check(sc, 3, ({"kernel": 0}, {"kernel": 1}, {"kernel": 2}), oracle=False, groups=(5, 3, 0))
    for r in range(3):
        check(sc, 3, ({"kernel": 1}, {"kernel": 2}), tile=(r, 3, 8))


def test_group_context():
    try:
        capi.RtLib(CUDA_LIB).create_multi([0, 1]).destroy()
    except capi.RtError:
        pytest.skip("a group context needs two or more devices")
    sc = scenes.knot_room(40, 24, 3, 2, nu=30, nv=6)
    b, s = render_both(CUDA_LIB, sc, 3, devices=[0, 1])
    assert_same(b, s, "group of two")
    single = render_both(ORACLE_LIB, sc, 3)[0]
    assert_bit_equal(b["accum"], single["accum"], "group of two vs the oracle")


def test_frame_wraps_modulo_2_32():
    sc = scenes.cornell_spheres(16, 8, 3, 1)
    for kernel in (0, 1, 2):
        check(sc, 4, ({"kernel": kernel},), frame=2**31 - 2)
        check(sc, 3, ({"kernel": kernel},), frame=-1)


def test_one_frame_is_a_dispatch():
    sc = scenes.knot_room(24, 16, 3, 2, nu=30, nv=6)
    for opts in ({"kernel": 0}, {"kernel": 1}, {"kernel": 2, "countStats": 1}):
        b, s = render_both(CUDA_LIB, sc, 1, options=opts)
        assert_same(b, s, f"n = 1 {opts}")


def test_error_codes_and_the_frame_bound():
    sc = scenes.knot_room(16, 8, 3, 3, nu=30, nv=6)
    for lib in (CUDA_LIB, ORACLE_LIB):
        mgr, ctx = _open(lib, sc)
        for n in (0, -1, capi.RT_MAX_BATCH_SAMPLES // 3 + 1):
            with pytest.raises(capi.RtError) as e:
                ctx.dispatch_frames(n)
            assert e.value.code == capi.RT_E_INVALID, (lib, n)
        if lib == CUDA_LIB:                                             # (the oracle would loop over a million empty dispatches)
            ctx.dispatch_frames(capi.RT_MAX_BATCH_SAMPLES // 3, 2, 1, 0)  # inside the bound (gz = 0: nothing is traced)
        ctx.set_int("NumRaysPerPixel", 0)                               # the bound counts max(1, NumRaysPerPixel) samples per frame
        if lib == CUDA_LIB:
            ctx.dispatch_frames(capi.RT_MAX_BATCH_SAMPLES, 2, 1, 0)
        with pytest.raises(capi.RtError) as e:
            ctx.dispatch_frames(capi.RT_MAX_BATCH_SAMPLES + 1, 2, 1, 0)
        assert e.value.code == capi.RT_E_INVALID
        ctx.set_int("NumRaysPerPixel", 3)
        with pytest.raises(capi.RtError) as e:
            ctx.dispatch_frames(2, -1, 1, 1)
        assert e.value.code == capi.RT_E_INVALID
        ctx.set_bool("accumulate", False)
        for n in (1, 2):
            with pytest.raises(capi.RtError) as e:
                ctx.dispatch_frames(n)
            assert e.value.code == capi.RT_E_STATE, (lib, n)
        ctx.set_bool("accumulate", True)
        if lib == CUDA_LIB:                                             # the oracle has no sample chunks
            ctx.set_option("sampleChunks", 2)
            with pytest.raises(capi.RtError) as e:
                ctx.dispatch_frames(2)
            assert e.value.code == capi.RT_E_STATE
            ctx.dispatch_frames(1)                                      # n = 1 is a dispatch, chunks and all
            ctx.set_option("sampleChunks", 1)
            ctx.dispatch_frames(2)
        assert ctx.stats()["dispatches"] == (3 if lib == CUDA_LIB else 0)
        mgr.OnDestroy()


@pytest.mark.parametrize("accumulate", [True, False])
def test_manager_render_frames_equals_render_frame(accumulate):
    """RayComputeManager.RenderFrames(n) (Python, through the C++ manager's rcmRenderFrames) against n RenderFrame() calls."""
    sc = scenes.knot_room(24, 16, 3, 2, nu=30, nv=6)
    sc.settings["accumulate"] = accumulate
    out = []
    for batched in (True, False):
        mgr = rt.RayComputeManager(CUDA_LIB)
        scenes.apply(sc, mgr)
        mgr.OnEnable()
        mgr.RenderFrame()
        if batched:
            mgr.RenderFrames(4)
        else:
            for _ in range(4):
                mgr.RenderFrame()
        out.append((mgr.raytraceFrameTex, mgr.accumulatedResult, mgr.numAccumulatedFrames, mgr.context.stats()["dispatches"]))
        with pytest.raises(capi.RtError):
            mgr.RenderFrames(0)
        mgr.OnDestroy()
    (fb, ab, nb, db), (fs, as_, ns, ds) = out
    assert_bit_equal(fb, fs, "RenderFrames FrameRender")
    assert_bit_equal(ab, as_, "RenderFrames AccumulatedRender")
    assert nb == ns == (6 if accumulate else 1) and db == ds


def test_1080p_knot_batch_of_16():
    """The knot scene at 1080p, 1 spp: one batch of 16 frames equals 16 dispatches bitwise (automatic kernel choice)."""
    sc = scenes.knot_room(1920, 1080, 8, 1)
    b, s = render_both(CUDA_LIB, sc, 16)
    assert_same(b, s, "1080p knot, 16 frames")
