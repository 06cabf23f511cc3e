"""rtDispatchAdaptive and rtDisplayMean on the H100 (`-m gpu`): sessions of adaptive frames compared bit for bit with the oracle —
FrameRender, AccumulatedRender, AdaptiveMoments, the active counts, RtStats and PixelStats — and with the library's own rtDispatch;
the edges of the pixel list, the lifetime of the moments and every refusal.  The same bodies run in the CPU suite against the SIMT
interpreter build (tests/test_simt_adaptive.py)."""
import ctypes as C

import numpy as np
import pytest

from conftest import CUDA_LIB, ORACLE_LIB, assert_bit_equal
import ray_tracing_b200 as rt
from ray_tracing_b200 import capi, scenes

pytestmark = pytest.mark.gpu

COUNTS = ("rays", "boxTests", "triTests", "sphereTests", "sphereBoxTests")
EPS = np.float32(0.00390625)          # RT_ADAPTIVE_EPSILON

# a session: (threshold, minFrames, maxFrames) per call; the threshold changes midway
SESSION = [(0.3, 2, 8)] * 6 + [(0.05, 3, 8)] * 6


def _open(lib, sc, options=None, tile=None):
    mgr = rt.RayComputeManager(lib)
    scenes.apply(sc, mgr)
    ctx = mgr.context
    for k, v in (options or {}).items():
        ctx.set_option(k, v)
    if tile:
        ctx.set_tile(*tile)
    mgr.OnEnable()                      # uniforms set, AccumulatedRender zeroed, Frame = 1
    ctx.reset_stats()
    return mgr, ctx


def _groups(sc):
    return (sc.width + 7) // 8, (sc.height + 7) // 8, 1


def run_session(lib, sc, session=SESSION, options=None, tile=None, groups=None, first_frame=1):
    """The session's calls with "Frame" = first_frame, first_frame + 1, ...; returns the images, moments, counts and counters."""
    mgr, ctx = _open(lib, sc, options, tile)
    g = groups or _groups(sc)
    counts = []
    for k, (thr, mn, mx) in enumerate(session):
        ctx.set_int("Frame", first_frame + k)
        counts.append(ctx.dispatch_adaptive(thr, mn, mx, *g))
    out = dict(counts=counts, frame=mgr.raytraceFrameTex, accum=mgr.accumulatedResult, stats=ctx.stats(),
               moments=ctx.adaptive_moments() if any(counts) else None,
               pix=mgr.pixel_stats() if (options or {}).get("countStats") else None)
    mgr.OnDestroy()
    return out


def assert_same(a, b, what, fields=COUNTS):
    assert a["counts"] == b["counts"], f"{what}: active counts {a['counts']} vs {b['counts']}"
    assert_bit_equal(a["frame"], b["frame"], f"{what}: FrameRender")
    assert_bit_equal(a["accum"], b["accum"], f"{what}: AccumulatedRender")
    if a["moments"] is not None or b["moments"] is not None:
        assert_bit_equal(a["moments"], b["moments"], f"{what}: AdaptiveMoments")
    for k in ("rays", "dispatches"):
        assert a["stats"][k] == b["stats"][k], f"{what}: RtStats.{k} {a['stats'][k]} vs {b['stats'][k]}"
    if a["pix"] is not None and b["pix"] is not None:
        for k in fields:
            assert np.array_equal(a["pix"][k], b["pix"][k]), f"{what}: PixelStats.{k}"
            assert a["stats"][k] == b["stats"][k], f"{what}: RtStats.{k}"


def check_oracle(sc, options_list=({},), session=SESSION, fields=COUNTS, **kw):
    ref = run_session(ORACLE_LIB, sc, session, **kw)
    assert sum(ref["counts"]) > 0
    for opts in options_list:
        counting = dict(opts, countStats=1) if opts.get("countStats") else opts
        got = run_session(CUDA_LIB, sc, session, options=counting, **kw)
        r = ref if not counting.get("countStats") else run_session(ORACLE_LIB, sc, session, options={"countStats": 1}, **kw)
        assert_same(got, r, f"{sc.name} {opts}", fields)
    return ref


# ---- against the oracle ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kernel", [0, 1, 2])
def test_cornell_spheres_against_the_oracle(kernel):
    check_oracle(scenes.cornell_spheres(24, 16, 4, 1), ({"kernel": kernel}, {"kernel": kernel, "countStats": 1}))


@pytest.mark.parametrize("kernel", [0, 1, 2])
def test_glass_knot_room_against_the_oracle(kernel):
    sc = scenes.knot_room(24, 16, 6, 1, nu=40, nv=8, glass=True)
    check_oracle(sc, ({"kernel": kernel, "modelSkip": 0}, {"kernel": kernel, "modelSkip": 1}, {"kernel": kernel, "countStats": 1}))


def test_three_rays_per_pixel_and_pool_sizes_against_the_oracle():
    sc = scenes.knot_room(24, 16, 5, 3, nu=40, nv=8, glass=True)
    check_oracle(sc, ({"kernel": 0}, {"kernel": 1}, {"kernel": 2, "poolSlots": 32}, {"kernel": 2, "poolSlots": 96},
                      {"kernel": 2, "poolSlots": 32, "countStats": 1}))


def test_checker_soup_against_the_oracle():
    check_oracle(scenes.random_soup(24, 16, 4, 1, triangles=400, spheres=40), ({"kernel": 1}, {"kernel": 2}, {"kernel": 2, "countStats": 1}))


@pytest.mark.parametrize("tlas", [-1, 0, 1])
def test_152_instanced_knots_with_the_tlas_against_the_oracle(tlas):
    check_oracle(scenes.instanced_knots(24, 16, 4, 1, instances=150), ({"kernel": 1, "tlas": tlas}, {"kernel": 2, "tlas": tlas}))


def test_10000_spheres_sphere_accelerator_against_the_oracle():
    # the accelerator's sphere counters differ from the oracle's linear scan by design (tests/test_gpu_pixel_stats.py)
    check_oracle(scenes.random_soup(24, 16, 4, 1, triangles=300, spheres=10000),
                 ({"kernel": 1}, {"kernel": 2}, {"kernel": 2, "countStats": 1}), fields=("rays", "boxTests", "triTests"))


def test_unity_fixture_against_the_oracle():
    from test_round2_abi import load_fixture
    check_oracle(load_fixture(24, 16), ({"kernel": 0}, {"kernel": 1}, {"kernel": 2}))


def test_nan_pixels_against_the_oracle():
    """A NaN sun with the sky on (tests/test_gpu_parity.py): NaN frames make NaN moments, and those pixels drop out after minFrames."""
    sc = scenes.random_soup(24, 16, max_bounces=3, rays_per_pixel=1, triangles=600, spheres=8)
    sc.settings["sunIntensity"] = float("nan")
    ref = check_oracle(sc, ({"kernel": 0}, {"kernel": 1}, {"kernel": 2}))
    nan = np.isnan(ref["moments"][..., 0])
    assert nan.any()
    assert np.all(ref["moments"][..., 2][nan] <= 3.0)          # never traced again once minFrames (2, then 3) is reached


# ---- against rtDispatch itself -----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kernel", [0, 1, 2])
def test_threshold_zero_equals_plain_dispatches(kernel):
    """threshold 0 and minFrames = maxFrames = k: k calls equal k rtDispatch calls in every image and counter; then nothing is active."""
    sc = scenes.knot_room(24, 16, 4, 2, nu=30, nv=6)
    k = 3
    for opts in ({"kernel": kernel}, {"kernel": kernel, "countStats": 1}):
        a = run_session(CUDA_LIB, sc, [(0.0, k, k)] * (k + 1), options=opts)
        assert a["counts"] == [sc.width * sc.height] * k + [0]
        mgr, ctx = _open(CUDA_LIB, sc, opts)
        for f in range(1, k + 1):
            ctx.set_int("Frame", f)
            ctx.dispatch(capi.RT_KERNEL_RAYTRACE, *_groups(sc))
        b = dict(frame=mgr.raytraceFrameTex, accum=mgr.accumulatedResult, stats=ctx.stats(), pix=mgr.pixel_stats() if opts.get("countStats") else None)
        mgr.OnDestroy()
        assert_bit_equal(a["frame"], b["frame"], f"{opts}: FrameRender")
        assert_bit_equal(a["accum"], b["accum"], f"{opts}: AccumulatedRender")
        for key in COUNTS + ("dispatches",):
            assert a["stats"][key] == b["stats"][key], f"{opts}: RtStats.{key}"
        if b["pix"] is not None:
            for key in COUNTS:
                assert np.array_equal(a["pix"][key], b["pix"][key]), f"{opts}: PixelStats.{key}"


def criterion(m, threshold, min_frames, max_frames):
    """The header's selection, restated in numpy binary32 (NaN-ignoring max)."""
    m = m.astype(np.float32)
    with np.errstate(all="ignore"):
        n = m[..., 2]
        mu = m[..., 0] / n
        v = np.fmax(m[..., 1] / n - mu * mu, np.float32(0))
        t = np.float32(threshold)
        return (n < np.float32(min_frames)) | ((n < np.float32(max_frames)) & (v > ((t * t) * n) * (mu * mu + EPS)))


@pytest.mark.parametrize("kernel", [1, 2])
def test_active_set_is_the_criterion_and_equals_a_plain_dispatch(kernel):
    """Before every call the numpy criterion on the moments names the active set; those pixels' FrameRender equals an rtDispatch at
    the same Frame on a second context, and every other pixel is byte-unchanged in both images and the moments."""
    sc = scenes.knot_room(24, 16, 5, 1, nu=40, nv=8, glass=True)
    mgr, ctx = _open(CUDA_LIB, sc, {"kernel": kernel})
    mgr2, ctx2 = _open(CUDA_LIB, sc, {"kernel": kernel})
    mom = np.zeros((sc.height, sc.width, 4), np.float32)
    for k, (thr, mn, mx) in enumerate([(0.4, 2, 6)] * 8):
        f0, a0 = mgr.raytraceFrameTex, mgr.accumulatedResult
        want = criterion(mom, thr, mn, mx)
        ctx.set_int("Frame", 1 + k)
        n = ctx.dispatch_adaptive(thr, mn, mx)
        assert n == int(want.sum()), f"call {k}"
        f1, a1, m1 = mgr.raytraceFrameTex, mgr.accumulatedResult, ctx.adaptive_moments()
        ctx2.set_int("Frame", 1 + k)
        ctx2.dispatch(capi.RT_KERNEL_RAYTRACE, *_groups(sc))
        plain = mgr2.raytraceFrameTex
        assert_bit_equal(f1[want], plain[want], f"call {k}: active pixels vs rtDispatch")
        for before, after, name in ((f0, f1, "FrameRender"), (a0, a1, "AccumulatedRender"), (mom, m1, "AdaptiveMoments")):
            assert np.array_equal(before[~want].view(np.uint32), after[~want].view(np.uint32)), f"call {k}: inactive {name}"
        l = (np.float32(0.2126) * f1[..., 0] + np.float32(0.7152) * f1[..., 1]) + np.float32(0.0722) * f1[..., 2]
        exp = mom.copy()
        exp[..., 0] = np.where(want, mom[..., 0] + l, mom[..., 0])
        exp[..., 1] = np.where(want, mom[..., 1] + l * l, mom[..., 1])
        exp[..., 2] = np.where(want, mom[..., 2] + np.float32(1), mom[..., 2])
        assert_bit_equal(m1, exp, f"call {k}: moments update")
        mom = m1
    mgr.OnDestroy(); mgr2.OnDestroy()


# ---- edges of the list -------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("k", [0, 1, 31, 32, 33, 65])
@pytest.mark.parametrize("kernel", [0, 1, 2])
def test_exactly_k_pixels_stay_active(k, kernel):
    """Image (8 + k) x 1: the first 8x8 group's region reaches maxFrames in two partial calls, then exactly the k pixels right of it are
    active (twice), then none."""
    sc = scenes.cornell_spheres(8 + k, 1, 3, 1)
    session = [(0.0, 2, 2)] * 5
    groups = [(1, 1, 1), (1, 1, 1), None, None, None]

    def run(lib, opts):
        mgr, ctx = _open(lib, sc, opts)
        counts = []
        for i, ((thr, mn, mx), g) in enumerate(zip(session, groups)):
            ctx.set_int("Frame", 1 + i)
            counts.append(ctx.dispatch_adaptive(thr, mn, mx, *(g or _groups(sc))))
        out = dict(counts=counts, frame=mgr.raytraceFrameTex, accum=mgr.accumulatedResult, moments=ctx.adaptive_moments(),
                   stats=ctx.stats(), pix=None)
        mgr.OnDestroy()
        return out
    ref = run(ORACLE_LIB, {})
    assert ref["counts"] == [8, 8, k, k, 0]
    assert_same(run(CUDA_LIB, {"kernel": kernel}), ref, f"k={k} kernel={kernel}")


@pytest.mark.parametrize("size", [(1, 1), (70, 41), (56, 4), (64, 4), (72, 4), (255, 1), (256, 1), (257, 1)])
def test_image_sizes_around_the_selection_block(size):
    """1x1, 70x41, and covered pixels / jobs on either side of the selection's 256-job block (7, 8 and 9 tiles; 255 .. 257 pixels)."""
    sc = scenes.cornell_spheres(size[0], size[1], 3, 1)
    session = [(0.3, 2, 4)] * 5
    ref = run_session(ORACLE_LIB, sc, session)
    for kernel in (0, 1, 2):
        assert_same(run_session(CUDA_LIB, sc, session, options={"kernel": kernel}), ref, f"{size} kernel={kernel}")


def test_selection_over_more_than_1024_blocks():
    """600 x 500 (1172 selection blocks: the scan runs in two chunks) with NumRaysPerPixel = 0: every frame is NaN (0 / 0, as in
    rtDispatch), so the pixels drop out after minFrames and the selection itself is what is exercised."""
    sc = scenes.cornell_spheres(600, 500, 1, 0)
    session = [(0.1, 2, 4)] * 3
    ref = run_session(ORACLE_LIB, sc, session)
    assert ref["counts"] == [300000, 300000, 0]
    assert_same(run_session(CUDA_LIB, sc, session), ref, "600x500")


def _cluster_session(lib, sc, tile=None):
    """Two whole-image calls, then one over the lower-left 960 x 560 (several hundred thousand active pixels)."""
    mgr, ctx = _open(lib, sc, tile=tile)
    counts = []
    for f, (mn, mx, g) in enumerate(((2, 2, (480, 270)), (2, 3, (480, 270)), (3, 3, (120, 70))), start=1):
        ctx.set_int("Frame", f)
        counts.append(ctx.dispatch_adaptive(0.0, mn, mx, g[0], g[1], 1))
    out = dict(counts=counts, frame=mgr.raytraceFrameTex, accum=mgr.accumulatedResult, moments=ctx.adaptive_moments())
    mgr.OnDestroy()
    return out


def test_4k_knot_cluster_against_ten_oracle_rows():
    """3840 x 2160 against the oracle on ten seeded rows: bands of one row with the row as the rank make the oracle trace that row
    alone (as the features test does)."""
    sc = scenes.knot_cluster(3840, 2160, 4, 1)
    got = _cluster_session(CUDA_LIB, sc)
    assert got["counts"] == [3840 * 2160, 3840 * 2160, 960 * 560]
    ys = np.sort(np.concatenate([np.random.RandomState(23).choice(560, 6, replace=False),
                                 560 + np.random.RandomState(24).choice(2160 - 560, 4, replace=False)]))
    for y in ys:
        ref = _cluster_session(ORACLE_LIB, sc, tile=(int(y), 2160, 1))
        assert ref["counts"] == [3840, 3840, 960 if y < 560 else 0]
        for k in ("frame", "accum", "moments"):
            assert_bit_equal(got[k][y], ref[k][y], f"4K cluster row {y}: {k}")


# ---- lifetime, state and refusals ----------------------------------------------------------------------------------------------

def _snapshot(mgr, ctx):
    st = ctx.stats()
    try:
        mom = ctx.adaptive_moments()
    except capi.RtError:
        mom = None
    return dict(frame=mgr.raytraceFrameTex, accum=mgr.accumulatedResult, moments=mom, stats={k: st[k] for k in COUNTS + ("dispatches",)})


def _assert_unchanged(a, b, what):
    assert_bit_equal(a["frame"], b["frame"], f"{what}: FrameRender")
    assert_bit_equal(a["accum"], b["accum"], f"{what}: AccumulatedRender")
    assert (a["moments"] is None) == (b["moments"] is None), f"{what}: moments allocated"
    if a["moments"] is not None:
        assert_bit_equal(a["moments"], b["moments"], f"{what}: AdaptiveMoments")
    assert a["stats"] == b["stats"], f"{what}: RtStats"


def test_partial_dispatch_and_row_bands_against_the_oracle():
    sc = scenes.knot_room(40, 30, 4, 1, nu=30, nv=6)
    for tile in (None, (0, 3, 2), (1, 3, 2), (2, 3, 8)):
        for groups in ((3, 2, 1), (5, 4, 1), (0, 4, 1), (5, 4, 0)):
            ref = run_session(ORACLE_LIB, sc, [(0.3, 2, 4)] * 4, tile=tile, groups=groups)
            for kernel in (0, 1, 2):
                assert_same(run_session(CUDA_LIB, sc, [(0.3, 2, 4)] * 4, options={"kernel": kernel}, tile=tile, groups=groups), ref,
                            f"tile={tile} groups={groups} kernel={kernel}")


def _lifetime(lib):
    sc = scenes.cornell_spheres(24, 16, 3, 1)
    mgr, ctx = _open(lib, sc)
    out = {}
    with pytest.raises(capi.RtError) as e:
        ctx.adaptive_moments()
    out["before"] = e.value.code
    for f in (1, 2, 3):
        ctx.set_int("Frame", f)
        ctx.dispatch_adaptive(0.0, 3, 3)
    m0 = ctx.adaptive_moments()
    ctx.set_int("Frame", 4)
    ctx.dispatch(capi.RT_KERNEL_RAYTRACE, 3, 2, 1)                     # plain dispatches leave the moments alone
    ctx.dispatch_frames(2)
    out["plain"] = np.array_equal(ctx.adaptive_moments().view(np.uint32), m0.view(np.uint32))
    ctx.reset_stats()
    out["reset_stats"] = np.array_equal(ctx.adaptive_moments().view(np.uint32), m0.view(np.uint32))
    ctx.dispatch(capi.RT_KERNEL_RESET_ACCUMULATED, 2, 1, 1)              # zeroes the 16 x 8 region of the moments too
    out["after_reset"] = ctx.adaptive_moments()
    ctx.set_int("Frame", 6)
    out["count_after_reset"] = ctx.dispatch_adaptive(0.0, 3, 3)         # only the zeroed region is below maxFrames
    out["accum"] = mgr.accumulatedResult
    ctx.resize(16, 8)
    ctx.set_ints("Resolution", [16, 8])
    out["resized"] = ctx.adaptive_moments()
    mgr.OnDestroy()
    return out, m0


def test_moments_lifetime_against_the_oracle():
    got, m0 = _lifetime(CUDA_LIB)
    ref, r0 = _lifetime(ORACLE_LIB)
    assert got["before"] == ref["before"] == capi.RT_E_STATE
    assert got["plain"] and got["reset_stats"] and ref["plain"] and ref["reset_stats"]
    assert_bit_equal(m0, r0, "moments")
    assert np.all(got["after_reset"][:8, :16] == 0) and np.all(got["after_reset"][8:, :] == m0[8:, :])
    assert_bit_equal(got["after_reset"], ref["after_reset"], "after ResetAccumulated")
    assert got["count_after_reset"] == ref["count_after_reset"] == 16 * 8
    assert_bit_equal(got["accum"], ref["accum"], "AccumulatedRender")
    assert got["resized"].shape == (8, 16, 4) and not np.any(got["resized"])
    assert_bit_equal(got["resized"], ref["resized"], "after resize")


def test_device_pointer_before_and_after_the_first_call():
    sc = scenes.cornell_spheres(24, 16, 3, 1)
    mgr, ctx = _open(CUDA_LIB, sc)
    L = ctx._L
    p, n = C.c_void_p(), C.c_size_t()
    assert L.rtGetDevicePointer(ctx._h, b"AdaptiveMoments", C.byref(p), C.byref(n)) == capi.RT_E_STATE
    ctx.dispatch_adaptive()
    assert L.rtGetDevicePointer(ctx._h, b"AdaptiveMoments", C.byref(p), C.byref(n)) == capi.RT_OK
    assert p.value and n.value == 24 * 16 * 16
    mgr.OnDestroy()


def test_refusals_change_nothing():
    sc = scenes.cornell_spheres(24, 16, 3, 1)
    mgr, ctx = _open(CUDA_LIB, sc)
    L, h = ctx._L, ctx._h
    act = C.c_int64(-7)

    def call(*a):
        return L.rtDispatchAdaptive(h, *a, C.byref(act))
    assert L.rtDispatchAdaptive(None, 3, 2, 1, 0.1, 2, 4, C.byref(act)) == capi.RT_E_INVALID
    ctx.set_int("Frame", 1)
    ctx.dispatch_adaptive(0.3, 2, 6)
    ctx.set_int("Frame", 2)
    before = _snapshot(mgr, ctx)
    inf, nan = float("inf"), float("nan")
    for args in ((-1, 2, 1, 0.1, 2, 4), (3, -1, 1, 0.1, 2, 4), (3, 2, -1, 0.1, 2, 4), (3, 2, 1, nan, 2, 4), (3, 2, 1, inf, 2, 4),
                 (3, 2, 1, -0.5, 2, 4), (3, 2, 1, 2e19, 2, 4), (3, 2, 1, 0.1, 1, 4), (3, 2, 1, 0.1, -3, 4), (3, 2, 1, 0.1, 5, 4),
                 (3, 2, 1, 0.1, 2, (1 << 24) + 1)):
        assert call(*args) == capi.RT_E_INVALID, args
        _assert_unchanged(before, _snapshot(mgr, ctx), f"refused {args}")
    assert act.value == -7
    # state refusals
    ctx.set_bool("accumulate", 0)
    assert call(3, 2, 1, 0.1, 2, 4) == capi.RT_E_STATE
    ctx.set_bool("accumulate", 1)
    ctx.set_option("sampleChunks", 2)
    assert call(3, 2, 1, 0.1, 2, 4) == capi.RT_E_STATE
    ctx.set_option("sampleChunks", -1)
    ctx.set_int("MaxBounceCount", 201)
    assert call(3, 2, 1, 0.1, 2, 4) == capi.RT_E_STATE
    ctx.set_int("MaxBounceCount", 3)
    ctx.set_ints("Resolution", [25, 16])
    assert call(3, 2, 1, 0.1, 2, 4) == capi.RT_E_STATE
    ctx.set_ints("Resolution", [24, 16])
    ctx.set_int("modelCount", 5)
    assert call(3, 2, 1, 0.1, 2, 4) == capi.RT_E_STATE
    ctx.set_int("modelCount", 0)
    _assert_unchanged(before, _snapshot(mgr, ctx), "state refusals")
    assert act.value == -7
    # the maximum is accepted
    assert call(3, 2, 1, 0.1, 2, 1 << 24) == capi.RT_OK
    mgr.OnDestroy()
    # before rtResize
    lib = capi.RtLib(CUDA_LIB)
    c2 = lib.create()
    assert lib.lib.rtDispatchAdaptive(c2._h, 1, 1, 1, C.c_float(0.1), 2, 4, None) == capi.RT_E_STATE
    c2.destroy()


def test_group_context_is_refused():
    lib = capi.RtLib(CUDA_LIB)
    h = C.c_void_p()
    devs = (C.c_int * 2)(0, 1)
    if lib.lib.rtCreateMulti(C.byref(h), devs, 2) != capi.RT_OK:
        pytest.skip("no two-device group here")
    lib.lib.rtResize(h, 16, 8)
    lib.lib.rtSetInts(h, b"Resolution", (C.c_int * 2)(16, 8), 2)
    assert lib.lib.rtDispatchAdaptive(h, 2, 1, 1, C.c_float(0.1), 2, 4, None) == capi.RT_E_STATE
    lib.lib.rtDestroy(h)


def _display_case(lib):
    sc = scenes.knot_room(24, 16, 4, 1, nu=30, nv=6)
    mgr, ctx = _open(lib, sc)
    out = {"empty": ctx.display_mean()}
    for f in range(1, 7):
        ctx.set_int("Frame", f)
        ctx.dispatch_adaptive(0.4, 2, 5, 2, 2, 1)                       # a partial region: the rest stays at A.w = 0
    out["mean"] = ctx.display_mean()
    out["accum"] = mgr.accumulatedResult
    mgr.OnDestroy()
    mgr, ctx = _open(lib, sc)
    for f in range(1, 4):
        ctx.set_int("Frame", f)
        ctx.dispatch_adaptive(0.0, 3, 3)
    out["uniform_mean"], out["uniform_display"] = ctx.display_mean(), ctx.display(True, 3)
    mgr.OnDestroy()
    return out


def test_display_mean():
    got, ref = _display_case(CUDA_LIB), _display_case(ORACLE_LIB)
    assert np.all(got["empty"] == np.array([0, 0, 0, 255], np.uint8))
    for k in ("mean", "uniform_mean"):
        assert np.array_equal(got[k], ref[k]), k
    w = got["accum"][..., 3]
    assert np.all(got["mean"][w == 0] == np.array([0, 0, 0, 255], np.uint8))
    assert np.all(got["mean"][w > 0][..., 3] == 255)
    assert np.array_equal(got["uniform_mean"], got["uniform_display"])


def test_display_mean_refusals():
    sc = scenes.cornell_spheres(24, 16, 3, 1)
    mgr, ctx = _open(CUDA_LIB, sc)
    buf = np.empty(24 * 16 * 4 - 1, np.uint8)
    assert ctx._L.rtDisplayMean(ctx._h, buf.ctypes.data_as(C.c_void_p), buf.nbytes) == capi.RT_E_INVALID
    assert ctx._L.rtDisplayMean(ctx._h, None, 24 * 16 * 4) == capi.RT_E_INVALID
    mgr.OnDestroy()


def _manager_run(lib):
    sc = scenes.knot_room(24, 16, 4, 1, nu=30, nv=6)
    mgr = rt.RayComputeManager(lib)
    scenes.apply(sc, mgr)
    mgr.OnEnable()
    counts = [mgr.RenderFrameAdaptive(0.3, 2, 5) for _ in range(7)]
    out = dict(counts=counts, accum=mgr.accumulatedResult, frames=mgr.numAccumulatedFrames, mean=mgr.mean_result, shown=mgr.display_mean())
    mgr.OnDestroy()
    return out


def test_managers_against_the_oracle():
    got, ref = _manager_run(CUDA_LIB), _manager_run(ORACLE_LIB)
    assert got["counts"] == ref["counts"] and got["counts"][0] == 24 * 16 and got["counts"][-1] == 0
    assert got["frames"] == ref["frames"] == 1 + 7
    assert_bit_equal(got["accum"], ref["accum"], "manager AccumulatedRender")
    assert_bit_equal(got["mean"], ref["mean"], "mean_result")
    assert np.array_equal(got["shown"], ref["shown"])


def test_stream_order_on_a_caller_stream():
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device for torch")
    sc = scenes.knot_room(24, 16, 4, 1, nu=30, nv=6)
    ref = run_session(CUDA_LIB, sc, [(0.3, 2, 4)] * 4)
    mgr, ctx = _open(CUDA_LIB, sc)
    s = torch.cuda.Stream()
    ctx.set_stream(s.cuda_stream)
    counts = []
    for k in range(4):
        ctx.set_int("Frame", 1 + k)
        counts.append(ctx.dispatch_adaptive(0.3, 2, 4))
    s.synchronize()
    assert counts == ref["counts"]
    assert_bit_equal(mgr.accumulatedResult, ref["accum"], "caller stream")
    assert_bit_equal(ctx.adaptive_moments(), ref["moments"], "caller stream moments")
    ctx.set_stream(0)
    mgr.OnDestroy()


# ---- randomised search -------------------------------------------------------------------------------------------------------

def test_randomised_adaptive_sessions():
    import os
    import subprocess
    import sys
    import conftest
    tool = os.path.join(conftest.REPO, "tools", "simt_fuzz_session.py")
    r = subprocess.run([sys.executable, tool, "--adaptive", "--lib", CUDA_LIB, "--cases", "12", "--seed", "31", "--steps", "6"],
                       capture_output=True, text=True, timeout=3000)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    last = r.stdout.strip().splitlines()[-1]
    assert "0 findings" in last and "adaptive steps equal: 0" not in last, last
