"""The named per-pixel images of the C ABI on the H100 (`-m gpu`), across all of them at once: the return codes of rtReadback and
rtGetDevicePointer before rtResize, before each image's producer and after it (with the byte counts); which images
RT_KERNEL_RESET_ACCUMULATED, rtResize and rtResetStats zero and which they leave alone; and the codes through a group's leader.  The
same bodies run in the CPU suite against the SIMT interpreter build (tests/test_simt_named_images.py)."""
import ctypes as C

import numpy as np
import pytest

from conftest import CUDA_LIB
import ray_tracing_b200 as rt
from ray_tracing_b200 import capi, scenes

pytestmark = pytest.mark.gpu

FRAME = (20, 12)
OK, STATE, UNKNOWN, INVALID = capi.RT_OK, capi.RT_E_STATE, capi.RT_E_UNKNOWN_NAME, capi.RT_E_INVALID

# bytes per pixel of the W x H images; TileSend / TileRecv are sized by the tile pattern instead
ELEMENT = {"FrameRender": 16, "AccumulatedRender": 16, "PixelStats": 20, "FeatureFrame": 32, "AccumulatedAlbedo": 16,
           "AccumulatedNormal": 16, "DenoisedRender": 16, "TemporalFrame": 16, "AdaptiveMoments": 16}
NAMES = tuple(ELEMENT) + ("TileSend", "TileRecv", "NoSuchImage")
READ_BACK = tuple(n for n in ELEMENT if n != "PixelStats")          # rtReadback serves these; PixelStats has rtReadbackPixelStats
FEATURES = ("FeatureFrame", "AccumulatedAlbedo", "AccumulatedNormal")
RESET_BY_RESET_ACCUMULATED = ("AccumulatedRender", "AccumulatedAlbedo", "AccumulatedNormal", "AdaptiveMoments")

# (rtReadback, rtGetDevicePointer) per name
BEFORE_RESIZE = dict({n: (STATE, STATE) for n in ELEMENT}, PixelStats=(UNKNOWN, STATE), TileSend=(UNKNOWN, STATE),
                     TileRecv=(UNKNOWN, STATE), NoSuchImage=(UNKNOWN, UNKNOWN))
BEFORE_PRODUCERS = dict(BEFORE_RESIZE, FrameRender=(OK, OK), AccumulatedRender=(OK, OK), TileSend=(UNKNOWN, OK), TileRecv=(UNKNOWN, OK))
AFTER_PRODUCERS = dict({n: (OK, OK) for n in ELEMENT}, PixelStats=(UNKNOWN, OK), TileSend=(UNKNOWN, OK), TileRecv=(UNKNOWN, OK),
                       NoSuchImage=(UNKNOWN, UNKNOWN))


def codes(ctx, name, nbytes=None):
    """(rtReadback's code, rtGetDevicePointer's code, its pointer, its byte count) for `name`; rtReadback gets nbytes (default: the
    image's W*H*element bytes at FRAME) into a buffer large enough for any of them."""
    w, h = FRAME
    nbytes = w * h * ELEMENT.get(name, 16) if nbytes is None else nbytes
    buf = np.zeros((w + 8) * h * 32 + 64, np.uint8)
    rb = ctx._L.rtReadback(ctx.handle, name.encode(), buf.ctypes.data_as(C.c_void_p), nbytes)
    p, n = C.c_void_p(), C.c_size_t()
    dp = ctx._L.rtGetDevicePointer(ctx.handle, name.encode(), C.byref(p), C.byref(n))
    return rb, dp, p.value, n.value


def assert_codes(ctx, want, what):
    got = {name: codes(ctx, name)[:2] for name in NAMES}
    bad = {name: (got[name], want[name]) for name in NAMES if got[name] != want[name]}
    assert not bad, f"{what}: (got, want) {bad}"


def open_ctx(lib, enable=True):
    sc = scenes.knot_room(*FRAME, 3, 1, nu=30, nv=6)
    mgr = rt.RayComputeManager(lib)
    scenes.apply(sc, mgr)
    if enable:
        mgr.OnEnable()
        mgr.context.set_bool("accumulate", True)
    return mgr, mgr.context


def run_producers(ctx):
    """Every producer once: a counting rtDispatch, rtDispatchFeatures, rtDenoise, rtDenoiseTemporal and rtDispatchAdaptive."""
    ctx.set_option("countStats", 1)
    ctx.set_int("Frame", 1)
    ctx.dispatch_full()
    ctx.dispatch_features()
    ctx.denoise()
    ctx.denoise_temporal()
    ctx.set_int("Frame", 2)
    assert ctx.dispatch_adaptive() == FRAME[0] * FRAME[1]


def snapshot(ctx):
    """Every W x H image as (H, W, bytes per pixel) uint8."""
    out = {name: ctx.readback(name) for name in READ_BACK}
    out["PixelStats"] = ctx.pixel_stats()
    return {name: np.ascontiguousarray(a).view(np.uint8).reshape(ctx.height, ctx.width, -1) for name, a in out.items()}


def test_codes_before_resize_before_the_producers_and_after_them():
    mgr, ctx = open_ctx(CUDA_LIB, enable=False)
    assert_codes(ctx, BEFORE_RESIZE, "before rtResize")
    mgr.OnEnable()
    ctx.set_bool("accumulate", True)
    assert_codes(ctx, BEFORE_PRODUCERS, "after rtResize")
    run_producers(ctx)
    assert_codes(ctx, AFTER_PRODUCERS, "after the producers")
    w, h = FRAME
    for name in ELEMENT:
        _, _, ptr, nbytes = codes(ctx, name)
        assert ptr and nbytes == w * h * ELEMENT[name], name
    for name in ("TileSend", "TileRecv"):                     # one rank: the whole image, frame and accumulated
        _, _, ptr, nbytes = codes(ctx, name)
        assert ptr and nbytes == w * h * 2 * 16, name
    for name in READ_BACK:
        right = w * h * ELEMENT[name]
        assert codes(ctx, name, right)[0] == OK, name
        assert codes(ctx, name, right - 16)[0] == INVALID, name
        assert codes(ctx, name, right + 16)[0] == INVALID, name
    mgr.OnDestroy()


def test_reset_accumulated_zeroes_the_accumulators_in_its_region_only():
    mgr, ctx = open_ctx(CUDA_LIB)
    run_producers(ctx)
    before = snapshot(ctx)
    ctx.dispatch(capi.RT_KERNEL_RESET_ACCUMULATED, 1, 1, 1)
    after = snapshot(ctx)
    inside = np.zeros((ctx.height, ctx.width), bool)
    inside[:8, :8] = True
    for name in before:
        if name in RESET_BY_RESET_ACCUMULATED:
            assert before[name][inside].any(), f"{name}: nothing to reset"
            assert not after[name][inside].any(), f"{name}: not zeroed inside the region"
            assert np.array_equal(after[name][~inside], before[name][~inside]), f"{name}: changed outside the region"
        else:
            assert np.array_equal(after[name], before[name]), f"{name}: changed by ResetAccumulated"
    mgr.OnDestroy()


def test_resize_keeps_every_image_at_the_same_size_and_zeroes_it_at_a_new_one():
    mgr, ctx = open_ctx(CUDA_LIB)
    run_producers(ctx)
    before = snapshot(ctx)
    w, h = ctx.width, ctx.height
    ctx.resize(w, h)
    after = snapshot(ctx)
    for name in before:
        assert np.array_equal(after[name], before[name]), f"{name}: changed by rtResize to the same size"
    ctx.resize(w + 8, h)
    ctx.set_ints("Resolution", [w + 8, h])
    after = snapshot(ctx)
    for name, a in after.items():
        assert a.shape[:2] == (h, w + 8) and not a.any(), f"{name}: not zero-filled at the new size"
        assert codes(ctx, name)[3] == (w + 8) * h * ELEMENT[name], name
    ctx.dispatch_full()
    ctx.dispatch_features()
    ctx.denoise_temporal()
    assert ctx.temporal_frame()[..., 2].max() == 1, "a resize discards the temporal history"
    mgr.OnDestroy()


def test_reset_stats_zeroes_pixel_stats_and_no_other_image():
    mgr, ctx = open_ctx(CUDA_LIB)
    run_producers(ctx)
    before = snapshot(ctx)
    assert before["PixelStats"].any()
    ctx.reset_stats()
    after = snapshot(ctx)
    assert not after["PixelStats"].any()
    for name in READ_BACK:
        assert np.array_equal(after[name], before[name]), f"{name}: changed by rtResetStats"
    mgr.OnDestroy()


def check_group_leader(lib, devices):
    """Through the leader of a group: the images of the camera render, the per-pixel counters' pointer (not their readback), tile
    buffers; the producers of the other images refuse the group, which leaves their codes as they were."""
    sc = scenes.knot_room(*FRAME, 3, 1, nu=30, nv=6)
    mgr = rt.RayComputeManager(lib, devices=devices)
    scenes.apply(sc, mgr)
    mgr.OnEnable()
    ctx = mgr.context
    ctx.set_bool("accumulate", True)
    assert_codes(ctx, BEFORE_PRODUCERS, "group leader after rtResize")
    ctx.set_option("countStats", 1)
    ctx.dispatch_full()
    for call in (ctx.dispatch_features, ctx.denoise, ctx.denoise_temporal, ctx.dispatch_adaptive, ctx.pixel_stats):
        with pytest.raises(capi.RtError) as e:
            call()
        assert e.value.code == STATE and "group" in str(e.value), call.__name__
    assert_codes(ctx, dict(BEFORE_PRODUCERS, PixelStats=(UNKNOWN, OK)), "group leader after a counting dispatch")
    w, h = FRAME
    assert codes(ctx, "PixelStats")[3] == w * h * 20
    rows = sum(min(8, h - y0) for b, y0 in enumerate(range(0, h, 8)) if b % len(devices) == 0)     # rank 0's share of 8-row bands
    assert codes(ctx, "TileSend")[3] == rows * w * 2 * 16
    assert codes(ctx, "TileRecv")[3] == rows * w * 2 * 16 * len(devices)
    mgr.OnDestroy()


def test_group_leader():
    torch = pytest.importorskip("torch")
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    check_group_leader(CUDA_LIB, [0, 1])
