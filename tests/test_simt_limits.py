"""The limits of the C ABI's ranges on the SIMT interpreter build (tests/simt): a NumRaysPerPixel past the pooled kernel's 20-bit
sample field, and image sides past 65535.  The H100 runs the same edges at full size in tests/test_gpu_limits.py."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import ORACLE_LIB, REPO, assert_bit_equal, render
import ray_tracing_b200 as rt
from ray_tracing_b200 import capi, scenes
from test_gpu_limits import SPP_FIELD, limits_scene

sys.path.insert(0, os.path.join(REPO, "tests", "simt"))
import build as simt_build   # noqa: E402


@pytest.fixture(scope="session")
def simt_lib():
    return simt_build.build()


def _snapshot(ctx, names):
    """Bytes of the named images that exist (device pointers of the interpreter build are host pointers)."""
    out = {}
    for n in names:
        try:
            ptr, nbytes = ctx.device_pointer(n)
        except capi.RtError:
            continue
        out[n] = C.string_at(ptr, nbytes)
    return out


def forced_pool_kernel_is_refused(lib):
    """"kernel" = 2 with NumRaysPerPixel = 2^20 + 1: rtDispatch and rtDispatchAdaptive are refused with RT_E_STATE and change nothing;
    the render then goes on from the same frame as if the refused calls had not been made.  (Run in a child process: a pooled kernel
    that took such a count would count sample 2^20 as sample 0 and never finish.)"""
    sc = limits_scene(2, 2, bounces=0, spp=1)
    mgr = rt.RayComputeManager(lib)
    scenes.apply(sc, mgr)
    ctx = mgr.context
    ctx.set_option("kernel", 2)
    mgr.OnEnable()
    mgr.RenderFrame()
    assert mgr.RenderFrameAdaptive(0.0, 2, 64) == 4          # the adaptive state (moments, pixel list) exists before the refusals
    names = ("FrameRender", "AccumulatedRender", "AdaptiveMoments")
    before, frames = _snapshot(ctx, names), mgr.numAccumulatedFrames
    assert set(before) == set(names)
    mgr.numRaysPerPixel = SPP_FIELD + 1
    for call in (mgr.RenderFrame, lambda: mgr.RenderFrameAdaptive(0.0, 2, 64)):
        with pytest.raises(capi.RtError) as e:
            call()
        assert e.value.code == capi.RT_E_STATE
    assert mgr.numAccumulatedFrames == frames
    after = _snapshot(ctx, names)
    for n in names:
        assert after[n] == before[n], f"{n} changed by a refused call"
    mgr.numRaysPerPixel = 1
    mgr.RenderFrame()
    fo, ao = render(ORACLE_LIB, sc, frames=frames)             # the frames of RenderFrame, RenderFrameAdaptive (every pixel) and this one
    assert_bit_equal(mgr.raytraceFrameTex, fo, "FrameRender after the refused calls")
    assert_bit_equal(mgr.accumulatedResult, ao, "AccumulatedRender after the refused calls")
    mgr.OnDestroy()


def test_simt_forced_pool_kernel_refuses_samples_past_its_field(simt_lib):
    """forced_pool_kernel_is_refused in a child process with a timeout, so that a regression fails the test instead of hanging it."""
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + \
          ["-c", "import sys; sys.path[:0] = sys.argv[1:3]; import test_simt_limits as T; T.forced_pool_kernel_is_refused(sys.argv[3])",
           REPO, os.path.join(REPO, "tests"), simt_lib]
    try:
        r = subprocess.run(cmd, capture_output=True, text=True, timeout=60)
    except subprocess.TimeoutExpired:
        pytest.fail("a forced kernel 2 dispatch of 2^20 + 1 samples per pixel did not return within 60 s")
    assert r.returncode == 0, r.stdout + r.stderr


def test_simt_automatic_kernel_past_the_pool_field_equals_the_oracle(simt_lib):
    """NumRaysPerPixel = 2^20 + 1 with the automatic kernel on a mesh scene (sky, one bounce): two pixels, bit for bit against the
    oracle; the count runs through the persistent kernel's int sample loop.  At two pixels the small-tile rule already picks kernel 1,
    so this does not reach the rule that keeps such counts off kernel 2 on large images (effectiveKernel): that rule is not covered."""
    sc = limits_scene(2, 1, bounces=1, spp=SPP_FIELD + 1)
    fo, ao = render(ORACLE_LIB, sc)
    assert np.all(fo[..., :3].sum(axis=-1) > 0)
    fg, ag = render(simt_lib, sc)
    assert_bit_equal(fg, fo, "FrameRender, automatic kernel")
    assert_bit_equal(ag, ao, "AccumulatedRender, automatic kernel")


@pytest.mark.parametrize("size", [(65536, 1), (1, 65536)])
def test_simt_camera_entry_points_refuse_sides_past_65535(simt_lib, size):
    """The pixel lists and the pooled slots store a pixel as (y << 16) | x: every camera entry point refuses a side of 65536 with
    RT_E_STATE and leaves every image as it was."""
    W, H = size
    mgr = rt.RayComputeManager(simt_lib)
    scenes.apply(limits_scene(W, H, bounces=0, spp=1), mgr)
    mgr.OnEnable()                                              # (clearing the accumulation is not a camera entry point)
    ctx = mgr.context
    rng = np.random.RandomState(3)
    for n in ("FrameRender", "AccumulatedRender"):
        ptr, nbytes = ctx.device_pointer(n)
        pattern = rng.randint(0, 256, nbytes).astype(np.uint8).tobytes()
        C.memmove(ptr, pattern, nbytes)
    names = ("FrameRender", "AccumulatedRender", "FeatureFrame", "AccumulatedAlbedo", "AccumulatedNormal", "AdaptiveMoments", "PixelStats")
    before = _snapshot(ctx, names)
    calls = {"rtDispatch": lambda: ctx.dispatch_full(), "rtDispatchFrames": lambda: ctx.dispatch_frames(2),
             "rtDispatchAdaptive": lambda: ctx.dispatch_adaptive(0.0, 2, 64), "rtDispatchFeatures": lambda: ctx.dispatch_features(),
             "rtCameraRays": lambda: ctx.camera_rays()}
    for what, call in calls.items():
        with pytest.raises(capi.RtError) as e:
            call()
        assert e.value.code == capi.RT_E_STATE, what
    assert _snapshot(ctx, names) == before
    mgr.OnDestroy()


def test_simt_widest_image_equals_the_oracle(simt_lib):
    """65535 x 2: x = 65534 is the largest x a (y << 16) | x pixel word holds; kernels 1 and 2 against the oracle, one frame."""
    sc = limits_scene(65535, 2, bounces=0, spp=1)
    fo, ao = render(ORACLE_LIB, sc)
    for kernel in (1, 2):
        fg, ag = render(simt_lib, sc, options={"kernel": kernel})
        assert_bit_equal(fg, fo, f"65535 x 2, kernel {kernel}")
        assert_bit_equal(ag, ao, f"65535 x 2 accumulated, kernel {kernel}")
