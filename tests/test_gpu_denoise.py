"""rtDenoise / rtDisplayDenoised on the H100 (`-m gpu`): the a-trous denoiser equals the oracle bit for bit on rendered scenes (both
sources, every iteration count, two sigma sets, after 1 / 3 / 8 frames, with the feature images rendered every frame or only on some) and
on synthetic images written through rtGetDevicePointer (the oracle's orDenoiseImages on the same arrays: zero and sub-floor albedo,
denormals, signed zeros, overflowing demodulation, NaN and infinities, L.w = 0, extreme depth ratios, sigmas at the edges, 1x1 to
ragged shapes); background pixels pass through and never weigh; a crease stops the filter; the call changes nothing else; resize,
device pointer, stream order, the managers and every refusal.  The same bodies run in the CPU suite against the SIMT interpreter build
(tests/test_simt_denoise.py)."""
import ctypes as C

import numpy as np
import pytest

from conftest import CUDA_LIB, ORACLE_LIB, assert_bit_equal
from ray_tracing_b200 import capi, scenes
import test_gpu_features as F

pytestmark = pytest.mark.gpu

FRAME = (40, 24)                # size of the rendered images (the interpreter twin uses a smaller one)
SIGMAS = ((capi.DENOISE_SIGMA_COLOUR, capi.DENOISE_SIGMA_NORMAL, capi.DENOISE_SIGMA_DEPTH), (0.3, 0.1, 2.0))
INPUTS = ("FrameRender", "AccumulatedRender") + capi.FEATURE_IMAGES


def write_device(ptr, arr):
    """Copies a host array into device memory of the context's GPU (the interpreter twin replaces this with a memmove)."""
    import torch

    class _Dev:
        def __init__(self, p, n):
            self.__cuda_array_interface__ = {"shape": (n,), "typestr": "|u1", "data": (p, False), "version": 3, "strides": None}
    b = np.ascontiguousarray(arr).view(np.uint8).reshape(-1)
    torch.as_tensor(_Dev(ptr, b.size), device="cuda").copy_(torch.from_numpy(b.copy()))
    torch.cuda.synchronize()


def oracle_hook(W, H, use_acc, colour, albedo, normal_or_features, iterations, sigma):
    """orDenoiseImages of the oracle on caller arrays: (return code, (H, W, 4) float32)."""
    L = C.CDLL(ORACLE_LIB)
    f = L.orDenoiseImages
    f.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    out = np.zeros((H, W, 4), np.float32)
    colour = np.ascontiguousarray(colour, np.float32)
    albedo = None if albedo is None else np.ascontiguousarray(albedo, np.float32)
    nf = np.ascontiguousarray(normal_or_features)
    s = np.asarray(sigma, np.float32)
    rc = f(W, H, use_acc, colour.ctypes.data, None if albedo is None else albedo.ctypes.data, nf.ctypes.data, iterations, s.ctypes.data,
           out.ctypes.data)
    return rc, out


def render(ctx, frames, feature_frames):
    """Frames with accumulation, the feature images of the frames in feature_frames dispatched before them; returns after the last."""
    for f in frames:
        ctx.set_int("Frame", f)
        if f in feature_frames:
            ctx.dispatch_features()
        ctx.dispatch_full()


def denoised_all(ctx, iterations=range(1, 6)):
    """DenoisedRender for both sources, every iteration count and both sigma sets."""
    out = {}
    for acc in (1, 0):
        for k in iterations:
            for si, s in enumerate(SIGMAS):
                ctx.denoise(bool(acc), k, *s)
                out[(acc, k, si)] = ctx.readback("DenoisedRender")
    return out


SCHEDULES = {"every": (lambda f: True), "some": (lambda f: f in (1, 2, 5))}       # L.w < A.w after frame 2


def check_scene(make, checkpoints=(1, 3, 8), size=None):
    """Rendered, accumulated and denoised on the oracle and the product (model skipping on and off); DenoisedRender equal after each
    checkpoint for every source, iteration count and sigma set."""
    for sched, use in SCHEDULES.items():
        frames = range(1, max(checkpoints) + 1)
        feats = {f for f in frames if use(f)}
        want = {}
        mgr, octx = F.open_ctx(ORACLE_LIB, make(), size=size)
        done = 0
        for cp in checkpoints:
            render(octx, range(done + 1, cp + 1), feats)
            done = cp
            want[cp] = denoised_all(octx)
        mgr.OnDestroy()
        for skip in (1, 0):
            mgr, ctx = F.open_ctx(CUDA_LIB, make(), {"modelSkip": skip}, size=size)
            done = 0
            for cp in checkpoints:
                render(ctx, range(done + 1, cp + 1), feats)
                done = cp
                got = denoised_all(ctx)
                for key, img in want[cp].items():
                    assert_bit_equal(got[key], img, f"{make().name} {sched} modelSkip={skip} frames={cp} (acc, iterations, sigma)={key}")
            mgr.OnDestroy()
    return want


# ---- 1. rendered scenes against the oracle -------------------------------------------------------------------------------------------
def test_cornell_box():
    want = check_scene(lambda: scenes.cornell_spheres(24, 16, 4, 1))
    assert any(not np.array_equal(v, want[8][(1, 1, 0)]) for v in want[8].values())


def test_knot_room_with_glass():
    check_scene(lambda: scenes.knot_room(24, 16, 6, 1, nu=40, nv=8, glass=True))


def test_checker_soup_with_sky_defocus_and_spheres():
    check_scene(F.checker_soup)


def test_152_instanced_knots_with_the_tlas():
    check_scene(lambda: scenes.instanced_knots(24, 16, 4, 1, instances=150), checkpoints=(1, 3))


def test_ten_thousand_spheres():
    check_scene(lambda: scenes.random_soup(24, 16, 4, 1, triangles=300, spheres=10000), checkpoints=(1, 3))


def test_unity_fixture():
    from test_round2_abi import load_fixture
    check_scene(lambda: load_fixture(24, 16), checkpoints=(1, 3))


# ---- 2. synthetic images through the oracle's hook -----------------------------------------------------------------------------------
def blank_ctx(lib, W, H):
    """A context of W x H whose five input images exist (a feature dispatch that covers nothing allocates them)."""
    ctx = capi.RtLib(lib).create(0)
    ctx.resize(W, H)
    ctx.set_ints("Resolution", [W, H])
    ctx.dispatch_features(0, 0, 1)
    return ctx


def synthetic(W, H, seed, adversarial=True):
    """The five input images, random with adversarial values sprinkled in."""
    r = np.random.RandomState(seed)
    n = W * H
    frame = (r.rand(n, 4) * 3).astype(np.float32)
    accum = (r.rand(n, 4) * 6).astype(np.float32)
    accum[:, 3] = r.randint(1, 9, n)
    alb = r.rand(n, 4).astype(np.float32)
    alb[:, 3] = np.minimum(accum[:, 3], r.randint(0, 9, n))
    nrm = np.concatenate([r.randn(n, 3), r.rand(n, 1) * 10 + 1], axis=1).astype(np.float32) * alb[:, 3:4]
    feat = np.zeros(n, capi.PIXEL_FEATURES_DTYPE)
    feat["albedo"] = r.rand(n, 3)
    feat["dst"] = r.rand(n) * 10 + 0.5
    nn = r.randn(n, 3)
    feat["normal"] = nn / np.linalg.norm(nn, axis=1, keepdims=True)
    feat["object"] = r.randint(-3, 4, n)
    if adversarial:
        bits = lambda u: np.uint32(u).view(np.float32)
        specials = np.float32([0.0, -0.0, np.nan, np.inf, -np.inf, bits(1), bits(0x807fffff), 3e38, 1e-3, 2.0 ** -9, -5.0, 1e30, 1e-30])
        for img in (frame, accum, alb, nrm):
            k = r.rand(*img.shape) < 0.06
            img[k] = r.choice(specials, k.sum())
        for fld in ("albedo", "dst", "normal"):
            v = feat[fld].reshape(n, -1)
            k = r.rand(*v.shape) < 0.06
            v[k] = r.choice(specials, k.sum())
            feat[fld] = v.reshape(feat[fld].shape)
        accum[r.rand(n) < 0.05, 3] = 0                                   # never accumulated
        alb[r.rand(n) < 0.05, 3] = 0                                     # frames, but no feature ray hit
        alb[r.rand(n) < 0.05, :3] = 0                                    # black albedo: demodulated by the 2^-8 floor
        with np.errstate(over="ignore"):
            nrm[r.rand(n) < 0.05, 3] *= np.float32(1e30)                 # depth ratios that overflow D ...
        nrm[r.rand(n) < 0.05, 3] *= np.float32(1e-30)                    # ... and underflow it
    return {"FrameRender": frame.reshape(H, W, 4), "AccumulatedRender": accum.reshape(H, W, 4), "FeatureFrame": feat.reshape(H, W),
            "AccumulatedAlbedo": alb.reshape(H, W, 4), "AccumulatedNormal": nrm.reshape(H, W, 4)}


def load_images(ctx, imgs):
    for name, img in imgs.items():
        ptr, nbytes = ctx.device_pointer(name)
        assert nbytes == img.nbytes
        write_device(ptr, img)


def check_synthetic(ctx, imgs, W, H, iterations_list=range(1, 6), sigmas=SIGMAS, what=""):
    load_images(ctx, imgs)
    for acc in (1, 0):
        colour = imgs["AccumulatedRender" if acc else "FrameRender"]
        albedo = imgs["AccumulatedAlbedo"] if acc else None
        nf = imgs["AccumulatedNormal"] if acc else imgs["FeatureFrame"]
        for k in iterations_list:
            for s in sigmas:
                rc, want = oracle_hook(W, H, acc, colour, albedo, nf, k, s)
                assert rc == capi.RT_OK
                ctx.denoise(bool(acc), k, *s)
                assert_bit_equal(ctx.readback("DenoisedRender"), want, f"{what} {W}x{H} acc={acc} iterations={k} sigma={s}")


@pytest.mark.parametrize("W,H", [(1, 1), (1, 19), (23, 1), (37, 13), (70, 41)])
def test_synthetic_images_against_the_oracle_hook(W, H):
    ctx = blank_ctx(CUDA_LIB, W, H)
    for seed in (1, 2):
        check_synthetic(ctx, synthetic(W, H, seed), W, H, what=f"seed {seed}")
    check_synthetic(ctx, synthetic(W, H, 3, adversarial=False), W, H, what="clean")


def test_sigmas_at_the_edges_of_the_accepted_range():
    W, H = 33, 17
    ctx = blank_ctx(CUDA_LIB, W, H)
    imgs = synthetic(W, H, 5)
    tiny = np.float32(2.0 ** -63)           # 1 / tiny^2 = 2^126: finite
    edges = [(float(tiny * 16), 1.0, 1.0),  # invC * 4^4 = 2^118 at five iterations
             (1.0, float(tiny), 1.0), (1.0, 1.0, float(np.float32(2.0 ** -126) * 4)),
             (3e38, 3e38, 3e38)]            # sigma^2 overflows: the constants are 0, an infinite difference gives a NaN D (weight 0)
    check_synthetic(ctx, imgs, W, H, iterations_list=(1, 5), sigmas=edges, what="edge sigmas")


# ---- 3. semantics --------------------------------------------------------------------------------------------------------------------
def test_background_passes_through_and_never_weighs():
    W, H = 31, 21
    ctx = blank_ctx(CUDA_LIB, W, H)
    imgs = synthetic(W, H, 7, adversarial=False)
    feat = imgs["FeatureFrame"]
    feat["object"] = 1
    feat["object"][5:9, 3:30] = -1                                              # sky
    imgs["FrameRender"][10, 10, :3] = np.nan                                    # a NaN pixel (the NaN specularCol of the features tests)
    imgs["FrameRender"][12, 12, :3] = np.float32(1e30)                          # and a huge one that demodulates to inf ...
    feat["albedo"][12, 12] = np.float32(1e-9)
    load_images(ctx, imgs)
    ctx.denoise(False, 5, 1.0, 0.5, 0.25)
    base = ctx.readback("DenoisedRender")
    bg = feat["object"] == -1
    bg[10, 10] = bg[12, 12] = True
    want = imgs["FrameRender"].copy()
    want[..., 3] = 1
    assert_bit_equal(base[bg], want[bg], "background passes through as (c, 1)")
    # ... and its values never reach a neighbour: change every background pixel's colour, nothing else moves
    imgs["FrameRender"][bg] = np.float32(77.0)
    load_images(ctx, imgs)
    ctx.denoise(False, 5, 1.0, 0.5, 0.25)
    again = ctx.readback("DenoisedRender")
    assert_bit_equal(again[~bg], base[~bg], "background colours do not reach other pixels")
    assert np.isfinite(base[~bg]).all()


def test_a_crease_with_a_small_sigma_normal_stops_the_filter():
    """Two halves at 90 degrees: with sigmaNormal small, no weight crosses (each half filtered as if the other were background)."""
    W, H = 32, 16
    ctx = blank_ctx(CUDA_LIB, W, H)
    imgs = synthetic(W, H, 9, adversarial=False)
    feat = imgs["FeatureFrame"]
    feat["object"] = 0
    feat["normal"][:, :16] = (1, 0, 0)
    feat["normal"][:, 16:] = (0, 1, 0)
    feat["dst"] = 5.0
    load_images(ctx, imgs)
    ctx.denoise(False, 5, 1.0, 0.01, 1.0)
    got = ctx.readback("DenoisedRender")
    for side in (slice(0, 16), slice(16, 32)):
        alone = {k: v.copy() for k, v in imgs.items()}
        other = np.ones(W, bool)
        other[side] = False
        alone["FeatureFrame"]["object"][:, other] = -1
        load_images(ctx, alone)
        ctx.denoise(False, 5, 1.0, 0.01, 1.0)
        assert_bit_equal(got[:, side], ctx.readback("DenoisedRender")[:, side], f"crease: columns {side}")


def test_the_call_changes_nothing_else_and_repeats():
    make = F.checker_soup
    results = []
    for with_denoise in (False, True):
        mgr, ctx = F.open_ctx(CUDA_LIB, make(), {"countStats": 1})
        ctx.reset_stats()
        for f in range(1, 4):
            mgr.RenderFeatures()
            mgr.RenderFrame()
            if with_denoise:
                before = {n: ctx.readback(n) for n in INPUTS}
                st, pix, frame_no = ctx.stats(), ctx.pixel_stats(), mgr.numAccumulatedFrames
                mgr.Denoise()
                first = mgr.denoised_result
                ctx.denoise(False, 3, 0.5, 0.2, 0.1)
                ctx.denoise(True, capi.DENOISE_ITERATIONS, capi.DENOISE_SIGMA_COLOUR, capi.DENOISE_SIGMA_NORMAL, capi.DENOISE_SIGMA_DEPTH)
                assert ctx.readback("DenoisedRender").tobytes() == first.tobytes(), "the same call twice gives the same bits"
                for n in INPUTS:
                    assert ctx.readback(n).tobytes() == before[n].tobytes(), f"{n} changed by rtDenoise"
                assert ctx.stats() == st and ctx.pixel_stats().tobytes() == pix.tobytes() and mgr.numAccumulatedFrames == frame_no
        results.append({n: ctx.readback(n) for n in INPUTS})
        mgr.OnDestroy()
    for n in INPUTS:
        assert results[1][n].tobytes() == results[0][n].tobytes(), f"{n}: later dispatches render other bits after rtDenoise"


def test_managers_equal_the_raw_context():
    make = lambda: scenes.knot_room(24, 16, 4, 1, nu=40, nv=8, glass=True)
    for lib in (ORACLE_LIB, CUDA_LIB):
        mgr, ctx = F.open_ctx(lib, make())
        for _ in range(2):
            mgr.RenderFeatures()
            mgr.RenderFrame()
        mgr.Denoise()
        via_mgr = mgr.denoised_result
        ctx.denoise(True)
        assert_bit_equal(via_mgr, ctx.readback("DenoisedRender"), f"{lib}: Denoise() vs rtDenoise")
        mgr.accumulate = False
        mgr.RenderFeatures()
        mgr.RenderFrame()
        mgr.Denoise(2, 0.5, 0.25, 0.5)
        ctx.denoise(False, 2, 0.5, 0.25, 0.5)
        assert_bit_equal(mgr.denoised_result, ctx.readback("DenoisedRender"), f"{lib}: Denoise() with accumulate off")
        mgr.OnDestroy()


def test_display_resize_and_readback_states():
    got = {}
    for lib in (ORACLE_LIB, CUDA_LIB):
        mgr, ctx = F.open_ctx(lib, F.checker_soup())
        mgr.RenderFeatures()
        mgr.RenderFrame()
        ctx.denoise(True, 3)
        got[lib] = (ctx.readback("DenoisedRender"), ctx.display_denoised())
        if lib == CUDA_LIB:                # rtDisplay's encode with Frame = 1: the same image through FrameRender and rtDisplay
            ptr, _ = ctx.device_pointer("FrameRender")
            write_device(ptr, got[lib][0])
            assert ctx.display(False, 1).tobytes() == got[lib][1].tobytes(), "rtDisplayDenoised vs rtDisplay(FrameRender, 1)"
        w, h = ctx.width, ctx.height
        ctx.resize(w + 8, h)
        ctx.set_ints("Resolution", [w + 8, h])
        img = ctx.readback("DenoisedRender")
        assert img.shape == (h, w + 8, 4) and not img.any(), f"{lib}: a resize zeroes DenoisedRender"
        assert not ctx.display_denoised().any()
        ctx.dispatch_features()
        ctx.denoise(False, 2)
        assert ctx.readback("DenoisedRender").shape == (h, w + 8, 4)
        mgr.OnDestroy()
    assert_bit_equal(got[CUDA_LIB][0], got[ORACLE_LIB][0], "DenoisedRender")
    assert got[CUDA_LIB][1].tobytes() == got[ORACLE_LIB][1].tobytes(), "rtDisplayDenoised"


def test_every_refusal_and_state():
    sc = scenes.knot_room(16, 12, 3, 1, nu=30, nv=6)
    for lib in (ORACLE_LIB, CUDA_LIB):
        mgr = F.T.open_mgr(lib, sc, enable=False)
        ctx, L, h = mgr.context, mgr.context._L, mgr.context.handle
        ok = (1, 3, 1.0, 0.5, 0.25)
        rgba = np.zeros(16 * 12 * 4, np.uint8)
        assert L.rtDenoise(h, *ok) == capi.RT_E_STATE                          # before rtResize
        mgr.OnEnable()
        assert L.rtDenoise(h, *ok) == capi.RT_E_STATE                          # before the first rtDispatchFeatures
        for call in (lambda: ctx.readback("DenoisedRender"), ctx.display_denoised):
            with pytest.raises(capi.RtError) as e:
                call()
            assert e.value.code == capi.RT_E_STATE, lib
        ctx.dispatch_features()
        inf, nan = float("inf"), float("nan")
        assert L.rtDenoise(None, *ok) == capi.RT_E_INVALID
        for bad in ((2, 3, 1.0, 0.5, 0.25), (-1, 3, 1.0, 0.5, 0.25), (1, 0, 1.0, 0.5, 0.25), (1, 6, 1.0, 0.5, 0.25),
                    (1, 3, 0.0, 0.5, 0.25), (1, 3, -1.0, 0.5, 0.25), (1, 3, inf, 0.5, 0.25), (1, 3, nan, 0.5, 0.25),
                    (1, 3, 1.0, 0.0, 0.25), (1, 3, 1.0, inf, 0.25), (1, 3, 1.0, 0.5, -0.0), (1, 3, 1.0, 0.5, nan),
                    (1, 5, 2.0 ** -60, 0.5, 0.25),       # invC * 4^4 = 2^128: not finite (2^-60 alone passes at three iterations)
                    (1, 3, 1.0, 2.0 ** -64, 0.25),       # 1 / sigmaNormal^2 = 2^128
                    (1, 3, 1.0, 0.5, 2.0 ** -140)):      # 1 / sigmaDepth overflows
            assert L.rtDenoise(h, *bad) == capi.RT_E_INVALID, (lib, bad)
        assert L.rtDenoise(h, 1, 3, 2.0 ** -60, 0.5, 0.25) == capi.RT_OK
        assert L.rtDisplayDenoised(None, rgba.ctypes.data, rgba.nbytes) == capi.RT_E_INVALID
        assert L.rtDisplayDenoised(h, None, rgba.nbytes) == capi.RT_E_INVALID
        assert L.rtDisplayDenoised(h, rgba.ctypes.data, rgba.nbytes - 4) == capi.RT_E_INVALID
        assert L.rtDisplayDenoised(h, rgba.ctypes.data, rgba.nbytes) == capi.RT_OK
        out = np.zeros(16 * 12 * 5, np.float32)
        assert L.rtReadback(h, b"DenoisedRender", out.ctypes.data, out.nbytes) == capi.RT_E_INVALID
        ctx.set_ints("Resolution", [8, 12])
        assert L.rtDenoise(h, *ok) == capi.RT_E_STATE
        ctx.set_ints("Resolution", [16, 12])
        ctx.set_tile(0, 2, 4)
        assert L.rtDenoise(h, *ok) == capi.RT_E_STATE                          # its images hold its own bands only
        ctx.set_tile(0, 1, 1)
        assert L.rtDenoise(h, *ok) == capi.RT_OK
        mgr.OnDestroy()


# ---- 4. GPU only ----------------------------------------------------------------------------------------------------------------------
def test_group_context_is_refused():
    torch = pytest.importorskip("torch")
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    check_group_refusal(CUDA_LIB, [0, 1])


def check_group_refusal(lib, devices):
    import ray_tracing_b200 as rt
    mgr = rt.RayComputeManager(lib, devices=devices)
    scenes.apply(scenes.knot_room(16, 12, 3, 1, nu=30, nv=6), mgr)
    mgr.OnEnable()
    with pytest.raises(capi.RtError) as e:
        mgr.context.denoise(True)
    assert e.value.code == capi.RT_E_STATE and "group" in str(e.value)
    mgr.OnDestroy()


def test_device_pointer_and_stream_order():
    """rtDenoise on a caller's stream, DenoisedRender copied on that stream right after it with no host synchronisation between."""
    torch = pytest.importorskip("torch")
    W, H = 64, 40
    ctx = blank_ctx(CUDA_LIB, W, H)
    imgs = synthetic(W, H, 11)
    load_images(ctx, imgs)
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    for k in (1, 4):
        ctx.denoise(True, k, 0.5, 0.3, 0.2)
        ptr, nbytes = ctx.device_pointer("DenoisedRender")
        assert nbytes == W * H * 16

        class _Dev:
            __cuda_array_interface__ = {"shape": (nbytes // 4,), "typestr": "<f4", "data": (ptr, False), "version": 3, "strides": None}
        with torch.cuda.stream(stream):
            copy = torch.as_tensor(_Dev(), device="cuda").clone()
        stream.synchronize()
        rc, want = oracle_hook(W, H, 1, imgs["AccumulatedRender"], imgs["AccumulatedAlbedo"], imgs["AccumulatedNormal"], k, (0.5, 0.3, 0.2))
        assert rc == capi.RT_OK
        assert_bit_equal(copy.cpu().numpy().reshape(H, W, 4), want, f"iterations {k} on a caller stream")
    ctx.set_stream(0)


def test_720p_five_iterations_against_the_oracle_hook():
    W, H = 1280, 720
    ctx = blank_ctx(CUDA_LIB, W, H)
    check_synthetic(ctx, synthetic(W, H, 13), W, H, iterations_list=(5,), sigmas=SIGMAS[:1], what="720p")
