"""The kernels at the edges of the C ABI's ranges on the H100 (`-m gpu`): NumRaysPerPixel around the pooled kernel's 20-bit sample
field, forced sample chunks past 2^32 jobs, image sides of 65535, and an image past 4 GiB per float4 image.  Large images are read
through rtGetDevicePointer and compared on the device or at sampled pixels; the oracle traces only the sampled pixels.

Every case opens one context at a time and destroys it before the next, and skips (naming its need) when the device has less free
memory than the case needs: the machines are shared.  On an H100 80GB HBM3 (700 W) the file took about 180 s, most of it the single-lane
renders of millions of samples per pixel in part a, and the device's memory use peaked at 38.8 GB (nvidia-smi, sampled each second:
the 4 GiB images with their copies).  The CPU twin of the sample-field and 65536-pixel cases is
tests/test_simt_limits.py."""
import ctypes as C

import numpy as np
import pytest

from conftest import CUDA_LIB, ORACLE_LIB, assert_bit_equal, render
import ray_tracing_b200 as rt
from ray_tracing_b200 import capi, scenes

pytestmark = pytest.mark.gpu

SPP_FIELD = 1 << 20          # the pooled kernel's slot counts a pixel's samples in 20 bits: RT_MAX_BATCH_SAMPLES = SPP_FIELD - 1
GB = 1 << 30


def limits_scene(width, height, bounces=1, spp=1, floor=True):
    """A cheap scene with every kind of geometry: sky, three spheres (one emissive) and one small mesh model — a knot on a floor that
    reaches the horizon, so that even a 65535 x 3 strip has pixels that hit something (floor=False: the knot alone, for the cases whose
    cost is millions of samples per pixel)."""
    knot = scenes.knot_mesh(nu=16, nv=4)
    if floor:
        plane = scenes.quad_mesh((-2e4, -1.75, -2e4), (-2e4, -1.75, 2e4), (2e4, -1.75, 2e4), (2e4, -1.75, -2e4))    # y = -0.7 in the world
        knot = scenes.merge_meshes([knot, plane])
    l2w, w2l = scenes.trs(position=(0.0, 0.0, 0.5), euler_deg=(0.0 if floor else 20.0, 35.0, 0.0), scale=(0.4, 0.4, 0.4))   # (the floor stays level)
    models = [scenes.ModelDesc(0, l2w, w2l, scenes.material(diffuse=(0.85, 0.55, 0.3), smoothness=0.6, specularProbability=0.1))]
    sph = np.array([scenes._sphere((-1.3, -0.2, 0.8), 0.5, scenes.material(diffuse=(0.3, 0.7, 0.3), specularProbability=0.0)),
                    scenes._sphere((1.3, -0.2, 0.8), 0.5, scenes.material(flag=scenes.MAT_GLASS, ior=1.5, smoothness=1.0, specularProbability=1.0)),
                    scenes._sphere((0.0, 1.2, 1.5), 0.3, scenes.material(diffuse=(0, 0, 0), emission=(1, 0.9, 0.8), emissionStrength=6.0))],
                   dtype=scenes.SPHERE_DTYPE)
    cam, _ = scenes.trs(position=(0.0, 0.0, -4.0))
    return scenes.Scene(name="limits", width=width, height=height, meshes=[knot], models=models, spheres=sph, cam_local_to_world=cam, fov=60.0,
                        settings=dict(maxBounceCount=bounces, numRaysPerPixel=spp, useSky=True))


def need_free(gb, what):
    """Skip the case when the device has less than `gb` GiB free (shared machines)."""
    torch = pytest.importorskip("torch")
    free, _ = torch.cuda.mem_get_info()
    if free < gb * GB:
        pytest.skip(f"{what} needs {gb} GiB of free device memory; {free / GB:.1f} GiB free")


class _Dev:
    def __init__(self, ptr, nbytes, typestr, item):
        self.__cuda_array_interface__ = {"shape": (nbytes // item,), "typestr": typestr, "data": (ptr, False), "version": 3, "strides": None}


def dev_image(ctx, name, H, W, comps=4, typestr="<f4"):
    """The context's image as a (H, W, comps) torch CUDA tensor over its device memory (no copy)."""
    import torch
    ptr, nbytes = ctx.device_pointer(name)
    assert nbytes == H * W * comps * 4, name
    return torch.as_tensor(_Dev(ptr, nbytes, typestr, 4), device="cuda").view(H, W, comps)


def bit_equal_dev(a, b):
    """Bitwise equality of two float32 CUDA tensors."""
    import torch
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


def oracle_pixels(sc, xy, frame):
    """The oracle's FrameRender values of the listed pixels (n x 2 int32, x y) at the given Frame."""
    mgr = rt.RayComputeManager(ORACLE_LIB)
    scenes.apply(sc, mgr)
    mgr.OnEnable()
    mgr.context.set_int("Frame", frame)
    out = np.empty((len(xy), 4), dtype=np.float32)
    xy = np.ascontiguousarray(xy, dtype=np.int32)
    assert C.CDLL(ORACLE_LIB).orRenderPixels(C.c_void_p(mgr.context.handle.value), xy.ctypes.data_as(C.c_void_p), len(xy),
                                             out.ctypes.data_as(C.c_void_p)) == 0
    mgr.OnDestroy()
    return out


def display_encode(values, frame):
    """rtDisplay's encode (tests/test_gpu_pixel_stats.py and the ingest tests pin it to the oracle's) of n float4 values as an n x 1
    AccumulatedRender with the given Frame: n x 4 uint8."""
    import torch
    ctx = capi.RtLib(CUDA_LIB).create(0)
    n = len(values)
    ctx.resize(n, 1)
    ctx.set_ints("Resolution", [n, 1])
    ptr, nbytes = ctx.device_pointer("AccumulatedRender")
    torch.as_tensor(_Dev(ptr, nbytes, "<f4", 4), device="cuda").copy_(torch.from_numpy(np.ascontiguousarray(values, np.float32).reshape(-1)))
    torch.cuda.synchronize()
    out = ctx.display(True, frame).reshape(n, 4)
    ctx.destroy()
    return out


def gather(img, xy):
    """The listed pixels (n x 2, x y) of a device image, copied out.  The library renders on a stream of its own: synchronise the
    context before reading what a call wrote."""
    import torch
    x = torch.as_tensor(xy[:, 0].astype(np.int64), device="cuda")
    y = torch.as_tensor(xy[:, 1].astype(np.int64), device="cuda")
    return img[y, x].cpu().numpy()


# ---- a. samples per pixel around the pooled kernel's 20-bit field ----------------------------------------------------------------

_ORACLE_A = {}


def _oracle_a(spp):
    if spp not in _ORACLE_A:
        _ORACLE_A[spp] = render(ORACLE_LIB, limits_scene(4, 2, 1, spp, floor=False), frames=2)
    return _ORACLE_A[spp]


@pytest.mark.parametrize("spp", [SPP_FIELD - 1, SPP_FIELD, SPP_FIELD + 1, 2 * SPP_FIELD + 3])
def test_samples_per_pixel_around_the_pool_field(spp):
    """4 x 2 pixels, one bounce, two frames: kernels 0, 1, the automatic choice and (up to RT_MAX_BATCH_SAMPLES) kernel 2 equal the
    oracle bit for bit; a forced kernel 2 above it is refused and the images stay as they were.  (At 4 x 2 pixels the automatic choice
    is kernel 1 by the small-tile rule; the rule that keeps more than RT_MAX_BATCH_SAMPLES samples off kernel 2 on large images is not
    covered: it needs about 3 x 10^11 samples.)"""
    fo, ao = _oracle_a(spp)
    assert np.all(fo[..., :3].sum(axis=-1) > 0)
    sc = limits_scene(4, 2, 1, spp, floor=False)
    for kernel in (0, 1, -1, 2):
        if kernel == 2 and spp > capi.RT_MAX_BATCH_SAMPLES:
            continue
        fg, ag = render(CUDA_LIB, sc, frames=2, options={"kernel": kernel})
        assert_bit_equal(fg, fo, f"spp {spp} kernel {kernel}: FrameRender")
        assert_bit_equal(ag, ao, f"spp {spp} kernel {kernel}: AccumulatedRender")
    if spp > capi.RT_MAX_BATCH_SAMPLES:
        mgr = rt.RayComputeManager(CUDA_LIB)
        scenes.apply(limits_scene(4, 2, 1, 1, floor=False), mgr)
        mgr.context.set_option("kernel", 2)
        mgr.OnEnable()
        mgr.RenderFrame()
        f0, a0 = mgr.raytraceFrameTex, mgr.accumulatedResult
        mgr.numRaysPerPixel = spp
        for call in (mgr.RenderFrame, lambda: mgr.RenderFrameAdaptive(0.0, 2, 2)):
            with pytest.raises(capi.RtError) as e:
                call()
            assert e.value.code == capi.RT_E_STATE
        assert mgr.numAccumulatedFrames == 2
        assert_bit_equal(mgr.raytraceFrameTex, f0, "FrameRender after the refused calls")
        assert_bit_equal(mgr.accumulatedResult, a0, "AccumulatedRender after the refused calls")
        mgr.OnDestroy()


def _adaptive_run(lib, sc, options):
    mgr = rt.RayComputeManager(lib)
    scenes.apply(sc, mgr)
    for k, v in options.items():
        mgr.context.set_option(k, v)
    mgr.OnEnable()
    counts = [mgr.RenderFrameAdaptive(0.0, 2, 2) for _ in range(2)]
    out = (counts, mgr.raytraceFrameTex, mgr.accumulatedResult, mgr.context.adaptive_moments())
    mgr.OnDestroy()
    return out


def test_adaptive_past_the_pool_field():
    """rtDispatchAdaptive with threshold 0 at 2^20 + 1 samples per pixel: the list-driven kernels 0, 1 and the automatic choice
    equal the oracle's two calls bit for bit."""
    sc = limits_scene(4, 2, 1, SPP_FIELD + 1, floor=False)
    ref = _adaptive_run(ORACLE_LIB, sc, {})
    assert ref[0] == [8, 8]
    for kernel in (0, 1, -1):
        got = _adaptive_run(CUDA_LIB, sc, {"kernel": kernel})
        assert got[0] == ref[0]
        for a, b, what in zip(got[1:], ref[1:], ("FrameRender", "AccumulatedRender", "AdaptiveMoments")):
            assert_bit_equal(a, b, f"kernel {kernel}: {what}")


# ---- b. forced sample chunks past 2^32 jobs -----------------------------------------------------------------------------------

def _edge_pixels(W, H, n, seed):
    rng = np.random.RandomState(seed)
    xy = [np.stack([rng.randint(0, W, n), rng.randint(0, H, n)], axis=1)]
    xy.append(np.stack([np.arange(W), np.full(W, H - 1)], axis=1))                 # last row
    xy.append(np.stack([np.full(H, W - 1), np.arange(H)], axis=1))                 # last column
    return np.concatenate(xy).astype(np.int32)


@pytest.mark.parametrize("W,H", [(8192, 8192), (8192, 8448), (35848, 1872)])
def test_forced_chunks_past_2_to_the_32_jobs(W, H):
    """Kernel 1 with "sampleChunks" = 64 on 2^26 and more pixel jobs: 64 x jobs does not fit the 32-bit work counter, so the dispatch
    takes fewer chunks — and the same bits as whole pixels.  8192 x 8192 is exactly 2^32 chunk jobs, 8192 x 8448 wraps to 2^27, and
    35848 x 1872 (67,107,456 jobs) would leave 64 x jobs only 90,112 short of 2^32: fewer than the resident lanes that each draw once
    more after the last job.  The chunked dispatch really runs in chunks (it allocates the hand-off buffer of 32 bytes per pixel job;
    whole pixels do not).  Its frame equals the same context's frame with sampleChunks = 1 (on the device) and, at 2048 seeded pixels
    plus the last row and column, the oracle."""
    import torch
    need_free(7, f"{W} x {H} with the chunk hand-off")
    jobs = ((W + 7) // 8) * ((H + 3) // 4) * 32
    sc = limits_scene(W, H, bounces=0, spp=64)
    mgr = rt.RayComputeManager(CUDA_LIB)
    scenes.apply(sc, mgr)
    ctx = mgr.context
    ctx.set_option("kernel", 1)
    ctx.set_option("sampleChunks", 64)
    mgr.OnEnable()
    ctx.synchronize()
    free0, _ = torch.cuda.mem_get_info()
    mgr.RenderFrame()
    ctx.synchronize()
    free1, _ = torch.cuda.mem_get_info()
    assert free0 - free1 >= 32 * jobs * 0.9, f"no chunk hand-off buffer: {(free0 - free1) / GB:.2f} GiB allocated for {jobs} jobs"
    frame = dev_image(ctx, "FrameRender", H, W)
    chunked = frame.clone()
    torch.cuda.synchronize()
    ctx.set_option("sampleChunks", 1)
    mgr.ResetAccumulatedRender()
    mgr.RenderFrame()
    ctx.synchronize()
    assert bit_equal_dev(chunked, frame), "sampleChunks 64 vs whole pixels"
    xy = _edge_pixels(W, H, 2048, 5)
    got = gather(chunked, xy)
    del frame, chunked
    mgr.OnDestroy()
    assert np.all(got[:, 3] == 1.0)
    assert_bit_equal(got, oracle_pixels(sc, xy, 1), f"{W} x {H}: sampled pixels")


# ---- c. sides of 65535 --------------------------------------------------------------------------------------------------------

def _session(lib, sc, options):
    """Every camera entry point in turn on one context; the images each leaves behind."""
    mgr = rt.RayComputeManager(lib)
    scenes.apply(sc, mgr)
    ctx = mgr.context
    for k, v in options.items():
        ctx.set_option(k, v)
    mgr.OnEnable()
    out = {}
    mgr.RenderFrame(); mgr.RenderFrame()
    out.update(frame2=mgr.raytraceFrameTex, accum2=mgr.accumulatedResult, display=ctx.display(True, 2), display_frame=ctx.display(False, 1))
    mgr.RenderFrames(3)
    out.update(frames_frame=mgr.raytraceFrameTex, frames_accum=mgr.accumulatedResult)
    ctx.set_option("countStats", 1)
    ctx.reset_stats()
    mgr.RenderFrame()
    out.update(pixel_stats=mgr.pixel_stats(), stats_frame=mgr.raytraceFrameTex)
    ctx.set_option("countStats", 0)
    mgr.ResetAccumulatedRender()
    counts = [mgr.RenderFrameAdaptive(0.3, 2, 8) for _ in range(3)]      # two calls of every pixel (minFrames 2), then a selection
    out.update(counts=counts, ad_frame=mgr.raytraceFrameTex, ad_accum=mgr.accumulatedResult, ad_moments=ctx.adaptive_moments(),
               display_mean=ctx.display_mean())
    ctx.dispatch_features()
    ctx.set_int("Frame", 5)
    ctx.dispatch_features()
    out.update({n: ctx.readback(n) for n in capi.FEATURE_IMAGES})
    out.update(camera_rays=ctx.camera_rays())
    ctx.denoise(True, 5)
    out.update(denoised=ctx.readback("DenoisedRender"))
    # the temporal filter over two camera positions
    ctx.denoise_temporal()
    mgr.set_camera(sc.fov, scenes.trs(position=(0.05, 0.02, -3.9), euler_deg=(0.5, 1.0, 0.0))[0])
    mgr.RenderFrame()
    ctx.dispatch_features()
    ctx.denoise_temporal()
    out.update(temporal=ctx.readback("DenoisedRender"), temporal_frame=ctx.temporal_frame())
    mgr.OnDestroy()
    return out


def _assert_session_equal(got, want, what):
    assert got["counts"] == want["counts"], f"{what}: adaptive counts"
    for k, v in want.items():
        if k == "counts":
            continue
        if v.dtype == np.uint8:
            assert np.array_equal(got[k], v), f"{what}: {k}"
        elif v.dtype.names:
            for f in v.dtype.names:
                a, b = np.ascontiguousarray(got[k][f]), np.ascontiguousarray(v[f])
                if a.dtype.kind == "f":
                    assert_bit_equal(a, b, f"{what}: {k}.{f}")
                else:
                    assert np.array_equal(a, b), f"{what}: {k}.{f}"
        else:
            assert_bit_equal(got[k], v, f"{what}: {k}")


@pytest.mark.parametrize("W,H", [(65535, 3), (3, 65535)])
def test_sides_of_65535(W, H):
    """65535 x 3 and 3 x 65535: pixel words (y << 16) | x with x or y = 65534 in the pooled slots and the adaptive pixel list.  Every
    camera entry point — rtDispatch (kernels 0, 1, 2; two frames), rtDispatchFrames(3), three rtDispatchAdaptive calls, countStats
    PixelStats, rtDispatchFeatures, rtCameraRays, rtDenoise (5 iterations), rtDenoiseTemporal over two camera positions, rtDisplay and
    rtDisplayMean — equals the oracle library's same calls."""
    sc = limits_scene(W, H, bounces=1, spp=1)
    want = _session(ORACLE_LIB, sc, {})
    assert 0 < want["counts"][2] < W * H and want["counts"][:2] == [W * H] * 2
    for kernel in (0, 1, 2):
        _assert_session_equal(_session(CUDA_LIB, sc, {"kernel": kernel}), want, f"{W} x {H} kernel {kernel}")


@pytest.mark.parametrize("W,H", [(65535, 3), (3, 65535)])
def test_sides_of_65535_in_row_bands(W, H):
    """Three ranks of row bands (rtSetTile; bands of 7 rows, of 1 row in the 3-row image so that every rank owns rows) for kernels 1
    and 2: the concatenated TileSend buffers unpack to the oracle's image."""
    import torch
    band = 1 if H < 21 else 7
    sc = limits_scene(W, H, bounces=1, spp=1)
    fo, ao = render(ORACLE_LIB, sc, frames=2)
    for kernel in (1, 2):
        sends = {}
        for r in (1, 2, 0):                              # rank 0 last: it unpacks the gathered buffer
            m = rt.RayComputeManager(CUDA_LIB)
            scenes.apply(sc, m)
            ctx = m.context
            ctx.set_option("kernel", kernel)
            ctx.set_tile(r, 3, band)
            m.OnEnable(); m.RenderFrame(); m.RenderFrame()
            ctx.pack_tile(); ctx.synchronize()
            ptr, nbytes = ctx.device_pointer("TileSend")
            sends[r] = torch.as_tensor(_Dev(ptr, nbytes, "<f4", 4), device="cuda").clone()
            if r != 0:
                m.OnDestroy()
        ptr, nbytes = ctx.device_pointer("TileRecv")
        torch.as_tensor(_Dev(ptr, nbytes, "<f4", 4), device="cuda").copy_(torch.cat([sends[r] for r in range(3)]))
        torch.cuda.synchronize()
        ctx.unpack_tiles(); ctx.synchronize()
        assert_bit_equal(m.raytraceFrameTex, fo, f"{W} x {H} kernel {kernel}: FrameRender reassembled")
        assert_bit_equal(m.accumulatedResult, ao, f"{W} x {H} kernel {kernel}: AccumulatedRender reassembled")
        m.OnDestroy()


# ---- d. past 4 GiB per image ----------------------------------------------------------------------------------------------------

BIG_W, BIG_H = 16384, 16392          # 268,566,528 pixels: indices past 2^28, float4 offsets past 2^32 bytes, uchar4 past 2^30 bytes


def _big_pixels():
    W, H = BIG_W, BIG_H
    xy = [_edge_pixels(W, H, 4096, 11)]
    for y in (8192, 16384):                                         # the rows where the pixel index crosses 2^27 and 2^28
        xy.append(np.stack([np.arange(W), np.full(W, y)], axis=1))
    return np.concatenate(xy).astype(np.int32)


def test_past_4_gib_kernels_frames_stats_and_display():
    """16384 x 16392, one sample, one bounce.  Kernels 0, 1 and 2 equal the oracle at the sampled pixels in frames 1 and 2 (and the
    accumulation is their sum); their PixelStats are equal (on the device); rtDispatchFrames(2) equals two rtDispatch calls (on the
    device); rtDisplay's bytes at the sampled pixels (past 2^30 bytes) equal the encode of the oracle's values in a one-row image."""
    import torch
    need_free(26, "the 16384 x 16392 frame, accumulation, PixelStats and their copies")
    W, H = BIG_W, BIG_H
    sc = limits_scene(W, H, bounces=1, spp=1)
    xy = _big_pixels()
    o1, o2 = oracle_pixels(sc, xy, 1), oracle_pixels(sc, xy, 2)
    mgr = rt.RayComputeManager(CUDA_LIB)
    scenes.apply(sc, mgr)
    ctx = mgr.context
    mgr.OnEnable()
    frame, accum = dev_image(ctx, "FrameRender", H, W), dev_image(ctx, "AccumulatedRender", H, W)
    stats0 = None
    for kernel in (0, 1, 2):
        ctx.set_option("kernel", kernel)
        mgr.ResetAccumulatedRender()
        mgr.RenderFrame()
        ctx.synchronize()
        assert_bit_equal(gather(frame, xy), o1, f"kernel {kernel}: frame 1")
        mgr.RenderFrame()
        ctx.synchronize()
        assert_bit_equal(gather(frame, xy), o2, f"kernel {kernel}: frame 2")
        a = gather(accum, xy)
        assert_bit_equal(a[:, :3], o1[:, :3] + o2[:, :3], f"kernel {kernel}: accumulation")
        assert np.all(a[:, 3] == 2.0)
        ctx.set_option("countStats", 1)
        ctx.reset_stats()
        mgr.RenderFrame()
        ctx.synchronize()
        stats = dev_image(ctx, "PixelStats", H, W, comps=5, typestr="<u4")
        if stats0 is None:
            stats0 = stats.clone()
            torch.cuda.synchronize()
            assert int(stats0[..., 0].sum()) >= W * H
        else:
            assert torch.equal(stats, stats0), f"kernel {kernel}: PixelStats"
        del stats
        ctx.set_option("countStats", 0)
    del stats0
    ctx.set_option("kernel", -1)
    mgr.ResetAccumulatedRender()
    mgr.RenderFrame(); mgr.RenderFrame()
    ctx.synchronize()
    f2, a2 = frame.clone(), accum.clone()
    torch.cuda.synchronize()
    mgr.ResetAccumulatedRender()
    mgr.RenderFrames(2)
    ctx.synchronize()
    assert bit_equal_dev(frame, f2) and bit_equal_dev(accum, a2), "rtDispatchFrames(2) vs two rtDispatch calls"
    del f2, a2, frame, accum
    disp = ctx.display(True, 2)[xy[:, 1], xy[:, 0]]          # (1 GiB to the host: the ABI hands the display out to host memory only)
    mgr.OnDestroy()
    assert np.array_equal(disp, display_encode(o1 + o2, 2)), "rtDisplay at the sampled pixels"


def oracle_features(sc, xy, frame):
    """orFeaturePixels: the oracle's FeatureFrame records of the listed pixels (n x 2 int32, x y) at the given Frame."""
    mgr = rt.RayComputeManager(ORACLE_LIB)
    scenes.apply(sc, mgr)
    mgr.OnEnable()
    mgr.context.set_int("Frame", frame)
    out = np.empty(len(xy), dtype=capi.PIXEL_FEATURES_DTYPE)
    xy = np.ascontiguousarray(xy, dtype=np.int32)
    assert C.CDLL(ORACLE_LIB).orFeaturePixels(C.c_void_p(mgr.context.handle.value), xy.ctypes.data_as(C.c_void_p), len(xy),
                                              out.ctypes.data_as(C.c_void_p)) == 0
    mgr.OnDestroy()
    return out


def test_past_4_gib_features_and_denoise():
    """rtDispatchFeatures and rtDenoise at 16384 x 16392, where the 32-byte feature records pass 2^32 bytes at pixel 2^27.  For frames 1
    and 2, FeatureFrame at the sampled pixels equals orFeaturePixels, and AccumulatedAlbedo / AccumulatedNormal there equal the oracle
    records summed as the accumulators sum them.  rtDenoise (5 iterations) of the two accumulated frames equals orDenoiseImages run on
    256 x 256 crops of the same colour, albedo and normal images, at the crop pixels at least 62 from a crop border inside the image (the
    filter's support after 5 iterations, 2 (1 + 2 + 4 + 8 + 16)); the crops lie at the image's corners, across the row where the pixel
    index crosses 2^27, and on the top rows, past 2^28."""
    import torch
    from test_gpu_denoise import oracle_hook
    need_free(44, "the 16384 x 16392 frame, accumulation, feature images, denoised image and denoise scratch")
    W, H = BIG_W, BIG_H
    sc = limits_scene(W, H, bounces=1, spp=1)
    xy = _big_pixels()
    mgr = rt.RayComputeManager(CUDA_LIB)
    scenes.apply(sc, mgr)
    ctx = mgr.context
    mgr.OnEnable()
    mgr.RenderFrame(); mgr.RenderFrame()
    hits = np.zeros(len(xy), np.float32)
    alb = np.zeros((len(xy), 4), np.float32)
    nrm = np.zeros((len(xy), 4), np.float32)
    for f in (1, 2):
        ctx.set_int("Frame", f)
        ctx.dispatch_features()
        ctx.synchronize()
        got = gather(dev_image(ctx, "FeatureFrame", H, W, comps=8, typestr="<i4"), xy).view(capi.PIXEL_FEATURES_DTYPE).reshape(-1)
        want = oracle_features(sc, xy, f)
        for k in ("albedo", "dst", "normal"):
            assert_bit_equal(np.ascontiguousarray(got[k]), np.ascontiguousarray(want[k]), f"frame {f}: FeatureFrame.{k}")
        assert np.array_equal(got["object"], want["object"]), f"frame {f}: FeatureFrame.object"
        hit = want["object"] != -1
        alb[hit, :3] += want["albedo"][hit]; alb[hit, 3] += np.float32(1)
        nrm[hit, :3] += want["normal"][hit]; nrm[hit, 3] += want["dst"][hit]
        hits += hit
    assert 0 < hits.sum() < 2 * len(xy)
    assert_bit_equal(gather(dev_image(ctx, "AccumulatedAlbedo", H, W), xy), alb, "AccumulatedAlbedo")
    assert_bit_equal(gather(dev_image(ctx, "AccumulatedNormal", H, W), xy), nrm, "AccumulatedNormal")
    sigma = (capi.DENOISE_SIGMA_COLOUR, capi.DENOISE_SIGMA_NORMAL, capi.DENOISE_SIGMA_DEPTH)
    ctx.denoise(True, 5, *sigma)
    ctx.synchronize()
    images = {n: dev_image(ctx, n, H, W) for n in ("AccumulatedRender", "AccumulatedAlbedo", "AccumulatedNormal", "DenoisedRender")}
    S, M = 256, 62
    for x0, y0 in ((0, 0), (W - S, H - S), (W // 2 - S // 2, 8192 - S // 2), (4000, H - S)):
        crop = {n: img[y0:y0 + S, x0:x0 + S].cpu().numpy() for n, img in images.items()}
        rc, want = oracle_hook(S, S, 1, crop["AccumulatedRender"], crop["AccumulatedAlbedo"], crop["AccumulatedNormal"], 5, sigma)
        assert rc == capi.RT_OK
        # a crop side on the image's border needs no margin: the filter meets the same border in both
        ya, yb = (0 if y0 == 0 else M), S - (0 if y0 + S == H else M)
        xa, xb = (0 if x0 == 0 else M), S - (0 if x0 + S == W else M)
        assert_bit_equal(crop["DenoisedRender"][ya:yb, xa:xb], want[ya:yb, xa:xb], f"DenoisedRender, crop at ({x0}, {y0})")
    del images
    mgr.OnDestroy()


def _criterion_dev(m, threshold, min_frames, max_frames):
    """test_gpu_adaptive.criterion in torch float32 on the device."""
    import torch
    n = m[..., 2]
    mu = m[..., 0] / n
    v = torch.fmax(m[..., 1] / n - mu * mu, torch.zeros_like(mu))
    t = torch.tensor(threshold, dtype=torch.float32, device="cuda")
    eps = torch.tensor(0.00390625, dtype=torch.float32, device="cuda")
    return (n < min_frames) | ((n < max_frames) & (v > ((t * t) * n) * (mu * mu + eps)))


def _same_where(a, b, mask, rows=1024):
    """Bitwise equality of a and b where mask is set, a band of rows at a time (no image-sized temporaries)."""
    import torch
    for y in range(0, a.shape[0], rows):
        m = mask[y:y + rows]
        if not torch.equal(a[y:y + rows][m].view(torch.int32), b[y:y + rows][m].view(torch.int32)):
            return False
    return True


def test_past_4_gib_adaptive():
    """rtDispatchAdaptive at 16384 x 16392: after two calls of every pixel, the selective third call traces exactly the pixels the
    criterion names (on the device); their FrameRender equals a plain rtDispatch of the same Frame and every other pixel of FrameRender,
    AccumulatedRender and AdaptiveMoments is unchanged."""
    import torch
    need_free(32, "the 16384 x 16392 frame, accumulation, moments, pixel list and copies of the three images")
    W, H = BIG_W, BIG_H
    mgr = rt.RayComputeManager(CUDA_LIB)
    scenes.apply(limits_scene(W, H, bounces=1, spp=1), mgr)
    ctx = mgr.context
    mgr.OnEnable()
    for f in (1, 2):
        ctx.set_int("Frame", f)
        assert ctx.dispatch_adaptive(0.3, 2, 8) == W * H
    ctx.synchronize()
    frame, accum, mom = (dev_image(ctx, n, H, W) for n in ("FrameRender", "AccumulatedRender", "AdaptiveMoments"))
    want = _criterion_dev(mom, 0.3, 2, 8)
    f0, a0, m0 = frame.clone(), accum.clone(), mom.clone()
    torch.cuda.synchronize()
    ctx.set_int("Frame", 3)
    n = ctx.dispatch_adaptive(0.3, 2, 8)
    ctx.synchronize()
    assert n == int(want.sum()) and 0 < n < W * H
    for before, after, name in ((f0, frame, "FrameRender"), (a0, accum, "AccumulatedRender"), (m0, mom, "AdaptiveMoments")):
        assert _same_where(before, after, ~want), f"untraced {name}"
    del a0, m0
    traced = frame[want].clone()
    torch.cuda.synchronize()
    ctx.dispatch(capi.RT_KERNEL_RAYTRACE, (W + 7) // 8, (H + 7) // 8, 1)
    ctx.synchronize()
    assert torch.equal(traced.view(torch.int32), frame[want].view(torch.int32)), "traced pixels vs rtDispatch"
    del f0, traced, frame, accum, mom, want
    mgr.OnDestroy()
