"""ctypes binding of the C-ABI declared in include/rt_b200.h.

`RtLib()` loads the product library, librt_b200.so (CUDA, sm_90a).  There is no CPU fallback: if the
library is missing it raises, and `RtLib.create()` raises when no H100-class (sm_90) GPU is present.  Tests and
bench.py may pass another path implementing the same ABI (the CPU oracle) — the product never does.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import numpy as np

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
DEFAULT_LIB = os.path.join(PKG_DIR, "librt_b200.so")

RT_OK = 0
RT_E_INVALID, RT_E_UNKNOWN_NAME, RT_E_NO_DEVICE, RT_E_CUDA, RT_E_STATE = -1, -2, -3, -4, -5
RT_KERNEL_RAYTRACE, RT_KERNEL_RESET_ACCUMULATED = 0, 1
RT_MAX_BATCH_SAMPLES = (1 << 20) - 1      # rtDispatchFrames: frameCount * max(1, NumRaysPerPixel) at most this

# numpy dtypes of the blittable structs in include/rt_types.h
MATERIAL_DTYPE = np.dtype([
    ("diffuseCol", "<f4", 4), ("emissionCol", "<f4", 4), ("specularCol", "<f4", 4), ("absorption", "<f4", 4),
    ("absorptionStrength", "<f4"), ("emissionStrength", "<f4"), ("smoothness", "<f4"),
    ("specularProbability", "<f4"), ("ior", "<f4"), ("flag", "<i4")])
NODE_DTYPE = np.dtype([("boundsMin", "<f4", 3), ("boundsMax", "<f4", 3), ("startIndex", "<i4"), ("triangleCount", "<i4")])
TRIANGLE_DTYPE = np.dtype([("posA", "<f4", 3), ("posB", "<f4", 3), ("posC", "<f4", 3),
                           ("normA", "<f4", 3), ("normB", "<f4", 3), ("normC", "<f4", 3)])
MODEL_DTYPE = np.dtype([("nodeOffset", "<i4"), ("triOffset", "<i4"), ("worldToLocal", "<f4", 16),
                        ("localToWorld", "<f4", 16), ("material", MATERIAL_DTYPE)])
SPHERE_DTYPE = np.dtype([("centre", "<f4", 3), ("radius", "<f4"), ("material", MATERIAL_DTYPE)])
assert MATERIAL_DTYPE.itemsize == 88 and NODE_DTYPE.itemsize == 32 and TRIANGLE_DTYPE.itemsize == 72
assert MODEL_DTYPE.itemsize == 224 and SPHERE_DTYPE.itemsize == 104

BUFFER_DTYPES = {"Triangles": TRIANGLE_DTYPE, "Nodes": NODE_DTYPE, "ModelInfo": MODEL_DTYPE, "Spheres": SPHERE_DTYPE}

# RtPixelStats: the per-pixel counters of the counting launches ("countStats" = 1), uint32, wrapping modulo 2^32
PIXEL_STATS_DTYPE = np.dtype([("rays", "<u4"), ("boxTests", "<u4"), ("triTests", "<u4"), ("sphereTests", "<u4"), ("sphereBoxTests", "<u4")])
assert PIXEL_STATS_DTYPE.itemsize == 20
# rtDisplayPixelStats visMode: what the heat map shows per pixel
VIS_MODES = {1: "boxTests per ray", 2: "triTests per ray", 3: "sphere tests per ray", 4: "rays"}

# rtTraceRays: a caller-supplied ray and its closest hit (RtRay / RtRayHit)
RAY_DTYPE = np.dtype([("origin", "<f4", 3), ("dir", "<f4", 3)])
RAY_HIT_DTYPE = np.dtype([("dst", "<f4"), ("pos", "<f4", 3), ("normal", "<f4", 3), ("isBackface", "<i4"), ("kind", "<i4"),
                          ("index", "<i4"), ("pad", "<i4", 2)])
assert RAY_DTYPE.itemsize == 24 and RAY_HIT_DTYPE.itemsize == 48
RT_HIT_NONE, RT_HIT_SPHERE, RT_HIT_MODEL = 0, 1, 2
RT_TRACE_CHUNK_RAYS = 1 << 20      # rtTraceRays: host arrays travel in batches of at most this many rays
RT_TRACE_NO_CULL = 1      # forceDontCullBack (RayCommon.hlsl:356): back faces count for every model, not only glass


def make_rays(origins, dirs=None) -> np.ndarray:
    """A RAY_DTYPE array from a structured array (returned as it is) or from (n, 3) origins and (n, 3) directions."""
    if dirs is None:
        rays = np.asarray(origins)
        if rays.dtype != RAY_DTYPE:
            raise TypeError(f"rays must have dtype {RAY_DTYPE} (or pass origins and dirs)")
        return np.ascontiguousarray(rays).reshape(-1)
    o = np.asarray(origins, dtype=np.float32).reshape(-1, 3)
    d = np.asarray(dirs, dtype=np.float32).reshape(-1, 3)
    if o.shape != d.shape:
        raise ValueError("origins and dirs must both be (n, 3)")
    rays = np.empty(o.shape[0], dtype=RAY_DTYPE)
    rays["origin"], rays["dir"] = o, d
    return rays


# rtTraceOcclusion: a caller-supplied segment, origin + t * dir for 0 <= t < tMax (RtRaySegment)
SEGMENT_DTYPE = np.dtype([("origin", "<f4", 3), ("dir", "<f4", 3), ("tMax", "<f4")])
assert SEGMENT_DTYPE.itemsize == 28


def make_segments(origins, dirs=None, t_max=None) -> np.ndarray:
    """A SEGMENT_DTYPE array from a structured array (returned as it is) or from (n, 3) origins, (n, 3) directions and n tMax values
    (a scalar applies to every segment)."""
    if dirs is None:
        segs = np.asarray(origins)
        if segs.dtype != SEGMENT_DTYPE:
            raise TypeError(f"segments must have dtype {SEGMENT_DTYPE} (or pass origins, dirs and t_max)")
        return np.ascontiguousarray(segs).reshape(-1)
    if t_max is None:
        raise ValueError("t_max is required with origins and dirs")
    o = np.asarray(origins, dtype=np.float32).reshape(-1, 3)
    d = np.asarray(dirs, dtype=np.float32).reshape(-1, 3)
    if o.shape != d.shape:
        raise ValueError("origins and dirs must both be (n, 3)")
    segs = np.empty(o.shape[0], dtype=SEGMENT_DTYPE)
    segs["origin"], segs["dir"] = o, d
    segs["tMax"] = np.broadcast_to(np.asarray(t_max, dtype=np.float32).reshape(-1), (o.shape[0],))
    return segs


# rtTracePaths: a caller-supplied path start (RtPathRay) and the radiance along it (RtPathRadiance)
PATH_RAY_DTYPE = np.dtype([("origin", "<f4", 3), ("dir", "<f4", 3), ("rngState", "<u4")])
PATH_RADIANCE_DTYPE = np.dtype([("rgb", "<f4", 3), ("rngState", "<u4")])
assert PATH_RAY_DTYPE.itemsize == 28 and PATH_RADIANCE_DTYPE.itemsize == 16


def make_path_rays(origins, dirs=None, rng_state=None) -> np.ndarray:
    """A PATH_RAY_DTYPE array from a structured array (returned as it is) or from (n, 3) origins, (n, 3) directions (used as given,
    not normalised) and n uint32 RNG states (a scalar applies to every ray)."""
    if dirs is None:
        rays = np.asarray(origins)
        if rays.dtype != PATH_RAY_DTYPE:
            raise TypeError(f"path rays must have dtype {PATH_RAY_DTYPE} (or pass origins, dirs and rng_state)")
        return np.ascontiguousarray(rays).reshape(-1)
    if rng_state is None:
        raise ValueError("rng_state is required with origins and dirs")
    o = np.asarray(origins, dtype=np.float32).reshape(-1, 3)
    d = np.asarray(dirs, dtype=np.float32).reshape(-1, 3)
    if o.shape != d.shape:
        raise ValueError("origins and dirs must both be (n, 3)")
    rays = np.empty(o.shape[0], dtype=PATH_RAY_DTYPE)
    rays["origin"], rays["dir"] = o, d
    rays["rngState"] = np.broadcast_to(np.asarray(rng_state, dtype=np.uint64).astype(np.uint32).reshape(-1), (o.shape[0],))
    return rays


# rtBakeProbes: one probe's L2 spherical harmonics (RtProbeSH)
PROBE_SH_DTYPE = np.dtype([("sh", "<f4", (3, 9)), ("rejected", "<u4")])
assert PROBE_SH_DTYPE.itemsize == 112
RT_PROBE_CHUNK = 32
RT_PROBE_SCRATCH_CHUNKS = 1 << 20

# rtBakeCubemaps: one cube-map texel (RtCubeTexel)
CUBE_TEXEL_DTYPE = np.dtype([("rgb", "<f4", 3), ("rejected", "<u4")])
assert CUBE_TEXEL_DTYPE.itemsize == 16
RT_CUBE_MAX_FACE = 4096
RT_CUBE_SCRATCH_CHUNKS = 7 << 20

# rtBakeLightmap: one surface texel (RtSurfacePoint); its result is a CUBE_TEXEL_DTYPE record
SURFACE_POINT_DTYPE = np.dtype([("position", "<f4", 3), ("normal", "<f4", 3)])
assert SURFACE_POINT_DTYPE.itemsize == 24


def as_surface_points(points) -> np.ndarray:
    """An (n,) SURFACE_POINT_DTYPE array as given, or (n, 6) floats (position, normal) as one; contiguous."""
    if isinstance(points, np.ndarray) and points.dtype == SURFACE_POINT_DTYPE:
        return np.ascontiguousarray(points.reshape(-1))
    return np.ascontiguousarray(np.asarray(points, dtype=np.float32).reshape(-1, 6)).view(SURFACE_POINT_DTYPE).reshape(-1)


# rtDispatchFeatures: one pixel of "FeatureFrame" (RtPixelFeatures).  object: ModelInfo index m -> m, Spheres index s -> -2 - s, miss -> -1
PIXEL_FEATURES_DTYPE = np.dtype([("albedo", "<f4", 3), ("dst", "<f4"), ("normal", "<f4", 3), ("object", "<i4")])
assert PIXEL_FEATURES_DTYPE.itemsize == 32
FEATURE_IMAGES = ("FeatureFrame", "AccumulatedAlbedo", "AccumulatedNormal")

# rtDenoise: the defaults of the managers (the C ABI has none), chosen by the quality sweep of DESIGN.md section 7d''''''
DENOISE_MAX_ITERATIONS = 5
DENOISE_ITERATIONS = 5
DENOISE_SIGMA_COLOUR = 64.0
DENOISE_SIGMA_NORMAL = 1.0
DENOISE_SIGMA_DEPTH = 0.1

# rtDenoiseTemporal: the defaults of the managers, chosen by the quality sweep of DESIGN.md section 7d'''''''
TEMPORAL_ITERATIONS = 5
TEMPORAL_SIGMA_LUMINANCE = 8.0
TEMPORAL_SIGMA_NORMAL = 1.0
TEMPORAL_SIGMA_DEPTH = 0.1
TEMPORAL_ALPHA = 0.1
TEMPORAL_MAX_HISTORY = 32          # RT_TEMPORAL_MAX_HISTORY

# rtDispatchAdaptive: the defaults of the managers, chosen by the quality sweep of DESIGN.md section 7d''''''''
ADAPTIVE_MAX_FRAMES_LIMIT = 1 << 24     # RT_ADAPTIVE_MAX_FRAMES
ADAPTIVE_THRESHOLD = 0.2
ADAPTIVE_MIN_FRAMES = 8
ADAPTIVE_MAX_FRAMES = 64


class RtStats(C.Structure):
    _fields_ = [("rays", C.c_uint64), ("boxTests", C.c_uint64), ("triTests", C.c_uint64), ("sphereTests", C.c_uint64),
                ("dispatches", C.c_uint64), ("kernelMs", C.c_double), ("sphereBoxTests", C.c_uint64), ("exchangeMs", C.c_double)]


class RtError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"rt error {code}: {msg}")
        self.code = code


class RtLib:
    """A loaded implementation of the rt_b200.h ABI."""

    def __init__(self, path: Optional[str] = None):
        self.path = path or DEFAULT_LIB
        if not os.path.exists(self.path):
            raise FileNotFoundError(
                f"{self.path} not found — build it with `python -m ray_tracing_b200.build` "
                "(librt_b200 is CUDA-only; there is no CPU fallback)")
        L = self.lib = C.CDLL(self.path)
        vp, cp, ci, cf = C.c_void_p, C.c_char_p, C.c_int, C.c_float
        sig = {
            "rtGetVersion": ([], ci),
            "rtCreate": ([C.POINTER(vp), ci], ci),
            "rtDestroy": ([vp], ci),
            "rtLastError": ([vp], cp),
            "rtSetBuffer": ([vp, cp, vp, ci, ci], ci),
            "rtSetInt": ([vp, cp, ci], ci),
            "rtSetInts": ([vp, cp, C.POINTER(ci), ci], ci),
            "rtSetFloat": ([vp, cp, cf], ci),
            "rtSetVector": ([vp, cp, C.POINTER(cf)], ci),
            "rtSetMatrix": ([vp, cp, C.POINTER(cf)], ci),
            "rtSetBool": ([vp, cp, ci], ci),
            "rtResize": ([vp, ci, ci], ci),
            "rtDispatch": ([vp, ci, ci, ci, ci], ci),
            "rtReadback": ([vp, cp, vp, C.c_size_t], ci),
            "rtSynchronize": ([vp], ci),
            "rtDisplay": ([vp, ci, ci, vp, C.c_size_t], ci),
            "rtSetStream": ([vp, vp], ci),
            "rtSetTile": ([vp, ci, ci, ci], ci),
            "rtPackTile": ([vp], ci),
            "rtUnpackTiles": ([vp], ci),
            "rtGetDevicePointer": ([vp, cp, C.POINTER(vp), C.POINTER(C.c_size_t)], ci),
            "rtSetOption": ([vp, cp, ci], ci),
            "rtGetIpcHandles": ([vp, vp, C.c_size_t], ci),
            "rtSetPeers": ([vp, ci, vp, C.c_size_t], ci),
            "rtGetStats": ([vp, C.POINTER(RtStats)], ci),
            "rtResetStats": ([vp], ci),
            "rtBuildBVH": ([vp, vp, ci, vp, ci, vp, ci, vp, vp, ci, C.POINTER(ci)], ci),
            "rtCreateMulti": ([C.POINTER(vp), C.POINTER(ci), ci], ci),
            "rtGetUniqueId": ([vp, C.c_size_t], ci),
            "rtCommInit": ([vp, vp, C.c_size_t, ci, ci], ci),
            "rtCommDestroy": ([vp], ci),
            "rtExchangeTiles": ([vp], ci),
            "rtReadbackAsync": ([vp, cp, vp, C.c_size_t], ci),
            "rtDisplayAsync": ([vp, ci, ci, vp, C.c_size_t], ci),
            "rtReadbackWait": ([vp], ci),
            "rtReadbackPixelStats": ([vp, vp, C.c_size_t], ci),
            "rtDisplayPixelStats": ([vp, ci, cf, vp, C.c_size_t], ci),
            "rtDispatchFrames": ([vp, ci, ci, ci, ci], ci),
            "rtTraceRays": ([vp, vp, ci, vp, ci], ci),
            "rtTraceRaysDevice": ([vp, vp, vp, ci, ci], ci),
            "rtTraceOcclusion": ([vp, vp, ci, vp, ci], ci),
            "rtTraceOcclusionDevice": ([vp, vp, vp, ci, ci], ci),
            "rtTracePaths": ([vp, vp, ci, ci, vp], ci),
            "rtTracePathsDevice": ([vp, vp, vp, ci, ci], ci),
            "rtBakeProbes": ([vp, vp, ci, ci, C.c_uint32, vp], ci),
            "rtBakeProbesDevice": ([vp, vp, vp, ci, ci, C.c_uint32], ci),
            "rtBakeCubemaps": ([vp, vp, ci, ci, ci, C.c_uint32, vp], ci),
            "rtBakeCubemapsDevice": ([vp, vp, vp, ci, ci, ci, C.c_uint32], ci),
            "rtBakeLightmap": ([vp, vp, ci, ci, C.c_uint32, vp], ci),
            "rtBakeLightmapDevice": ([vp, vp, vp, ci, ci, C.c_uint32], ci),
            "rtDispatchFeatures": ([vp, ci, ci, ci], ci),
            "rtCameraRays": ([vp, vp, C.c_size_t], ci),
            "rtCameraRaysDevice": ([vp, vp, C.c_size_t], ci),
            "rtDenoise": ([vp, ci, ci, cf, cf, cf], ci),
            "rtDisplayDenoised": ([vp, vp, C.c_size_t], ci),
            "rtDenoiseTemporal": ([vp, ci, cf, cf, cf, cf, ci], ci),
            "rtDispatchAdaptive": ([vp, ci, ci, ci, cf, ci, ci, C.POINTER(C.c_int64)], ci),
            "rtDisplayMean": ([vp, vp, C.c_size_t], ci),
        }
        for name, (args, res) in sig.items():
            if not hasattr(L, name):
                if name in ("rtGetIpcHandles", "rtSetPeers", "rtBuildBVH", "rtCreateMulti", "rtGetUniqueId", "rtCommInit", "rtCommDestroy", "rtExchangeTiles", "rtReadbackAsync", "rtDisplayAsync", "rtReadbackWait",
                            "rtReadbackPixelStats", "rtDisplayPixelStats", "rtDispatchFrames", "rtTraceRays", "rtTraceRaysDevice",
                            "rtTraceOcclusion", "rtTraceOcclusionDevice", "rtTracePaths", "rtTracePathsDevice",
                            "rtBakeProbes", "rtBakeProbesDevice", "rtBakeCubemaps", "rtBakeCubemapsDevice", "rtBakeLightmap", "rtBakeLightmapDevice", "rtDispatchFeatures", "rtCameraRays", "rtCameraRaysDevice", "rtDenoise", "rtDisplayDenoised", "rtDenoiseTemporal",
                            "rtDispatchAdaptive", "rtDisplayMean"):      # absent from older experimental builds used in A/B runs
                    continue
                raise AttributeError(f"{self.path} does not export {name}")
            fn = getattr(L, name)
            fn.argtypes, fn.restype = args, res

    def create(self, device: int = 0) -> "RtContext":
        h = C.c_void_p()
        rc = self.lib.rtCreate(C.byref(h), device)
        if rc != RT_OK:
            raise RtError(rc, (self.lib.rtLastError(None) or b"").decode())
        return RtContext(self, h)

    def create_multi(self, devices) -> "RtContext":
        """rtCreateMulti: ONE context that renders on all `devices` of this process (row-band tiles + the all-gather inside rtDispatch)."""
        devices = list(devices)
        arr = (C.c_int * len(devices))(*devices)
        h = C.c_void_p()
        rc = self.lib.rtCreateMulti(C.byref(h), arr, len(devices))
        if rc != RT_OK:
            raise RtError(rc, (self.lib.rtLastError(None) or b"").decode())
        return RtContext(self, h)

    def unique_id(self) -> bytes:
        """rtGetUniqueId: the 128 bytes rank 0 hands to every rank for rtCommInit."""
        buf = C.create_string_buffer(128)
        rc = self.lib.rtGetUniqueId(buf, 128)
        if rc != RT_OK:
            raise RtError(rc, (self.lib.rtLastError(None) or b"").decode())
        return buf.raw


class RtContext:
    def __init__(self, lib: RtLib, handle: C.c_void_p):
        self._lib, self._L, self._h = lib, lib.lib, handle
        self.width = self.height = 0

    # -- plumbing
    def _ck(self, rc: int):
        if rc != RT_OK:
            raise RtError(rc, (self._L.rtLastError(self._h) or b"").decode())

    @property
    def handle(self) -> C.c_void_p:
        return self._h

    def destroy(self):
        if self._h:
            self._L.rtDestroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.destroy()
        except Exception:
            pass

    # -- ComputeShader-like surface
    def set_buffer(self, name: str, data: np.ndarray):
        dt = BUFFER_DTYPES.get(name)
        if dt is not None and data.dtype != dt:
            raise TypeError(f"{name} expects dtype {dt}")
        a = np.ascontiguousarray(data)
        self._ck(self._L.rtSetBuffer(self._h, name.encode(), a.ctypes.data_as(C.c_void_p) if a.size else None,
                                     int(a.shape[0]) if a.ndim else 0, a.dtype.itemsize))

    def set_buffer_raw(self, name: str, ptr, count: int, stride: int):
        self._ck(self._L.rtSetBuffer(self._h, name.encode(), ptr, count, stride))

    def set_int(self, name: str, v: int):
        self._ck(self._L.rtSetInt(self._h, name.encode(), int(v)))

    def set_ints(self, name: str, vals):
        arr = (C.c_int * len(vals))(*[int(v) for v in vals])
        self._ck(self._L.rtSetInts(self._h, name.encode(), arr, len(vals)))

    def set_float(self, name: str, v: float):
        self._ck(self._L.rtSetFloat(self._h, name.encode(), float(v)))

    def set_vector(self, name: str, v):
        vv = list(v) + [0.0] * (4 - len(v))
        arr = (C.c_float * 4)(*[float(x) for x in vv])
        self._ck(self._L.rtSetVector(self._h, name.encode(), arr))

    def set_matrix(self, name: str, m):
        """m: 4x4 array in ordinary (row, col) indexing; sent column-major like Unity's Matrix4x4."""
        a = np.asarray(m, dtype=np.float32).reshape(4, 4)
        flat = np.ascontiguousarray(a.T).reshape(16)
        arr = (C.c_float * 16)(*[float(x) for x in flat])
        self._ck(self._L.rtSetMatrix(self._h, name.encode(), arr))

    def set_bool(self, name: str, v: bool):
        self._ck(self._L.rtSetBool(self._h, name.encode(), 1 if v else 0))

    def resize(self, w: int, h: int):
        self._ck(self._L.rtResize(self._h, int(w), int(h)))
        self.width, self.height = int(w), int(h)

    def dispatch(self, kernel: int, gx: int, gy: int, gz: int = 1):
        self._ck(self._L.rtDispatch(self._h, kernel, gx, gy, gz))

    def dispatch_full(self, kernel: int = RT_KERNEL_RAYTRACE):
        """ComputeHelper.Dispatch(cs, width, height, kernelIndex) (ComputeHelper.cs:25-32)."""
        self.dispatch(kernel, (self.width + 7) // 8, (self.height + 7) // 8, 1)

    def dispatch_frames(self, n: int, gx: Optional[int] = None, gy: Optional[int] = None, gz: int = 1):
        """rtDispatchFrames: n accumulated RayTrace frames, Frame .. Frame + n - 1, in one launch — the same bytes as n dispatch()
        calls with "Frame" stepped by one each time; "Frame" is left unchanged.  Groups default to the whole image."""
        gx = (self.width + 7) // 8 if gx is None else gx
        gy = (self.height + 7) // 8 if gy is None else gy
        self._ck(self._L.rtDispatchFrames(self._h, int(gx), int(gy), int(gz), int(n)))

    def dispatch_adaptive(self, threshold: float = ADAPTIVE_THRESHOLD, min_frames: int = ADAPTIVE_MIN_FRAMES, max_frames: int = ADAPTIVE_MAX_FRAMES,
                          gx: Optional[int] = None, gy: Optional[int] = None, gz: int = 1) -> int:
        """rtDispatchAdaptive: the next accumulated RayTrace frame of the current "Frame", traced only in the covered pixels whose
        estimated error is still above `threshold` (or that have fewer than min_frames adaptive frames); their luminance moments go to
        "AdaptiveMoments" (adaptive_moments()).  Returns the number of pixels traced: 0 = converged.  Groups default to the whole image.
        Synchronises once before the render launch, which stays queued."""
        gx = (self.width + 7) // 8 if gx is None else gx
        gy = (self.height + 7) // 8 if gy is None else gy
        active = C.c_int64(0)
        self._ck(self._L.rtDispatchAdaptive(self._h, int(gx), int(gy), int(gz), float(threshold), int(min_frames), int(max_frames), C.byref(active)))
        return int(active.value)

    def adaptive_moments(self) -> np.ndarray:
        """"AdaptiveMoments": (H, W, 4) float32, row 0 = bottom, (sum of l, sum of l*l, frames, 0) per pixel over its adaptive frames."""
        return self.readback("AdaptiveMoments")

    def display_mean(self) -> np.ndarray:
        """rtDisplayMean: the per-pixel mean AccumulatedRender / AccumulatedRender.w encoded as rtDisplay encodes; (0, 0, 0, 255)
        where nothing was accumulated.  (H, W, 4) uint8, row 0 = bottom."""
        out = np.empty((self.height, self.width, 4), dtype=np.uint8)
        self._ck(self._L.rtDisplayMean(self._h, out.ctypes.data_as(C.c_void_p), out.nbytes))
        return out

    def trace_rays(self, rays, dirs=None, no_cull: bool = False) -> np.ndarray:
        """rtTraceRays: the closest hit of every ray against the current scene, as the path tracer computes it.  rays: a RAY_DTYPE
        array, or (n, 3) origins with (n, 3) directions in `dirs`.  Returns n RAY_HIT_DTYPE records (dst = inf, kind = RT_HIT_NONE,
        index = -1 on a miss).  no_cull: back faces count for every model (forceDontCullBack)."""
        r = make_rays(rays, dirs)
        hits = np.empty(r.shape[0], dtype=RAY_HIT_DTYPE)
        self._ck(self._L.rtTraceRays(self._h, r.ctypes.data if r.size else None, int(r.shape[0]), hits.ctypes.data if hits.size else None,
                                     RT_TRACE_NO_CULL if no_cull else 0))
        return hits

    def trace_rays_device(self, rays_ptr: int, hits_ptr: int, n: int, no_cull: bool = False):
        """rtTraceRaysDevice: n RtRay at rays_ptr -> n RtRayHit at hits_ptr (16-byte aligned), both device memory of the context's GPU
        (e.g. torch CUDA tensors' data_ptr()).  Asynchronous on the context's stream (set_stream)."""
        self._ck(self._L.rtTraceRaysDevice(self._h, C.c_void_p(rays_ptr), C.c_void_p(hits_ptr), int(n), RT_TRACE_NO_CULL if no_cull else 0))

    def trace_occlusion(self, segs, no_cull: bool = False) -> np.ndarray:
        """rtTraceOcclusion: for every segment (a SEGMENT_DTYPE array, see make_segments), whether anything lies on it — a hit with
        dst < tMax as the path tracer computes it.  Returns n bools.  no_cull: back faces count for every model (forceDontCullBack)."""
        s = make_segments(segs)
        occ = np.empty(s.shape[0], dtype=np.uint8)
        self._ck(self._L.rtTraceOcclusion(self._h, s.ctypes.data if s.size else None, int(s.shape[0]), occ.ctypes.data if occ.size else None,
                                          RT_TRACE_NO_CULL if no_cull else 0))
        return occ.view(np.bool_)

    def trace_occlusion_device(self, segs_ptr: int, occluded_ptr: int, n: int, no_cull: bool = False):
        """rtTraceOcclusionDevice: n RtRaySegment at segs_ptr (4-byte aligned) -> n bytes (1 = occluded) at occluded_ptr, both device
        memory of the context's GPU (e.g. torch CUDA tensors' data_ptr()).  Asynchronous on the context's stream (set_stream)."""
        self._ck(self._L.rtTraceOcclusionDevice(self._h, C.c_void_p(segs_ptr), C.c_void_p(occluded_ptr), int(n), RT_TRACE_NO_CULL if no_cull else 0))

    def trace_paths(self, rays, samples: int = 1) -> np.ndarray:
        """rtTracePaths: the path tracer's radiance along every ray (a PATH_RAY_DTYPE array, see make_path_rays), the mean of `samples`
        paths on the ray's RNG chain.  Returns n PATH_RADIANCE_DTYPE records: rgb and the RNG state after the last sample."""
        r = make_path_rays(rays)
        out = np.empty(r.shape[0], dtype=PATH_RADIANCE_DTYPE)
        self._ck(self._L.rtTracePaths(self._h, r.ctypes.data if r.size else None, int(r.shape[0]), int(samples), out.ctypes.data if out.size else None))
        return out

    def trace_paths_device(self, rays_ptr: int, out_ptr: int, n: int, samples: int = 1):
        """rtTracePathsDevice: n RtPathRay at rays_ptr (4-byte aligned) -> n RtPathRadiance at out_ptr (16-byte aligned), both device
        memory of the context's GPU (e.g. torch CUDA tensors' data_ptr()).  Asynchronous on the context's stream (set_stream)."""
        self._ck(self._L.rtTracePathsDevice(self._h, C.c_void_p(rays_ptr), C.c_void_p(out_ptr), int(n), int(samples)))

    def bake_probes(self, positions, samples: int, seed: int = 0):
        """rtBakeProbes: the L2 spherical harmonics of the radiance arriving at every probe position ((n, 3) floats) from `samples`
        spherical Fibonacci directions.  Returns (sh, rejected): (n, 3, 9) float32 as [probe][r, g, b][coefficient] in Unity's order,
        and (n,) uint32, the samples left out for a non-finite radiance."""
        pos = np.ascontiguousarray(np.asarray(positions, dtype=np.float32).reshape(-1, 3))
        out = np.empty(pos.shape[0], dtype=PROBE_SH_DTYPE)
        self._ck(self._L.rtBakeProbes(self._h, pos.ctypes.data if pos.size else None, int(pos.shape[0]), int(samples), int(seed) & 0xFFFFFFFF,
                                      out.ctypes.data if out.size else None))
        return out["sh"].copy(), out["rejected"].copy()

    def bake_probes_device(self, positions_ptr: int, out_ptr: int, n: int, samples: int, seed: int = 0):
        """rtBakeProbesDevice: n x 3 floats at positions_ptr (4-byte aligned) -> n RtProbeSH (PROBE_SH_DTYPE, 112 bytes) at out_ptr
        (16-byte aligned), both device memory of the context's GPU.  Asynchronous on the context's stream (set_stream)."""
        self._ck(self._L.rtBakeProbesDevice(self._h, C.c_void_p(positions_ptr), C.c_void_p(out_ptr), int(n), int(samples), int(seed) & 0xFFFFFFFF))

    def bake_cubemaps(self, positions, face_size: int, samples: int, seed: int = 0) -> np.ndarray:
        """rtBakeCubemaps: an HDR cube map of the radiance at every probe position ((n, 3) floats), each texel the mean of `samples`
        paths spread over its area.  Returns an (n, 6, N, N) CUBE_TEXEL_DTYPE array [probe][face +X, -X, +Y, -Y, +Z, -Z][row][column]
        (row 0 the top of the face): "rgb" the mean, "rejected" the samples left out for a non-finite radiance."""
        pos = np.ascontiguousarray(np.asarray(positions, dtype=np.float32).reshape(-1, 3))
        N = int(face_size)
        out = np.empty((pos.shape[0], 6, max(N, 0), max(N, 0)), dtype=CUBE_TEXEL_DTYPE)
        self._ck(self._L.rtBakeCubemaps(self._h, pos.ctypes.data if pos.size else None, int(pos.shape[0]), N, int(samples),
                                        int(seed) & 0xFFFFFFFF, out.ctypes.data if out.size else None))
        return out

    def bake_cubemaps_device(self, positions_ptr: int, out_ptr: int, n: int, face_size: int, samples: int, seed: int = 0):
        """rtBakeCubemapsDevice: n x 3 floats at positions_ptr (4-byte aligned) -> n * 6 * N^2 RtCubeTexel (CUBE_TEXEL_DTYPE, 16 bytes)
        at out_ptr (16-byte aligned), both device memory of the context's GPU.  Asynchronous on the context's stream (set_stream)."""
        self._ck(self._L.rtBakeCubemapsDevice(self._h, C.c_void_p(positions_ptr), C.c_void_p(out_ptr), int(n), int(face_size), int(samples),
                                              int(seed) & 0xFFFFFFFF))


    def bake_lightmap(self, points, samples: int, seed: int = 0) -> np.ndarray:
        """rtBakeLightmap: the cosine-weighted lighting arriving at every surface texel (an (n,) SURFACE_POINT_DTYPE array, or (n, 6) floats
        position then normal), each the mean of `samples` paths over the normal's hemisphere.  Returns an (n,) CUBE_TEXEL_DTYPE array:
        "rgb" estimates E / pi (a white Lambertian surface's radiance), "rejected" the samples left out for a non-finite radiance."""
        pts = as_surface_points(points)
        out = np.empty(pts.shape[0], dtype=CUBE_TEXEL_DTYPE)
        self._ck(self._L.rtBakeLightmap(self._h, pts.ctypes.data if pts.size else None, int(pts.shape[0]), int(samples),
                                        int(seed) & 0xFFFFFFFF, out.ctypes.data if out.size else None))
        return out

    def bake_lightmap_device(self, points_ptr: int, out_ptr: int, n: int, samples: int, seed: int = 0):
        """rtBakeLightmapDevice: n RtSurfacePoint (SURFACE_POINT_DTYPE, 24 bytes) at points_ptr (4-byte aligned) -> n RtCubeTexel
        (CUBE_TEXEL_DTYPE, 16 bytes) at out_ptr (16-byte aligned), both device memory of the context's GPU.  Asynchronous on the
        context's stream (set_stream)."""
        self._ck(self._L.rtBakeLightmapDevice(self._h, C.c_void_p(points_ptr), C.c_void_p(out_ptr), int(n), int(samples), int(seed) & 0xFFFFFFFF))

    def dispatch_features(self, gx: Optional[int] = None, gy: Optional[int] = None, gz: int = 1):
        """rtDispatchFeatures: the first-hit feature images (albedo, dst, normal, object id) of every pixel's own camera ray of the
        current "Frame", into "FeatureFrame" and, with "accumulate", the two accumulators.  Groups default to the whole image.  Read
        with readback("FeatureFrame") -> (H, W) PIXEL_FEATURES_DTYPE, readback("AccumulatedAlbedo" / "AccumulatedNormal")."""
        gx = (self.width + 7) // 8 if gx is None else gx
        gy = (self.height + 7) // 8 if gy is None else gy
        self._ck(self._L.rtDispatchFeatures(self._h, int(gx), int(gy), int(gz)))

    def camera_rays(self) -> np.ndarray:
        """rtCameraRays: (H, W) PATH_RAY_DTYPE, row 0 = bottom: every pixel's jittered camera ray for the current "Frame" / "renderSeed"
        and the RNG state after its four draws: what trace_paths takes, and trace_rays in origin / dir."""
        out = np.empty((self.height, self.width), dtype=PATH_RAY_DTYPE)
        self._ck(self._L.rtCameraRays(self._h, out.ctypes.data_as(C.c_void_p), out.nbytes))
        return out

    def camera_rays_device(self, rays_ptr: int, nbytes: int):
        """rtCameraRaysDevice: the same W*H RtPathRay into device memory of the context's GPU (4-byte aligned, nbytes = W*H*28).
        Asynchronous on the context's stream (set_stream)."""
        self._ck(self._L.rtCameraRaysDevice(self._h, C.c_void_p(rays_ptr), int(nbytes)))

    def denoise(self, use_accumulated: bool = True, iterations: int = DENOISE_ITERATIONS, sigma_colour: float = DENOISE_SIGMA_COLOUR,
                sigma_normal: float = DENOISE_SIGMA_NORMAL, sigma_depth: float = DENOISE_SIGMA_DEPTH):
        """rtDenoise: the a-trous filter of the accumulated mean (or of FrameRender) guided by the feature images, into
        "DenoisedRender" (readback("DenoisedRender") -> (H, W, 4) float32, the denoised mean colour, w = 1).  Asynchronous on the
        context's stream."""
        self._ck(self._L.rtDenoise(self._h, 1 if use_accumulated else 0, int(iterations), float(sigma_colour), float(sigma_normal),
                                   float(sigma_depth)))

    def denoise_temporal(self, iterations: int = TEMPORAL_ITERATIONS, sigma_luminance: float = TEMPORAL_SIGMA_LUMINANCE,
                         sigma_normal: float = TEMPORAL_SIGMA_NORMAL, sigma_depth: float = TEMPORAL_SIGMA_DEPTH, alpha: float = TEMPORAL_ALPHA,
                         reset_history: bool = False):
        """rtDenoiseTemporal: FrameRender filtered with its reprojected history (SVGF), guided by the feature images, into
        "DenoisedRender"; the motion vectors, history lengths and variances into "TemporalFrame" (temporal_frame()).  Asynchronous on
        the context's stream."""
        self._ck(self._L.rtDenoiseTemporal(self._h, int(iterations), float(sigma_luminance), float(sigma_normal), float(sigma_depth),
                                           float(alpha), 1 if reset_history else 0))

    def temporal_frame(self) -> np.ndarray:
        """"TemporalFrame": (H, W, 4) float32, row 0 = bottom, (prevX, prevY, history length, variance) per pixel."""
        return self.readback("TemporalFrame")

    def display_denoised(self) -> np.ndarray:
        """rtDisplayDenoised: DenoisedRender encoded as rtDisplay encodes (Frame = 1).  (H, W, 4) uint8, row 0 = bottom."""
        out = np.empty((self.height, self.width, 4), dtype=np.uint8)
        self._ck(self._L.rtDisplayDenoised(self._h, out.ctypes.data_as(C.c_void_p), out.nbytes))
        return out

    def readback(self, tex: str, out: Optional[np.ndarray] = None) -> np.ndarray:
        if out is None:
            out = (np.empty((self.height, self.width), dtype=PIXEL_FEATURES_DTYPE) if tex == "FeatureFrame" else
                   np.empty((self.height, self.width, 4), dtype=np.float32))
        self._ck(self._L.rtReadback(self._h, tex.encode(), out.ctypes.data_as(C.c_void_p), out.nbytes))
        return out

    def readback_into(self, tex: str, ptr: int, nbytes: int):
        self._ck(self._L.rtReadback(self._h, tex.encode(), C.c_void_p(ptr), nbytes))

    def display(self, use_accumulated: bool, frame: int) -> np.ndarray:
        """Display.shader: tex / Frame, encoded as the sRGB 8-bit back buffer.  Returns (H, W, 4) uint8, row 0 = bottom."""
        out = np.empty((self.height, self.width, 4), dtype=np.uint8)
        self._ck(self._L.rtDisplay(self._h, 1 if use_accumulated else 0, int(frame), out.ctypes.data_as(C.c_void_p), out.nbytes))
        return out

    def synchronize(self):
        self._ck(self._L.rtSynchronize(self._h))

    # -- extensions
    def set_stream(self, stream_ptr: int):
        self._ck(self._L.rtSetStream(self._h, C.c_void_p(stream_ptr)))

    def set_tile(self, rank: int, world: int, band_rows: int):
        self._ck(self._L.rtSetTile(self._h, rank, world, band_rows))

    def readback_async(self, tex: str, host_ptr: int, nbytes: int):
        """rtReadbackAsync into caller-owned (pinned) host memory; valid after readback_wait()."""
        self._ck(self._L.rtReadbackAsync(self._h, tex.encode(), C.c_void_p(host_ptr), nbytes))

    def display_async(self, use_accumulated: bool, frame: int, host_ptr: int, nbytes: int):
        self._ck(self._L.rtDisplayAsync(self._h, 1 if use_accumulated else 0, int(frame), C.c_void_p(host_ptr), nbytes))

    def readback_wait(self):
        self._ck(self._L.rtReadbackWait(self._h))

    def comm_init(self, unique_id: bytes, rank: int, world: int):
        """rtCommInit (collective over all ranks): NCCL communicator inside the context; RayTrace dispatches then end with the
        all-gather of the frame's tiles, and the context renders tile `rank` of `world`."""
        assert len(unique_id) == 128
        self._ck(self._L.rtCommInit(self._h, unique_id, 128, rank, world))

    def comm_destroy(self):
        self._ck(self._L.rtCommDestroy(self._h))

    def exchange_tiles(self):
        self._ck(self._L.rtExchangeTiles(self._h))

    def pack_tile(self):
        self._ck(self._L.rtPackTile(self._h))

    def unpack_tiles(self):
        self._ck(self._L.rtUnpackTiles(self._h))

    def device_pointer(self, name: str) -> tuple[int, int]:
        p, n = C.c_void_p(), C.c_size_t()
        self._ck(self._L.rtGetDevicePointer(self._h, name.encode(), C.byref(p), C.byref(n)))
        return int(p.value), int(n.value)

    def ipc_handles(self) -> bytes:
        buf = C.create_string_buffer(144)
        self._ck(self._L.rtGetIpcHandles(self._h, buf, 144))
        return buf.raw

    def set_peers(self, handles: list):
        """handles: one 144-byte blob (ipc_handles()) per peer rank."""
        blob = b"".join(handles)
        self._ck(self._L.rtSetPeers(self._h, len(handles), blob if handles else None, len(blob)))

    def build_bvh(self, vertices, indices, normals, quality: int = 1):
        """rtBuildBVH: BVH(verts, indices, normals, quality) of the reference (BVH.cs:26), built by the backend -> (triangles, nodes)."""
        v = np.ascontiguousarray(vertices, dtype=np.float32).reshape(-1, 3)
        n = np.ascontiguousarray(normals, dtype=np.float32).reshape(-1, 3)
        idx = np.ascontiguousarray(indices, dtype=np.int32).reshape(-1)
        ntri = idx.size // 3
        tris = np.empty(max(ntri, 1), dtype=TRIANGLE_DTYPE)
        nodes = np.empty(2 * max(ntri, 1) + 1, dtype=NODE_DTYPE)
        count = C.c_int()
        self._ck(self._L.rtBuildBVH(self._h, v.ctypes.data, v.shape[0], idx.ctypes.data, idx.size, n.ctypes.data, int(quality),
                                    tris.ctypes.data, nodes.ctypes.data, nodes.shape[0], C.byref(count)))
        return tris[:ntri], nodes[:count.value]

    def set_option(self, name: str, v: int):
        self._ck(self._L.rtSetOption(self._h, name.encode(), int(v)))

    def stats(self) -> dict:
        s = RtStats()
        self._ck(self._L.rtGetStats(self._h, C.byref(s)))
        return {k: getattr(s, k) for k, _ in RtStats._fields_}

    def reset_stats(self):
        """rtResetStats: zeroes RtStats and the PixelStats image."""
        self._ck(self._L.rtResetStats(self._h))

    def pixel_stats(self) -> np.ndarray:
        """rtReadbackPixelStats: (H, W) array of PIXEL_STATS_DTYPE, row 0 = bottom — each pixel's counts over the counting
        dispatches ("countStats" = 1) since the last reset_stats()."""
        out = np.empty((self.height, self.width), dtype=PIXEL_STATS_DTYPE)
        self._ck(self._L.rtReadbackPixelStats(self._h, out.ctypes.data_as(C.c_void_p), out.nbytes))
        return out

    def display_pixel_stats(self, vis_mode: int, debug_vis_scale: float) -> np.ndarray:
        """rtDisplayPixelStats: heat map of the PixelStats image as (H, W, 4) uint8, row 0 = bottom (VIS_MODES; values above
        debug_vis_scale are red)."""
        out = np.empty((self.height, self.width, 4), dtype=np.uint8)
        self._ck(self._L.rtDisplayPixelStats(self._h, int(vis_mode), float(debug_vis_scale), out.ctypes.data_as(C.c_void_p), out.nbytes))
        return out
