"""Python face of the C++ host (librt_host.so): the BVH builder and the RayComputeManager mirror.

`RayComputeManager` keeps the reference's public surface (Assets/Scripts/Tracer/RayComputeManager.cs:9-95):
the inspector fields by the same names, `ResetAccumulatedRender()`, `RenderFrame()`, and the two render
textures (`raytraceFrameTex`, `accumulatedResult`) as readbacks.  The work is done by the C++ class of the
same name in host/RayComputeManager.cpp, which drives the C-ABI (include/rt_b200.h).
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional, Sequence

import numpy as np

from . import capi
from .capi import MATERIAL_DTYPE, NODE_DTYPE, SPHERE_DTYPE, TRIANGLE_DTYPE

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
HOST_LIB = os.path.join(PKG_DIR, "librt_host.so")

QUALITY = {"Low": 0, "High": 1, "Disabled": 2}

_host = None


def host_lib() -> C.CDLL:
    global _host
    if _host is None:
        if not os.path.exists(HOST_LIB):
            raise FileNotFoundError(f"{HOST_LIB} not found — run `python -m ray_tracing_b200.build`")
        L = C.CDLL(HOST_LIB)
        vp, cp, ci, cf = C.c_void_p, C.c_char_p, C.c_int, C.c_float
        L.rthBuildBVH.argtypes = [vp, ci, vp, ci, vp, ci, vp, vp, ci, vp]
        L.rthBuildBVH.restype = ci
        L.rthLastError.restype = cp
        L.rthObjLoad.argtypes = [cp, ci, C.POINTER(ci), C.POINTER(ci)]
        L.rthObjCopy.argtypes = [vp, vp, vp]
        L.rthObjLastError.restype = cp
        L.rcmCreate.argtypes = [cp, ci, C.POINTER(vp)]
        L.rcmCreateMulti.argtypes = [cp, C.POINTER(ci), ci, C.POINTER(vp)]
        L.rcmDestroy.argtypes = [vp]
        L.rcmLastError.argtypes = [vp]
        L.rcmLastError.restype = cp
        L.rcmContext.argtypes = [vp]
        L.rcmContext.restype = vp
        L.rcmSetInt.argtypes = [vp, cp, ci]
        L.rcmGetInt.argtypes = [vp, cp, C.POINTER(ci)]
        L.rcmSetFloat.argtypes = [vp, cp, cf]
        L.rcmSetSun.argtypes = [vp, vp, vp]
        L.rcmSetScreen.argtypes = [vp, ci, ci]
        L.rcmSetCamera.argtypes = [vp, cf, vp]
        L.rcmAddMesh.argtypes = [vp, vp, ci, vp, ci, vp]
        L.rcmAddModel.argtypes = [vp, ci, vp, vp, vp]
        L.rcmSetModelTransform.argtypes = [vp, ci, vp, vp]
        L.rcmSetModelMaterial.argtypes = [vp, ci, vp]
        L.rcmSetSpheres.argtypes = [vp, vp, ci]
        for n in ("rcmOnEnable", "rcmResetAccumulatedRender", "rcmRenderFrame"):
            getattr(L, n).argtypes = [vp]
        L.rcmRenderFrames.argtypes = [vp, ci]
        L.rcmRenderFrameAdaptive.argtypes = [vp, cf, ci, ci, C.POINTER(C.c_int64)]
        L.rcmDisplayMean.argtypes = [vp, vp, C.c_size_t]
        L.rcmReadFrame.argtypes = [vp, vp, C.c_size_t]
        L.rcmReadAccumulated.argtypes = [vp, vp, C.c_size_t]
        L.rcmGetBVHStats.argtypes = [vp, vp, ci]
        L.rcmReadPixelStats.argtypes = [vp, vp, C.c_size_t]
        L.rcmDisplayDebugView.argtypes = [vp, ci, cf, vp, C.c_size_t]
        L.rcmTraceRays.argtypes = [vp, vp, ci, vp, ci]
        L.rcmTraceOcclusion.argtypes = [vp, vp, ci, vp, ci]
        L.rcmTracePaths.argtypes = [vp, vp, ci, ci, vp]
        L.rcmBakeProbes.argtypes = [vp, vp, ci, ci, C.c_uint32, vp]
        L.rcmBakeCubemaps.argtypes = [vp, vp, ci, ci, ci, C.c_uint32, vp]
        L.rcmBakeLightmap.argtypes = [vp, vp, ci, ci, C.c_uint32, vp]
        L.rcmRenderFeatures.argtypes = [vp]
        L.rcmReadFeatureImage.argtypes = [vp, cp, vp, C.c_size_t]
        L.rcmCameraRays.argtypes = [vp, vp, C.c_size_t]
        L.rcmDenoise.argtypes = [vp, ci, cf, cf, cf]
        L.rcmReadDenoised.argtypes = [vp, vp, C.c_size_t]
        L.rcmDenoiseTemporal.argtypes = [vp, ci, cf, cf, cf, cf, ci]
        L.rcmPick.argtypes = [vp, cf, cf, vp, vp]
        _host = L
    return _host


STAT_NAMES = ("TimeMs", "TriangleCount", "TotalNodeCount", "LeafNodeCount", "LeafDepthMin", "LeafDepthMax",
              "LeafDepthSum", "LeafMinTriCount", "LeafMaxTriCount")


def build_bvh(vertices: np.ndarray, indices: np.ndarray, normals: np.ndarray, quality: str | int = "High"):
    """BVH(verts, indices, normals, quality) of the reference (BVH.cs:26).  Returns (triangles, nodes, stats)."""
    L = host_lib()
    v = np.ascontiguousarray(vertices, dtype=np.float32).reshape(-1, 3)
    n = np.ascontiguousarray(normals, dtype=np.float32).reshape(-1, 3)
    idx = np.ascontiguousarray(indices, dtype=np.int32).reshape(-1)
    ntri = idx.size // 3
    tris = np.zeros(max(ntri, 1), dtype=TRIANGLE_DTYPE)
    nodes = np.zeros(2 * max(ntri, 1) + 1, dtype=NODE_DTYPE)
    stats = np.zeros(9, dtype=np.int32)
    q = QUALITY[quality] if isinstance(quality, str) else int(quality)
    rc = L.rthBuildBVH(v.ctypes.data, v.shape[0], idx.ctypes.data, idx.size, n.ctypes.data, q,
                       tris.ctypes.data, nodes.ctypes.data, nodes.shape[0], stats.ctypes.data)
    if rc < 0:
        raise ValueError("rthBuildBVH: " + L.rthLastError().decode())
    return tris[:ntri].copy(), nodes[:rc].copy(), dict(zip(STAT_NAMES, (int(s) for s in stats)))


def set_build_threads(threads: int) -> int:
    """Host threads a BVH build may use (0 = all, 1 = single-threaded like the reference); the result does not depend on it."""
    return int(host_lib().rthSetBuildThreads(int(threads)))


def load_obj(path: str, unity_handedness: bool = True):
    """Wavefront OBJ -> (vertices (n,3) f32, indices (3t,) i32, normals (n,3) f32) as Unity's importer hands them to the
    reference's manager (host/ObjLoader.cpp)."""
    L = host_lib()
    nv, ni = C.c_int(), C.c_int()
    if L.rthObjLoad(path.encode(), 1 if unity_handedness else 0, C.byref(nv), C.byref(ni)) != 0:
        raise ValueError("load_obj: " + L.rthObjLastError().decode())
    v = np.empty((nv.value, 3), dtype=np.float32)
    n = np.empty((nv.value, 3), dtype=np.float32)
    idx = np.empty(ni.value, dtype=np.int32)
    L.rthObjCopy(v.ctypes.data, n.ctypes.data, idx.ctypes.data)
    return v, idx, n


def column_major(m) -> np.ndarray:
    """4x4 (row, col) matrix -> 16 floats in Unity Matrix4x4 memory order."""
    return np.ascontiguousarray(np.asarray(m, dtype=np.float32).reshape(4, 4).T).reshape(16)


def vertex_texels(vertices, normals, local_to_world) -> np.ndarray:
    """One lightmap texel (capi.SURFACE_POINT_DTYPE) per vertex of a mesh placed by local_to_world (4x4, row, col): position
    (M [v, 1]).xyz and normal normalize(M3x3 n), the shading normal of HL:367, each row summed left to right in binary32.  For meshes
    without lightmap UVs (the reference's have none) this bakes vertex lighting; one texel per shared vertex leaves no seams."""
    f = np.float32
    M = np.asarray(local_to_world, dtype=f).reshape(4, 4)
    v = np.asarray(vertices, dtype=f).reshape(-1, 3)
    n = np.asarray(normals, dtype=f).reshape(-1, 3)
    out = np.zeros(len(v), dtype=capi.SURFACE_POINT_DTYPE)
    for r in range(3):
        out["position"][:, r] = (((M[r, 0] * v[:, 0] + M[r, 1] * v[:, 1]) + M[r, 2] * v[:, 2]) + M[r, 3]).astype(f)
        out["normal"][:, r] = ((M[r, 0] * n[:, 0] + M[r, 1] * n[:, 1]) + M[r, 2] * n[:, 2]).astype(f)
    w = out["normal"]
    out["normal"] = w * (f(1) / np.sqrt(((w[:, 0] * w[:, 0] + w[:, 1] * w[:, 1]) + w[:, 2] * w[:, 2]).astype(f)))[:, None]
    return out


class RayComputeManager:
    """Mirror of the reference's RayComputeManager (public fields + ResetAccumulatedRender / RenderFrame)."""

    _INT_FIELDS = ("maxBounceCount", "numRaysPerPixel", "renderSeed", "numAccumulatedFrames", "bvhQuality",
                   "rayTracingEnabled", "accumulate", "useSky", "randomizeSeedOnEnable", "buildBVHOnDevice")
    _FLOAT_FIELDS = ("defocusStrength", "divergeStrength", "focusDistance", "sunFocus", "sunIntensity")

    def __init__(self, backend_library: Optional[str] = None, device: int = 0, devices: Optional[Sequence[int]] = None):
        """device: the CUDA ordinal to render on; devices: several GPUs of this process behind ONE manager (rtCreateMulti: the
        image is row-tiled over them and every RenderFrame ends with one NCCL all-gather of the frame's tiles)."""
        object.__setattr__(self, "_h", None)
        L = host_lib()
        lib_path = backend_library or capi.DEFAULT_LIB
        if not os.path.exists(lib_path):
            raise FileNotFoundError(f"{lib_path} not found (librt_b200 is CUDA-only; there is no CPU fallback)")
        h = C.c_void_p()
        if devices is not None:
            arr = (C.c_int * len(devices))(*[int(d) for d in devices])
            rc = L.rcmCreateMulti(lib_path.encode(), arr, len(devices), C.byref(h))
        else:
            rc = L.rcmCreate(lib_path.encode(), device, C.byref(h))
        if rc != 0:
            raise capi.RtError(rc, L.rcmLastError(None).decode())
        object.__setattr__(self, "_L", L)
        object.__setattr__(self, "_h", h)
        object.__setattr__(self, "_lib", capi.RtLib(lib_path))
        object.__setattr__(self, "_size", (0, 0))
        object.__setattr__(self, "_floats", {})

    # -- field access by the reference's names
    def __setattr__(self, name, value):
        if name in self._INT_FIELDS:
            if name == "bvhQuality" and isinstance(value, str):
                value = QUALITY[value]
            self._ck(self._L.rcmSetInt(self._h, name.encode(), int(value)))
        elif name in self._FLOAT_FIELDS:
            self._floats[name] = float(value)
            self._ck(self._L.rcmSetFloat(self._h, name.encode(), float(value)))
        else:
            object.__setattr__(self, name, value)

    def __getattr__(self, name):
        if name in RayComputeManager._INT_FIELDS:
            v = C.c_int()
            self._ck(self._L.rcmGetInt(self._h, name.encode(), C.byref(v)))
            return v.value
        if name in RayComputeManager._FLOAT_FIELDS:
            return self._floats.get(name)
        raise AttributeError(name)

    def _ck(self, rc: int):
        if rc != 0:
            raise capi.RtError(rc, self._L.rcmLastError(self._h).decode())

    # -- scene set-up (what Unity's scene graph provides in the reference)
    def set_screen(self, width: int, height: int):
        self._ck(self._L.rcmSetScreen(self._h, width, height))
        object.__setattr__(self, "_size", (width, height))

    def set_camera(self, field_of_view: float, local_to_world):
        m = column_major(local_to_world)
        self._ck(self._L.rcmSetCamera(self._h, float(field_of_view), m.ctypes.data))

    def set_sun(self, color=(1, 1, 1, 1), forward: Optional[Sequence[float]] = None):
        c = np.asarray(color, dtype=np.float32)
        f = np.asarray(forward, dtype=np.float32) if forward is not None else None
        self._ck(self._L.rcmSetSun(self._h, c.ctypes.data, f.ctypes.data if f is not None else None))

    def add_mesh(self, vertices, indices, normals) -> int:
        v = np.ascontiguousarray(vertices, dtype=np.float32).reshape(-1, 3)
        n = np.ascontiguousarray(normals, dtype=np.float32).reshape(-1, 3)
        idx = np.ascontiguousarray(indices, dtype=np.int32).reshape(-1)
        rc = self._L.rcmAddMesh(self._h, v.ctypes.data, v.shape[0], idx.ctypes.data, idx.size, n.ctypes.data)
        if rc < 0:
            self._ck(rc)
        return rc

    def add_model(self, mesh_id: int, local_to_world, world_to_local, material: np.ndarray) -> int:
        a, b = column_major(local_to_world), column_major(world_to_local)
        mat = np.ascontiguousarray(material, dtype=MATERIAL_DTYPE).reshape(1)
        rc = self._L.rcmAddModel(self._h, mesh_id, a.ctypes.data, b.ctypes.data, mat.ctypes.data)
        if rc < 0:
            self._ck(rc)
        return rc

    def set_model_transform(self, model: int, local_to_world, world_to_local):
        a, b = column_major(local_to_world), column_major(world_to_local)
        self._ck(self._L.rcmSetModelTransform(self._h, model, a.ctypes.data, b.ctypes.data))

    def set_model_material(self, model: int, material: np.ndarray):
        mat = np.ascontiguousarray(material, dtype=MATERIAL_DTYPE).reshape(1)
        self._ck(self._L.rcmSetModelMaterial(self._h, model, mat.ctypes.data))

    def set_spheres(self, spheres: np.ndarray):
        s = np.ascontiguousarray(spheres, dtype=SPHERE_DTYPE)
        self._ck(self._L.rcmSetSpheres(self._h, s.ctypes.data if s.size else None, int(s.shape[0])))

    # -- the reference's methods
    def OnEnable(self):
        self._ck(self._L.rcmOnEnable(self._h))

    def ResetAccumulatedRender(self):
        self._ck(self._L.rcmResetAccumulatedRender(self._h))

    def RenderFrame(self):
        self._ck(self._L.rcmRenderFrame(self._h))

    Update = RenderFrame

    def RenderFrames(self, n: int):
        """n RenderFrame() calls of a still image as one batch (rtDispatchFrames): the same images, numAccumulatedFrames += n.
        With accumulate off it is n RenderFrame() calls."""
        self._ck(self._L.rcmRenderFrames(self._h, int(n)))

    def RenderFrameAdaptive(self, threshold: float = capi.ADAPTIVE_THRESHOLD, min_frames: int = capi.ADAPTIVE_MIN_FRAMES,
                            max_frames: int = capi.ADAPTIVE_MAX_FRAMES) -> int:
        """The next frame only where the estimated error is still above `threshold` (rtDispatchAdaptive over the whole image): the
        upload sequence and InitFrame of RenderFrame, then numAccumulatedFrames += 1.  Returns the number of pixels traced (0 =
        converged).  Needs accumulate.  Show the result with mean_result / display_mean (each pixel has its own frame count)."""
        active = C.c_int64(0)
        self._ck(self._L.rcmRenderFrameAdaptive(self._h, float(threshold), int(min_frames), int(max_frames), C.byref(active)))
        return int(active.value)

    def OnDestroy(self):
        if self._h:
            self._L.rcmDestroy(self._h)
            object.__setattr__(self, "_h", None)

    def __del__(self):
        try:
            self.OnDestroy()
        except Exception:
            pass

    # -- render textures
    def _read(self, fn, out):
        w, h = self._size
        if out is None:
            out = np.empty((h, w, 4), dtype=np.float32)
        self._ck(fn(self._h, out.ctypes.data, out.nbytes))
        return out

    @property
    def raytraceFrameTex(self) -> np.ndarray:
        return self._read(self._L.rcmReadFrame, None)

    @property
    def accumulatedResult(self) -> np.ndarray:
        return self._read(self._L.rcmReadAccumulated, None)

    @property
    def mean_result(self) -> np.ndarray:
        """(H, W, 4) float32, row 0 = bottom: the per-pixel mean accumulatedResult / accumulatedResult.w (0 where nothing was
        accumulated) — the image of an adaptively sampled render, whose pixels have different frame counts."""
        a = self.accumulatedResult
        w = a[..., 3:4]
        with np.errstate(divide="ignore", invalid="ignore"):
            return np.where(w != 0, a / np.where(w != 0, w, 1), np.float32(0)).astype(np.float32)

    def display_mean(self) -> np.ndarray:
        """rtDisplayMean: the per-pixel mean encoded as the display encodes, (0, 0, 0, 255) where nothing was accumulated.
        (H, W, 4) uint8, row 0 = bottom."""
        w, h = self._size
        out = np.empty((h, w, 4), dtype=np.uint8)
        self._ck(self._L.rcmDisplayMean(self._h, out.ctypes.data, out.nbytes))
        return out

    def read_accumulated_into(self, ptr: int, nbytes: int):
        self._ck(self._L.rcmReadAccumulated(self._h, C.c_void_p(ptr), nbytes))

    # -- the reference's debug view (visMode / debugVisScale, RayCommon.hlsl:24-26): per-pixel cost of the counting launches
    def pixel_stats(self) -> np.ndarray:
        """(H, W) array of capi.PIXEL_STATS_DTYPE, row 0 = bottom: each pixel's rays, box / triangle / sphere tests over the frames
        rendered with context.set_option("countStats", 1) since the last context.reset_stats()."""
        w, h = self._size
        out = np.empty((h, w), dtype=capi.PIXEL_STATS_DTYPE)
        self._ck(self._L.rcmReadPixelStats(self._h, out.ctypes.data, out.nbytes))
        return out

    def debug_view(self, visMode: int, debugVisScale: float) -> np.ndarray:
        """Heat map of pixel_stats() as (H, W, 4) uint8, row 0 = bottom.  visMode 1: box tests per ray, 2: triangle tests per ray,
        3: sphere tests per ray, 4: rays per pixel; debugVisScale is shown as white, anything above it as red."""
        w, h = self._size
        out = np.empty((h, w, 4), dtype=np.uint8)
        self._ck(self._L.rcmDisplayDebugView(self._h, int(visMode), float(debugVisScale), out.ctypes.data, out.nbytes))
        return out

    # -- closest-hit queries against the current scene (rtTraceRays): picking, autofocus, line of sight
    def trace_rays(self, rays, dirs=None, no_cull: bool = False) -> np.ndarray:
        """The closest hit of every ray (capi.RAY_DTYPE array, or (n, 3) origins with (n, 3) dirs) as n capi.RAY_HIT_DTYPE records.
        The scene is uploaded as a frame would upload it; the render textures are not touched."""
        r = capi.make_rays(rays, dirs)
        hits = np.empty(r.shape[0], dtype=capi.RAY_HIT_DTYPE)
        self._ck(self._L.rcmTraceRays(self._h, r.ctypes.data if r.size else None, int(r.shape[0]), hits.ctypes.data if hits.size else None,
                                      capi.RT_TRACE_NO_CULL if no_cull else 0))
        return hits

    # -- occlusion queries (rtTraceOcclusion): shadow and ambient-occlusion rays, line of sight
    def trace_occlusion(self, segs, no_cull: bool = False) -> np.ndarray:
        """Whether anything lies on each segment (a capi.SEGMENT_DTYPE array, see capi.make_segments) as n bools.  The scene is
        uploaded as a frame would upload it; the render textures are not touched."""
        s = capi.make_segments(segs)
        occ = np.empty(s.shape[0], dtype=np.uint8)
        self._ck(self._L.rcmTraceOcclusion(self._h, s.ctypes.data if s.size else None, int(s.shape[0]), occ.ctypes.data if occ.size else None,
                                           capi.RT_TRACE_NO_CULL if no_cull else 0))
        return occ.view(np.bool_)

    # -- radiance along caller rays (rtTracePaths): custom cameras, probe baking
    def trace_paths(self, rays, samples: int = 1) -> np.ndarray:
        """The path tracer's radiance along each ray (a capi.PATH_RAY_DTYPE array, see capi.make_path_rays), the mean of `samples`
        paths, as n capi.PATH_RADIANCE_DTYPE records.  The scene is uploaded as a frame would upload it; the render textures are not
        touched."""
        r = capi.make_path_rays(rays)
        out = np.empty(r.shape[0], dtype=capi.PATH_RADIANCE_DTYPE)
        self._ck(self._L.rcmTracePaths(self._h, r.ctypes.data if r.size else None, int(r.shape[0]), int(samples), out.ctypes.data if out.size else None))
        return out

    # -- light probes (rtBakeProbes): L2 spherical harmonics of the radiance at each position
    def bake_probes(self, positions, samples: int, seed: int = 0):
        """The L2 spherical harmonics of the radiance arriving at each probe position ((n, 3) floats) from `samples` spherical
        Fibonacci directions: ((n, 3, 9) float32 [probe][r, g, b][coefficient], (n,) uint32 rejected samples).  The scene is uploaded
        as a frame would upload it; the render textures are not touched."""
        pos = np.ascontiguousarray(np.asarray(positions, dtype=np.float32).reshape(-1, 3))
        out = np.empty(pos.shape[0], dtype=capi.PROBE_SH_DTYPE)
        self._ck(self._L.rcmBakeProbes(self._h, pos.ctypes.data if pos.size else None, int(pos.shape[0]), int(samples), int(seed) & 0xFFFFFFFF,
                                       out.ctypes.data if out.size else None))
        return out["sh"].copy(), out["rejected"].copy()

    # -- reflection probes (rtBakeCubemaps): an HDR cube map of the radiance at each position
    def bake_cubemaps(self, positions, face_size: int, samples: int, seed: int = 0) -> np.ndarray:
        """An HDR cube map of the radiance at each probe position ((n, 3) floats), each texel the mean of `samples` paths over its
        area: (n, 6, N, N) capi.CUBE_TEXEL_DTYPE [probe][face +X, -X, +Y, -Y, +Z, -Z][row][column].  The scene is uploaded as a frame
        would upload it; the render textures are not touched."""
        pos = np.ascontiguousarray(np.asarray(positions, dtype=np.float32).reshape(-1, 3))
        N = int(face_size)
        out = np.empty((pos.shape[0], 6, max(N, 0), max(N, 0)), dtype=capi.CUBE_TEXEL_DTYPE)
        self._ck(self._L.rcmBakeCubemaps(self._h, pos.ctypes.data if pos.size else None, int(pos.shape[0]), N, int(samples),
                                         int(seed) & 0xFFFFFFFF, out.ctypes.data if out.size else None))
        return out


    # -- lightmaps (rtBakeLightmap): the cosine-weighted lighting at surface texels
    def bake_lightmap(self, points, samples: int, seed: int = 0) -> np.ndarray:
        """The lighting arriving at each surface texel (SURFACE_POINT_DTYPE records or (n, 6) floats, e.g. from vertex_texels), each
        the mean of `samples` paths over the normal's hemisphere: (n,) capi.CUBE_TEXEL_DTYPE, "rgb" an estimate of E / pi.  The scene is
        uploaded as a frame would upload it; the render textures are not touched."""
        pts = capi.as_surface_points(points)
        out = np.empty(pts.shape[0], dtype=capi.CUBE_TEXEL_DTYPE)
        self._ck(self._L.rcmBakeLightmap(self._h, pts.ctypes.data if pts.size else None, int(pts.shape[0]), int(samples),
                                         int(seed) & 0xFFFFFFFF, out.ctypes.data if out.size else None))
        return out

    # -- denoiser guides (rtDispatchFeatures) and the camera's own rays (rtCameraRays)
    def RenderFeatures(self):
        """The first-hit feature images of the frame the NEXT RenderFrame() renders: the upload sequence of RenderFrame, then
        rtDispatchFeatures over the whole image; the frame counter does not move.  Read them with feature_frame / accumulated_albedo /
        accumulated_normal; ResetAccumulatedRender resets the two accumulated ones with the colour."""
        self._ck(self._L.rcmRenderFeatures(self._h))

    def _read_feature(self, name: str, out: np.ndarray) -> np.ndarray:
        self._ck(self._L.rcmReadFeatureImage(self._h, name.encode(), out.ctypes.data, out.nbytes))
        return out

    @property
    def feature_frame(self) -> np.ndarray:
        """(H, W) array of capi.PIXEL_FEATURES_DTYPE, row 0 = bottom: albedo, dst, normal and object id of each pixel's feature ray."""
        w, h = self._size
        return self._read_feature("FeatureFrame", np.empty((h, w), dtype=capi.PIXEL_FEATURES_DTYPE))

    @property
    def accumulated_albedo(self) -> np.ndarray:
        """(H, W, 4) float32: the sum of (albedo, 1) over the feature rays that hit since the last reset."""
        w, h = self._size
        return self._read_feature("AccumulatedAlbedo", np.empty((h, w, 4), dtype=np.float32))

    @property
    def accumulated_normal(self) -> np.ndarray:
        """(H, W, 4) float32: the sum of (normal, dst) over the feature rays that hit since the last reset."""
        w, h = self._size
        return self._read_feature("AccumulatedNormal", np.empty((h, w, 4), dtype=np.float32))

    def camera_rays(self) -> np.ndarray:
        """(H, W) array of capi.PATH_RAY_DTYPE, row 0 = bottom: every pixel's jittered camera ray for the frame the next RenderFrame()
        renders and the RNG state after its four draws: what trace_paths and (origin, dir) trace_rays take."""
        w, h = self._size
        out = np.empty((h, w), dtype=capi.PATH_RAY_DTYPE)
        self._ck(self._L.rcmCameraRays(self._h, out.ctypes.data, out.nbytes))
        return out

    # -- the a-trous denoiser (rtDenoise)
    def Denoise(self, iterations: int = capi.DENOISE_ITERATIONS, sigma_colour: float = capi.DENOISE_SIGMA_COLOUR,
                sigma_normal: float = capi.DENOISE_SIGMA_NORMAL, sigma_depth: float = capi.DENOISE_SIGMA_DEPTH):
        """rtDenoise over the whole image, guided by the feature images RenderFeatures() left: the accumulated mean when accumulate is
        on, else the last frame.  Read the result with denoised_result."""
        self._ck(self._L.rcmDenoise(self._h, int(iterations), float(sigma_colour), float(sigma_normal), float(sigma_depth)))

    def DenoiseTemporal(self, iterations: int = capi.TEMPORAL_ITERATIONS, sigma_luminance: float = capi.TEMPORAL_SIGMA_LUMINANCE,
                        sigma_normal: float = capi.TEMPORAL_SIGMA_NORMAL, sigma_depth: float = capi.TEMPORAL_SIGMA_DEPTH,
                        alpha: float = capi.TEMPORAL_ALPHA, reset_history: bool = False):
        """rtDenoiseTemporal of the last frame with its reprojected history, for a moving camera: once per frame after RenderFeatures()
        and RenderFrame(); reset_history on a jump cut.  Read the result with denoised_result."""
        self._ck(self._L.rcmDenoiseTemporal(self._h, int(iterations), float(sigma_luminance), float(sigma_normal), float(sigma_depth),
                                            float(alpha), 1 if reset_history else 0))

    @property
    def denoised_result(self) -> np.ndarray:
        """(H, W, 4) float32, row 0 = bottom: "DenoisedRender", the denoised mean colour, w = 1."""
        w, h = self._size
        out = np.empty((h, w, 4), dtype=np.float32)
        self._ck(self._L.rcmReadDenoised(self._h, out.ctypes.data, out.nbytes))
        return out

    def pick_ray(self, x: float, y: float) -> np.ndarray:
        """The un-jittered camera ray through pixel (x, y) (row 0 = bottom), as one capi.RAY_DTYPE record."""
        ray = np.zeros(1, dtype=capi.RAY_DTYPE)
        self._ck(self._L.rcmPick(self._h, float(x), float(y), ray.ctypes.data, None))
        return ray[0]

    def pick(self, x: float, y: float) -> np.ndarray:
        """What lies under pixel (x, y): the closest hit of pick_ray(x, y), one capi.RAY_HIT_DTYPE record (kind / index name the
        Spheres or ModelInfo entry; dst is the distance along the unit-length ray, e.g. for focusDistance)."""
        hit = np.zeros(1, dtype=capi.RAY_HIT_DTYPE)
        self._ck(self._L.rcmPick(self._h, float(x), float(y), None, hit.ctypes.data))
        return hit[0]

    def bvh_stats(self) -> list[dict]:
        buf = np.zeros(9 * 64, dtype=np.int32)
        n = self._L.rcmGetBVHStats(self._h, buf.ctypes.data, 64)
        return [dict(zip(STAT_NAMES, (int(x) for x in buf[9 * i:9 * i + 9]))) for i in range(min(n, 64))]

    # -- the underlying C-ABI context (extensions: options, stats, tiles, streams)
    @property
    def context(self) -> capi.RtContext:
        ctx = capi.RtContext(self._lib, C.c_void_p(self._L.rcmContext(self._h)))
        ctx.destroy = lambda: None          # owned by the C++ manager
        ctx.width, ctx.height = self._size
        return ctx
