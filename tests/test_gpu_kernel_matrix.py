"""Every __global__ of librt_b200.so, one row each, bit-exact against the oracle on the H100 (`-m gpu`).

The library holds 129 kernels.  Which instantiation a call launches is decided in one place — with_persistent_kernel / with_camera_kernel
(rt_kernel_wave.cuh) pick <STATS, EXT, TLAS> and the form, wave_kernel / pool_kernel map that to a __global__ — and the shared-memory limit
of every kernel that rule can reach is set by wave_configure / pool_configure.  TABLE below names, for each kernel, the call that must
launch it and the options that force every choice that could otherwise depend on the device ("kernel", "poolSlots", "sampleChunks",
"tlas", "modelSkip", "countStats", "extInstantiation", "smemNodes"), on a scene in which that variant's own code runs:

  * EXT rows: 80 spheres (more than 64: the sphere accelerator) beside the meshes;
  * TLAS rows: the three models of the room with "tlas" = 1 and model skipping on; the counting rows use the same TLAS, so that a rule
    that moved counting onto the TLAS kernel would launch another kernel than the row's;
  * CHUNKED rows: "sampleChunks" = 2 with 2 samples per pixel; FRAMES rows: 2 frames, compared with 2 oracle rtDispatch calls;
  * LIST rows: an adaptive session whose last call leaves some pixels active and some converged;
  * every mesh scene has a glass knot and a checkered floor.

SMEM_ROWS add one row for every kernel-1 instantiation that can stage tree tops in shared memory (the EXT and TLAS ones, in all three
forms): a knot of 2,880 triangles and "smemNodes" = 3072 take the launch above the 48 KB of dynamic shared memory a kernel gets without
cudaFuncSetAttribute.  Kernel-2 launches are always above 48 KB (their pools alone are).  The non-EXT kernel-1 kernels stage nothing,
and the query family never stages tree tops (queryParams zeroes smemPairs), so neither can go above 48 KB.

On the H100 a launch above 48 KB that configure missed is refused, so a row's RT_OK is the check that configure reached its kernel.  The
CPU twin (tests/test_simt_kernel_matrix.py) runs the same rows on the SIMT interpreter, whose launch log also checks that each row's call
launched exactly its own camera or query kernel, and that the table's keys are the kernels of both builds."""
import collections
import ctypes as C

import numpy as np
import pytest

from conftest import CUDA_LIB, ORACLE_LIB, assert_bit_equal
import ray_tracing_b200 as rt
from ray_tracing_b200 import capi, scenes
import test_gpu_probes as PR
import test_gpu_trace_rays as T

W, H, SPP, BOUNCES = 24, 16, 2, 3
SMEM_DEFAULT = 48 * 1024                  # dynamic shared memory a kernel may use without cudaFuncSetAttribute
COUNTS = ("rays", "boxTests", "triTests", "sphereTests", "sphereBoxTests")
EXT_SPHERES = 80
ADAPTIVE_SESSION = ((0.2, 2, 8),) * 3      # every pixel twice (minFrames), then only those whose error is still above 0.2

pytestmark = pytest.mark.gpu

Row = collections.namedtuple("Row", "entry options scene family")


# ---- scenes -----------------------------------------------------------------------------------------------------------------------
def matrix_scene(ext=False, big=False):
    """The glass knot in the room with a checkered floor; ext: 80 small spheres in the room; big: a knot of 2,880 triangles, whose tree
    has enough pair records to fill more than 48 KB of shared memory."""
    sc = scenes.knot_room(W, H, BOUNCES, SPP, nu=120 if big else 40, nv=12 if big else 6, glass=True)
    sc.models[1] = scenes.ModelDesc(1, np.eye(4), np.eye(4), scenes.material(diffuse=(0.78, 0.78, 0.78), emission=(0.2, 0.3, 0.8),
                                                                           specularProbability=0.0, flag=scenes.MAT_CHECKER))
    if ext:
        rng = np.random.RandomState(3)
        sph = np.zeros(EXT_SPHERES, dtype=capi.SPHERE_DTYPE)
        sph["centre"] = rng.uniform((-2.4, 0.2, -2.0), (2.4, 3.6, 2.4), (EXT_SPHERES, 3))
        sph["radius"] = rng.uniform(0.05, 0.25, EXT_SPHERES)
        for i in range(EXT_SPHERES):
            sph[i]["material"] = (scenes.material(flag=scenes.MAT_GLASS, ior=1.4, smoothness=1.0) if i % 4 == 0 else
                                  scenes.material(diffuse=tuple(rng.uniform(0.2, 0.9, 3)), emission=(1, 1, 1), emissionStrength=float(i % 9 == 0)))
        sc.spheres = sph
        sc.name += "+spheres"
    sc.name += "+big" if big else ""
    return sc


# ---- the table --------------------------------------------------------------------------------------------------------------------
B = {False: "false", True: "true"}
VARIANTS = ((0, 0, 0), (0, 1, 0), (1, 0, 0), (1, 1, 0), (0, 1, 1))          # what with_persistent_kernel can choose: <STATS, EXT, TLAS>
FORM_ENTRY = {"": "dispatch", "_frames": "frames", "_list": "adaptive"}


def _variant_options(s, x, t):
    """countStats = STATS; a TLAS for the TLAS rows and the counting rows; EXT from the sphere accelerator (the scene's 80 spheres)."""
    return dict(countStats=s, tlas=1 if (t or s) else 0, modelSkip=1, extInstantiation=0, smemNodes=0), x or t


def _camera_row(entry, kernel, s, x, t, slots=64, chunks=1):
    opts, ext = _variant_options(s, x, t)
    opts.update(kernel=kernel, poolSlots=slots, sampleChunks=chunks)
    return Row(entry, opts, (ext, False), "camera")


def _build_table():
    table = {}
    for form, entry in FORM_ENTRY.items():
        table[f"k_raytrace_mega{form}" + ("<64u>" if form == "_list" else "")] = _camera_row(entry, 0, 0, 0, 0)
        for s, x, t in VARIANTS:
            for m in (32, 64, 96):
                name = f"k_raytrace_pool_tlas{form}<{m}>" if t else f"k_raytrace_pool{form}<{B[bool(s)]}, {B[bool(x)]}, {m}>"
                table[name] = _camera_row(entry, 2, s, x, t, slots=m)
            if form == "_list":
                name = f"k_raytrace_wave_list<{B[bool(s)]}, {B[bool(x)]}, {B[bool(t)]}>"
            elif t:
                name = f"k_raytrace_wave_tlas{form}"
            elif form == "_frames":
                name = f"k_raytrace_wave_frames<{B[bool(s)]}, {B[bool(x)]}>"
            else:
                name = f"k_raytrace_wave<{B[bool(s)]}, {B[bool(x)]}, false>"
            table[name] = _camera_row(entry, 1, s, x, t)
    for s in (0, 1):                                     # sample chunks: <STATS, true, true> (the TLAS kernel carries the hand-off itself)
        opts, _ = _variant_options(s, 1, 0)
        table[f"k_raytrace_wave<{B[bool(s)]}, true, true>"] = Row("dispatch", dict(opts, kernel=1, poolSlots=64, sampleChunks=2), (True, False), "camera")
    table["k_raytrace_wave_tlas"] = _camera_row("dispatch", 1, 0, 1, 1, chunks=2)     # and the TLAS kernel in chunks
    for q in ("k_trace_rays", "k_trace_occlusion", "k_trace_paths", "k_camera_features", "k_bake_probes", "k_bake_cubemaps"):
        entry = q[2:].replace("camera_", "")
        for s, x, t in VARIANTS:
            opts, ext = _variant_options(s, x, t)
            table[f"{q}<{B[bool(s)]}, {B[bool(x)]}, {B[bool(t)]}>"] = Row(entry, opts, (ext, False), "query")
    table["k_camera_rays"] = Row("camera_rays", {}, (False, False), "query")
    single = {"bvh": ("k_bvh_init", "k_bvh_root", "k_bvh_level_begin", "k_bvh_evaluate", "k_bvh_best", "k_bvh_decide", "k_bvh_flags", "k_scan_tiles",
                      "k_scan_sums", "k_scan_add", "k_bvh_partition", "k_bvh_finish_level", "k_bvh_sizes", "k_bvh_indices", "k_bvh_emit_nodes", "k_bvh_emit_tris"),
              "denoise": ("k_denoise_prepare", "k_denoise_pass"),
              "temporal": ("k_temporal_reproject", "k_temporal_variance", "k_temporal_prefilter", "k_temporal_pass"),
              "adaptive": ("k_adaptive_flags", "k_adaptive_scan", "k_adaptive_scatter"), "display_mean": ("k_mean_image",),
              "probes": ("k_probe_sums",), "cubemaps": ("k_cube_sums",), "dispatch": ("k_repack_tris",), "tiles": ("k_pack_tile", "k_unpack_tiles"),
              "display": ("k_display", "k_pixel_stats_display")}
    for entry, names in single.items():
        for name in names:
            table[name] = Row(entry, dict(kernel=2, countStats=1) if entry in ("adaptive", "dispatch", "display") else {}, (False, False), "single")
    return table


TABLE = _build_table()

# kernel 1's instantiations that can stage tree tops (EXT and TLAS, every form), each once more with its launch above 48 KB
SMEM_ROWS = {k: r._replace(options=dict(r.options, smemNodes=3072), scene=(r.scene[0], True))
             for k, r in TABLE.items() if r.family == "camera" and r.options["kernel"] == 1 and r.scene[0]}


# ---- one row's call ---------------------------------------------------------------------------------------------------------------
def _open(lib, sc, options):
    oracle = lib == ORACLE_LIB
    opts = {k: v for k, v in options.items() if k == "countStats"} if oracle else options      # the oracle has one walk, and counts
    mgr = T.open_mgr(lib, sc, opts)
    mgr.context.reset_stats()
    return mgr, mgr.context


def _stats(ctx, out, options, sc):
    st = ctx.stats()
    out["RtStats.rays"] = st["rays"]
    if options.get("countStats"):
        # with the sphere accelerator the sphere counters are the accelerator's own, not the reference's linear scan
        for k in COUNTS if len(sc.spheres) <= 64 else COUNTS[:3]:
            out[f"RtStats.{k}"] = st[k]


def _images(mgr, ctx, out, options, sc):
    out["FrameRender"], out["AccumulatedRender"] = mgr.raytraceFrameTex, mgr.accumulatedResult
    _stats(ctx, out, options, sc)
    if options.get("countStats"):
        pix = ctx.pixel_stats()
        for k in COUNTS if len(sc.spheres) <= 64 else COUNTS[:3]:
            out[f"PixelStats.{k}"] = np.ascontiguousarray(pix[k])


HOST_POINTERS = False                   # device pointers are host pointers (the SIMT interpreter build)


class _Dev:
    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "|u1", "data": (ptr, False), "version": 3, "strides": None}


def _read_device(ptr, nbytes):
    if HOST_POINTERS:
        return C.string_at(ptr, nbytes)
    import torch
    return torch.as_tensor(_Dev(ptr, nbytes), device="cuda:0").clone()


def _write_device(ptr, nbytes, parts):
    if HOST_POINTERS:
        blob = b"".join(parts)
        assert len(blob) == nbytes
        C.memmove(ptr, blob, nbytes)
        return
    import torch
    blob = torch.cat(parts)
    assert blob.numel() == nbytes
    torch.as_tensor(_Dev(ptr, nbytes), device="cuda:0").copy_(blob)
    torch.cuda.synchronize()


def run_row(lib, row):
    """The row's call on `lib` (the oracle runs the same call; frames rows: as one rtDispatch per frame): {buffer name: value}."""
    oracle = lib == ORACLE_LIB
    sc = matrix_scene(*row.scene)
    e, opts, out = row.entry, row.options, {}
    if e == "bvh":
        ctx = capi.RtLib(lib).create(0)
        m = scenes.knot_mesh(nu=60, nv=8)
        for q in (0, 1, 2):
            tris, nodes = ctx.build_bvh(m.vertices, m.indices, m.normals, q)
            out[f"Triangles q={q}"], out[f"Nodes q={q}"] = tris.view(np.uint8), nodes.view(np.uint8)
        ctx.destroy()
        return out
    if e == "tiles" and oracle:
        e = "dispatch"                      # the image the two ranks' tiles reassemble to: one context's frame
    elif e == "tiles":
        # two ranks of 8-row bands; rank 1's TileSend appended to rank 0's is what the all-gather delivers to rank 0
        mgrs, sends = [], []
        for r in range(2):
            mgr = rt.RayComputeManager(lib)
            scenes.apply(sc, mgr)
            mgr.context.set_tile(r, 2, 8)
            mgr.OnEnable(); mgr.RenderFrame()
            mgr.context.pack_tile(); mgr.context.synchronize()
            sends.append(_read_device(*mgr.context.device_pointer("TileSend")))
            mgrs.append(mgr)
        _write_device(*mgrs[0].context.device_pointer("TileRecv"), sends)
        mgrs[0].context.unpack_tiles(); mgrs[0].context.synchronize()
        out["FrameRender"], out["AccumulatedRender"] = mgrs[0].raytraceFrameTex, mgrs[0].accumulatedResult
        for mgr in mgrs:
            mgr.OnDestroy()
        return out
    mgr, ctx = _open(lib, sc, opts)
    if e == "dispatch":
        mgr.RenderFrame()
        _images(mgr, ctx, out, opts, sc)
        if row.entry == "tiles":
            del out["RtStats.rays"]         # (the ranks' counters are their own tiles')
    elif e == "frames":
        ctx.set_int("Frame", 1)
        if oracle:
            for f in (1, 2):
                ctx.set_int("Frame", f)
                ctx.dispatch_full()
            ctx.set_int("Frame", 1)
        else:
            ctx.dispatch_frames(2)
        _images(mgr, ctx, out, opts, sc)
    elif e in ("adaptive", "display_mean"):
        counts = []
        for f, (thr, mn, mx) in enumerate(ADAPTIVE_SESSION, start=1):
            ctx.set_int("Frame", f)
            counts.append(ctx.dispatch_adaptive(thr, mn, mx))
        if oracle:
            assert 0 < counts[-1] < W * H, f"the adaptive session must leave some pixels active and some converged: {counts}"
        out["active counts"] = np.array(counts)
        out["AdaptiveMoments"] = ctx.adaptive_moments()
        _images(mgr, ctx, out, opts, sc)
        if e == "display_mean":
            out["rtDisplayMean"] = ctx.display_mean()
    elif e == "display":
        mgr.RenderFrame()
        out["rtDisplay"] = ctx.display(True, 1)
        out["rtDisplayPixelStats"] = ctx.display_pixel_stats(1, 200.0)
    elif e in ("trace_rays", "trace_occlusion", "trace_paths"):
        rays = T.ray_sets(sc, seed=11, n=48)["mixed"]
        if e == "trace_rays":
            out["RtRayHit"] = ctx.trace_rays(rays)
        elif e == "trace_occlusion":
            tmax = np.random.RandomState(12).uniform(0.25, 8.0, len(rays)).astype(np.float32)
            out["occluded"] = ctx.trace_occlusion(capi.make_segments(rays["origin"], rays["dir"], tmax)).view(np.uint8)
        else:
            rng = np.random.RandomState(13).randint(0, 2 ** 32, len(rays), dtype=np.uint64).astype(np.uint32)
            res = ctx.trace_paths(capi.make_path_rays(rays["origin"], rays["dir"], rng), samples=2)
            out["rgb"], out["rngState"] = np.ascontiguousarray(res["rgb"]), np.ascontiguousarray(res["rngState"])
        _stats(ctx, out, opts, sc)
    elif e == "features":
        for f in (1, 2):
            ctx.set_int("Frame", f)
            ctx.dispatch_features()
        for name in capi.FEATURE_IMAGES:
            img = ctx.readback(name)
            if name == "FeatureFrame":
                for f in ("albedo", "dst", "normal", "object"):
                    out[f"FeatureFrame.{f}"] = np.ascontiguousarray(img[f])
            else:
                out[name] = img
        _stats(ctx, out, opts, sc)
    elif e == "camera_rays":
        out["rtCameraRays"] = ctx.camera_rays().view(np.uint8)
    elif e in ("bake_probes", "probes"):
        sh, rejected = ctx.bake_probes(PR.probe_positions(sc, seed=14, n=2), 33, 5)
        out["RtProbeSH.sh"], out["RtProbeSH.rejected"] = sh, rejected
        _stats(ctx, out, opts, sc)
    elif e in ("bake_cubemaps", "cubemaps"):
        cube = ctx.bake_cubemaps(PR.probe_positions(sc, seed=15, n=2), 2, 3, 6)
        out["RtCubeTexel.rgb"], out["RtCubeTexel.rejected"] = np.ascontiguousarray(cube["rgb"]), np.ascontiguousarray(cube["rejected"])
        _stats(ctx, out, opts, sc)
    elif e == "denoise":
        mgr.RenderFrame(); mgr.RenderFrame()
        mgr.RenderFeatures()
        mgr.Denoise()
        out["DenoisedRender"] = mgr.denoised_result
    elif e == "temporal":
        mgr.accumulate = False
        for k in range(2):
            c, s_ = np.cos(np.radians(1.5 * k)), np.sin(np.radians(1.5 * k))
            mgr.set_camera(sc.fov, np.asarray(sc.cam_local_to_world) @ np.array([[c, 0, s_, 0], [0, 1, 0, 0], [-s_, 0, c, 0], [0, 0, 0, 1]]))
            mgr.RenderFeatures()
            mgr.RenderFrame()
            mgr.DenoiseTemporal()
            out[f"DenoisedRender {k}"], out[f"TemporalFrame {k}"] = mgr.denoised_result, ctx.temporal_frame()
    else:
        raise AssertionError(f"unknown entry point {e}")
    mgr.OnDestroy()
    return out


def assert_outputs_equal(got, want, what):
    assert sorted(got) == sorted(want), f"{what}: buffers {sorted(got)} vs {sorted(want)}"
    for name, w in want.items():
        g = got[name]
        if isinstance(w, np.ndarray) and w.dtype.names:
            assert g.tobytes() == w.tobytes(), f"{what}: {name} differs"
        elif isinstance(w, np.ndarray) and w.dtype.kind == "f":
            assert_bit_equal(np.ascontiguousarray(g), np.ascontiguousarray(w), f"{what}: {name}")
        else:
            assert np.array_equal(g, w), f"{what}: {name}: {g} vs {w}"


_oracle_cache = {}


def oracle_outputs(row):
    key = (row.entry, tuple(sorted((k, v) for k, v in row.options.items() if k == "countStats")), row.scene)
    if key not in _oracle_cache:
        _oracle_cache[key] = run_row(ORACLE_LIB, row)
    return _oracle_cache[key]


def check_row(key, row):
    assert_outputs_equal(run_row(CUDA_LIB, row), oracle_outputs(row), f"{key} {row.entry} {row.options}")


# ---- tests ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("key", sorted(TABLE))
def test_row_equals_the_oracle(key):
    check_row(key, TABLE[key])


@pytest.mark.parametrize("key", sorted(SMEM_ROWS))
def test_row_above_48_kb_equals_the_oracle(key):
    check_row(key, SMEM_ROWS[key])
