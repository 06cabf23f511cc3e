"""CPU tests of the host side: BVH builder, RayComputeManager call sequence, the C-ABI surface (symbols exported,
loud failure without a GPU), error behaviour, and the N>1 tile logic over gloo (world_size 2).
"""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from conftest import CUDA_LIB, ORACLE_LIB, REPO, assert_bit_equal, render
import ray_tracing_b200 as rt
from ray_tracing_b200 import capi, multigpu, scenes


# ---- BVH builder (host/BVH.cpp, after BVH.cs:26-318) ------------------------------------------------------------------

def _check_tree(tris, nodes, ntri):
    seen = np.zeros(ntri, dtype=np.int32)
    assert len(nodes) % 2 == 1                                   # root + adjacent child pairs (BVH.cs:161-162)
    stack = [0]
    visited = 0
    while stack:
        i = stack.pop()
        visited += 1
        nd = nodes[i]
        if nd["triangleCount"] > 0:
            s, c = int(nd["startIndex"]), int(nd["triangleCount"])
            seen[s:s + c] += 1
            t = tris[s:s + c]
            pts = np.concatenate([t["posA"], t["posB"], t["posC"]])
            assert np.all(pts >= nd["boundsMin"] - 0) and np.all(pts <= nd["boundsMax"] + 0)
        else:
            a = int(nd["startIndex"])
            for ch in (a, a + 1):
                assert np.all(nodes[ch]["boundsMin"] >= nd["boundsMin"]) and np.all(nodes[ch]["boundsMax"] <= nd["boundsMax"])
                stack.append(ch)
    assert visited == len(nodes)
    assert np.all(seen == 1)                                     # every triangle in exactly one leaf


def test_bvh_invariants_and_quality_modes():
    m = scenes.knot_mesh(nu=120, nv=10)
    ntri = m.triangle_count
    for q in ("High", "Low"):
        tris, nodes, st = rt.build_bvh(m.vertices, m.indices, m.normals, q)
        assert len(tris) == ntri and st["TriangleCount"] == ntri and st["TotalNodeCount"] == len(nodes)
        assert st["LeafDepthMax"] <= 32
        _check_tree(tris, nodes, ntri)
    tris, nodes, st = rt.build_bvh(m.vertices, m.indices, m.normals, "Disabled")
    assert len(nodes) == 1 and nodes[0]["triangleCount"] == ntri and nodes[0]["startIndex"] == 0
    # Disabled keeps the mesh's triangle order (BVH.cs:62-80)
    assert np.array_equal(tris["posA"], m.vertices[m.indices[0::3]])


def test_bvh_single_triangle_and_errors():
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], dtype=np.float32)
    n = np.tile(np.array([[0, 0, 1]], dtype=np.float32), (3, 1))
    tris, nodes, st = rt.build_bvh(v, np.array([0, 1, 2], dtype=np.int32), n)
    assert len(nodes) == 1 and nodes[0]["triangleCount"] == 1
    with pytest.raises(ValueError):
        rt.build_bvh(v, np.array([0, 1, 5], dtype=np.int32), n)
    with pytest.raises(ValueError):
        rt.build_bvh(v, np.array([0, 1], dtype=np.int32), n)


def test_bvh_is_deterministic_and_splits_reduce_cost():
    m = scenes.knot_mesh(nu=60, nv=8)
    a = rt.build_bvh(m.vertices, m.indices, m.normals)
    b = rt.build_bvh(m.vertices, m.indices, m.normals)
    assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes()
    assert a[2]["LeafMaxTriCount"] < 64 and a[2]["LeafNodeCount"] > m.triangle_count // 16


def _triangle_mesh(tri, seed=0):
    """MeshDesc of an (n, 3, 3) array of triangle corners: unshared vertices, random normals."""
    v = np.ascontiguousarray(np.asarray(tri).reshape(-1, 3), dtype=np.float32)
    nrm = np.ascontiguousarray(np.random.RandomState(seed).uniform(-1, 1, v.shape), dtype=np.float32)
    return scenes.MeshDesc(v, np.arange(len(v), dtype=np.int32), nrm)


def large_adversarial_meshes():
    """(name, MeshDesc) pairs at and above the host builder's parallel threshold (16,384 triangles, host/BVH.cpp kParallelMinTris):
    the classes of tools/simt_fuzz_bvh.py, non-finite vertices and extents whose surface area overflows FP32 (every split costs inf,
    ChooseSplit falls back to 'axis 0, position 0' and Split still splits, so the tree has empty leaves), and a first split that
    leaves one triangle on one side.  Also used by the device build's tests on the GPU."""
    rng = np.random.RandomState(2024)

    def soup(n, scale=1.0):
        return (rng.uniform(-1, 1, (n, 1, 3)) + rng.uniform(-0.05, 0.05, (n, 3, 3))) * scale

    def grid(n):
        k = int(np.ceil(np.sqrt(n))); gx, gy = np.meshgrid(np.arange(k), np.arange(k))
        g = np.stack([gx.ravel(), gy.ravel(), np.zeros(k * k)], 1)[:n]
        return g[:, None, :] + np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], dtype=np.float64)[None]

    def degenerate(n):
        t = soup(n); t[::3, 1] = t[::3, 0]; t[::5, 2] = t[::5, 0]
        return t

    def line(n):
        t = np.zeros((n, 3, 3)); t[:, :, 0] = np.arange(n)[:, None] + rng.uniform(0, 0.9, (n, 3))
        return t

    def far_clusters(n):
        c = rng.choice([-100.0, 0.0, 100.0], (n, 1, 3)) + rng.uniform(-1, 1, (n, 1, 3))
        return c + rng.uniform(-0.2, 0.2, (n, 3, 3))

    def special(t, value, at):
        t = t.copy(); t[at] = value
        return t

    def lone_first(n):                                                  # the root's split puts one triangle left, n - 1 right
        t = soup(n) * 0.5 + 0.5
        t[0] -= 1000.0
        return t

    meshes = [("soup 16383", soup(16383)), ("equal-cost grid 16384", grid(16384)),
              ("coincident 16385", np.repeat(rng.uniform(-1, 1, (1, 3, 3)), 16385, axis=0)),
              ("degenerate 16383", degenerate(16383)), ("+-0 planes 16384", rng.choice([-1.0, -0.0, 0.0, 1.0, 0.5], (16384, 3, 3))),
              ("line 16385", line(16385)), ("far clusters 16384", far_clusters(16384)),
              ("NaN vertex 16385", special(soup(16385), np.nan, (9000, 1, 0))),
              ("+inf vertex 16384", special(soup(16384), np.inf, (123, 2, 1))),
              ("-inf vertex 16383", special(soup(16383), -np.inf, (16000, 0, 2))),
              ("extents 1e19 16385", soup(16385, 1e19)), ("extents 1e20 16384", soup(16384, 1e20)),
              ("one triangle split off first 16385", lone_first(16385)),
              ("far clusters with a +inf vertex 100003", special(far_clusters(100003), np.inf, (50000, 0, 0))),
              # regressions: the multi-threaded build once rebased the empty leaves' startIndex as if it were a child index
              ("overflow soup 20000", soup(20000, 1e19)),
              ("+inf vertex 30000", special(soup(30000), np.inf, (7777, 1, 1)))]
    return [(name, _triangle_mesh(t, seed=k)) for k, (name, t) in enumerate(meshes)]


def _same_bytes(a, b):
    return len(a) == len(b) and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def test_bvh_build_does_not_depend_on_the_thread_count():
    """The multi-threaded build (independent subtrees on different threads, slices of a large node evaluated in parallel) returns the
    single-threaded recursion's buffers byte for byte: same node order, same bounds, same triangle order, same statistics.  The nodes
    and the triangle order are also those of the oracle's plain restatement of the reference's recursion (oracle/rt_oracle.cpp), on
    benign meshes and on the adversarial ones above."""
    knot = scenes.knot_mesh(nu=400, nv=24)                                          # 19,200 triangles: above the parallel threshold
    soup = max(scenes.random_soup(16, 16, 2, 1, triangles=60000, spheres=1).meshes, key=lambda m: m.triangle_count)
    orc = capi.RtLib(ORACLE_LIB).create(0)
    try:
        for name, mesh in [("knot 19200", knot), ("soup", soup)] + large_adversarial_meshes():
            for q in ("High", "Low", "Disabled"):
                to, no = orc.build_bvh(mesh.vertices, mesh.indices, mesh.normals, rt.manager.QUALITY[q])
                rt.set_build_threads(1)
                t1, n1, s1 = rt.build_bvh(mesh.vertices, mesh.indices, mesh.normals, q)
                assert _same_bytes(n1, no) and _same_bytes(t1, to), f"{name} {q}: 1 thread vs the oracle"
                assert q == "Disabled" or (s1["TotalNodeCount"] == len(n1) and s1["TriangleCount"] == mesh.triangle_count)
                for threads in (2, 3, 5, 16, 0):
                    rt.set_build_threads(threads)
                    t, n, st = rt.build_bvh(mesh.vertices, mesh.indices, mesh.normals, q)
                    assert _same_bytes(n, no) and _same_bytes(t, to), f"{name} {q}: {threads or 'all'} threads vs the oracle"
                    assert {k: v for k, v in st.items() if k != "TimeMs"} == {k: v for k, v in s1.items() if k != "TimeMs"}, (name, q, threads)
    finally:
        rt.set_build_threads(0)
        orc.destroy()


def test_large_adversarial_meshes_have_empty_leaves():
    """The meshes above reach what they are there for: trees with empty leaves (triangleCount 0 and a startIndex that is a triangle
    index, not a child index) built by the multi-threaded path."""
    empty = {}
    for name, mesh in large_adversarial_meshes():
        _, nodes, st = rt.build_bvh(mesh.vertices, mesh.indices, mesh.normals, "High")
        empty[name] = st["LeafMinTriCount"] == 0
    assert empty["overflow soup 20000"] and empty["+inf vertex 30000"] and empty["extents 1e20 16384"], empty
    assert not empty["soup 16383"] and not empty["equal-cost grid 16384"], empty


def test_infinite_vertex_knot_renders_the_same_at_every_thread_count(oracle_path):
    """A 38,400-triangle knot with one vertex coordinate at +inf, rendered through the oracle: the default (all threads) host build
    gives the single-threaded recursion's tree, so the frame is the same bits (the multi-threaded build once produced child indices
    out of range, which rtDispatch refuses)."""
    sc = scenes.knot_room(32, 18, 2, 1, nu=400, nv=48)
    knot = max(range(len(sc.meshes)), key=lambda i: sc.meshes[i].triangle_count)
    sc.meshes[knot].vertices = sc.meshes[knot].vertices.copy()
    sc.meshes[knot].vertices[1234, 0] = np.inf
    assert sc.meshes[knot].triangle_count == 38400
    try:
        rt.set_build_threads(1)
        f1, a1 = render(oracle_path, sc)
        rt.set_build_threads(0)
        f0, a0 = render(oracle_path, sc)
    finally:
        rt.set_build_threads(0)
    assert_bit_equal(f0, f1, "all threads vs 1 thread")
    assert_bit_equal(a0, a1, "all threads vs 1 thread (accumulated)")
    assert np.isfinite(f1).all() and f1[..., :3].sum() > 0


def test_bvh_vs_brute_force_image(oracle_path):
    # same rays, tree vs one big leaf: identical closest hits except exact-distance ties between triangles sharing an edge
    sc = scenes.knot_room(96, 54, max_bounces=3, rays_per_pixel=1, nu=90, nv=8)
    f_tree, _ = render(oracle_path, sc)
    sc.settings["bvhQuality"] = 2
    f_flat, _ = render(oracle_path, sc)
    same = np.all(f_tree.view(np.uint32) == f_flat.view(np.uint32), axis=-1)
    assert same.mean() > 0.995


# ---- C-ABI surface --------------------------------------------------------------------------------------------------------

def _declared_symbols():
    txt = open(os.path.join(REPO, "include", "rt_b200.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(rt[A-Z]\w*)\s*\(", txt)))


def test_header_symbols_exported_by_cuda_library():
    names = _declared_symbols()
    assert len(names) >= 20 and "rtDispatch" in names
    lib = C.CDLL(CUDA_LIB)                                       # loads without a GPU (static cudart); no compute call made
    for n in names:
        assert hasattr(lib, n), f"librt_b200.so does not export {n}"
    lib.rtGetVersion.restype = C.c_int
    assert lib.rtGetVersion() == (1 << 16) | 1


def test_oracle_exports_the_same_abi():
    lib = C.CDLL(ORACLE_LIB)
    for n in _declared_symbols():
        assert hasattr(lib, n)


def test_product_library_has_no_oracle_dependency():
    out = subprocess.run(["ldd", CUDA_LIB], capture_output=True, text=True).stdout
    assert "oracle" not in out
    src = "".join(open(os.path.join(REPO, "ray_tracing_b200", "csrc", f)).read()
                  for f in os.listdir(os.path.join(REPO, "ray_tracing_b200", "csrc")))
    assert "oracle/" not in src and "rt_oracle" not in src


def test_product_does_not_reference_the_simt_build():
    """tests/simt (the SIMT interpreter build of the kernels) is test infrastructure: neither the package, the bench nor the
    driver entry points may know about it, and the product build never defines its macro."""
    files = [os.path.join(REPO, "bench.py"), os.path.join(REPO, "__graft_entry__.py")]
    pkg = os.path.join(REPO, "ray_tracing_b200")
    files += [os.path.join(pkg, f) for f in os.listdir(pkg) if f.endswith(".py")]
    files += [os.path.join(pkg, "host", f) for f in os.listdir(os.path.join(pkg, "host"))]
    for f in files:
        text = open(f).read()
        assert "simt" not in text.lower(), f
    from ray_tracing_b200 import build
    assert not any("SIMT" in flag for flag in build.NVCC_FLAGS + build.GXX_FLAGS)
    syms = subprocess.run(["nm", "-D", "--defined-only", CUDA_LIB], capture_output=True, text=True).stdout
    assert "simt" not in syms


def test_product_does_not_reference_the_probe():
    """tests/gpu_probe (the primitive probe of the arithmetic tests) is test infrastructure: it includes the product's device headers,
    never the other way round, and neither the package, its sources nor the bench build or load it (building it next to the oracle
    in __graft_entry__.build() is not using it)."""
    pkg = os.path.join(REPO, "ray_tracing_b200")
    files = [os.path.join(REPO, "bench.py")] + [os.path.join(pkg, f) for f in os.listdir(pkg) if f.endswith(".py")]
    for d in ("host", "csrc"):
        files += [os.path.join(pkg, d, f) for f in os.listdir(os.path.join(pkg, d))]
    for f in files:
        text = open(f).read()
        assert "gpu_probe" not in text and "rt_probe" not in text and "rtpRun" not in text, f
    syms = subprocess.run(["nm", "-D", "--defined-only", CUDA_LIB], capture_output=True, text=True).stdout
    assert "rtpRun" not in syms and "orProbe" not in syms


@pytest.mark.skipif(os.path.exists("/dev/nvidiactl"), reason="a GPU is present")
def test_cuda_library_fails_loudly_without_a_gpu():
    with pytest.raises(capi.RtError) as e:
        capi.RtLib(CUDA_LIB).create(0)
    assert e.value.code == capi.RT_E_NO_DEVICE and "no CPU path" in str(e.value)
    with pytest.raises(capi.RtError):
        rt.RayComputeManager(CUDA_LIB)                            # the manager does not fall back either


def test_missing_library_raises():
    with pytest.raises(FileNotFoundError):
        capi.RtLib("/nonexistent/librt_b200.so")


# ---- error behaviour of the ABI (exercised on the oracle implementation; the CUDA one is covered by the gpu tests) -----------

def test_abi_error_codes(oracle_path):
    ctx = capi.RtLib(oracle_path).create(0)
    with pytest.raises(capi.RtError) as e:
        ctx.set_int("NoSuchUniform", 1)
    assert e.value.code == capi.RT_E_UNKNOWN_NAME
    with pytest.raises(capi.RtError) as e:
        ctx.set_buffer_raw("Nodes", (C.c_char * 64)(), 2, 31)    # wrong stride
    assert e.value.code == capi.RT_E_INVALID
    with pytest.raises(capi.RtError) as e:
        ctx.set_buffer_raw("Meshes", (C.c_char * 64)(), 2, 32)
    assert e.value.code == capi.RT_E_UNKNOWN_NAME
    with pytest.raises(capi.RtError) as e:
        ctx.dispatch(0, 1, 1, 1)                                 # before rtResize
    assert e.value.code == capi.RT_E_STATE
    ctx.resize(16, 8)
    with pytest.raises(capi.RtError) as e:
        ctx.readback("FrameRender", np.empty((4, 4, 4), dtype=np.float32))
    assert e.value.code == capi.RT_E_INVALID
    with pytest.raises(capi.RtError) as e:
        ctx.readback("Depth")
    assert e.value.code == capi.RT_E_UNKNOWN_NAME
    ctx.set_int("triangleCount", 7)                              # declared-but-unused names are accepted (RayCommon.hlsl:24,120)
    ctx.set_vector("debugParams", (1, 2, 3, 4))
    ctx.destroy()


def test_manager_mirrors_reference_fields(oracle_path):
    mgr = rt.RayComputeManager(oracle_path)
    # defaults of RayComputeManager.cs:9-27
    assert mgr.maxBounceCount == 4 and mgr.numRaysPerPixel == 1 and mgr.accumulate == 1 and mgr.useSky == 0
    scenes.apply(scenes.cornell_spheres(16, 16, 2, 1), mgr)
    mgr.OnEnable()
    assert mgr.numAccumulatedFrames == 1                          # counter starts at 1 (quirk Q2, :71)
    mgr.RenderFrame(); mgr.RenderFrame()
    assert mgr.numAccumulatedFrames == 3
    assert np.all(mgr.accumulatedResult[..., 3] == 2.0)
    mgr.ResetAccumulatedRender()
    assert mgr.numAccumulatedFrames == 1 and np.all(mgr.accumulatedResult == 0.0)


def test_shared_mesh_is_built_once(oracle_path):
    # two models referencing one Mesh share nodeOffset / triOffset (RayComputeManager.cs:209-232)
    m = scenes.knot_mesh(nu=40, nv=6)
    mgr = rt.RayComputeManager(oracle_path)
    mgr.set_screen(32, 32)
    l2w, w2l = scenes.trs((0, 0, 6))
    mgr.set_camera(60.0, np.eye(4))
    mid = mgr.add_mesh(m.vertices, m.indices, m.normals)
    mgr.add_model(mid, *scenes.trs((-1.5, 0, 8), (0, 0, 0), (0.4, 0.4, 0.4)), scenes.material(emission=(1, 1, 1), emissionStrength=1.0))
    mgr.add_model(mid, *scenes.trs((1.5, 0, 8), (0, 90, 0), (0.4, 0.4, 0.4)), scenes.material(emission=(1, 1, 1), emissionStrength=1.0))
    mgr.renderSeed = 1
    mgr.OnEnable(); mgr.RenderFrame()
    assert len(mgr.bvh_stats()) == 1
    img = mgr.raytraceFrameTex
    assert img[:, :16, :3].sum() > 0 and img[:, 16:, :3].sum() > 0     # both instances visible


# ---- N > 1: row-band tiling over gloo (world_size 2, CPU) ----------------------------------------------------------------------

def test_band_ownership_layout():
    for h, world, band in [(1080, 8, 8), (1080, 4, 5), (17, 2, 4), (9, 3, 1)]:
        rows = [multigpu.owned_rows(h, r, world, band) for r in range(world)]
        allrows = np.sort(np.concatenate(rows))
        assert np.array_equal(allrows, np.arange(h))
        assert all(len(r) <= multigpu.rows_per_rank(h, world, band) for r in rows)
    rng = np.random.RandomState(0)
    frame, accum = rng.rand(17, 5, 4).astype(np.float32), rng.rand(17, 5, 4).astype(np.float32)
    g = np.stack([multigpu.pack_rows(frame, accum, r, 2, 4) for r in range(2)])
    f2, a2 = multigpu.unpack_rows(g, 17, 2, 4)
    assert_bit_equal(f2, frame); assert_bit_equal(a2, accum)


_GLOO_WORKER = r"""
import os, sys, numpy as np, torch, torch.distributed as dist
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, os.path.join(sys.argv[1], 'tests'))
import ray_tracing_b200 as rt
from ray_tracing_b200 import scenes, multigpu
rank, world = int(os.environ['RANK']), int(os.environ['WORLD_SIZE'])
dist.init_process_group('gloo', rank=rank, world_size=world)
oracle, out, band = sys.argv[2], sys.argv[3], 4
sc = scenes.cornell_spheres(40, 26, 3, 2)
mgr = rt.RayComputeManager(oracle)
scenes.apply(sc, mgr)
mgr.context.set_tile(rank, world, band)
mgr.OnEnable()
for frame_no in range(2):
    mgr.RenderFrame()
    packed = multigpu.pack_rows(mgr.raytraceFrameTex, mgr.accumulatedResult, rank, world, band)
    send = torch.from_numpy(packed).reshape(-1)
    recv = torch.empty(world * send.numel(), dtype=torch.float32)
    dist.all_gather_into_tensor(recv, send)                      # the ONE collective per frame
    frame, accum = multigpu.unpack_rows(recv.numpy().reshape((world,) + packed.shape), 26, world, band)
if rank == 0:
    np.save(out, np.stack([frame, accum]))
dist.barrier(); dist.destroy_process_group()
"""


def test_two_rank_tiles_equal_single_rank(tmp_path, oracle_path):
    script = tmp_path / "worker.py"
    script.write_text(_GLOO_WORKER)
    out = str(tmp_path / "tiled.npy")
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", MASTER_PORT="29517", WORLD_SIZE="2")
    procs = [subprocess.Popen([sys.executable, str(script), REPO, oracle_path, out], env=dict(env, RANK=str(r)),
                              stdout=subprocess.PIPE, stderr=subprocess.STDOUT) for r in range(2)]
    for p in procs:
        o, _ = p.communicate(timeout=240)
        assert p.returncode == 0, o.decode()
    tiled = np.load(out)
    frame, accum = render(oracle_path, scenes.cornell_spheres(40, 26, 3, 2), frames=2)
    assert_bit_equal(tiled[0], frame, "N=2 FrameRender vs N=1")
    assert_bit_equal(tiled[1], accum, "N=2 AccumulatedRender vs N=1")


# ---- the C++ host stands on its own (no Python in the loop) ------------------------------------------------------------------

def test_cpp_example_drives_the_abi_like_the_reference_manager(tmp_path, oracle_path):
    """examples/render_cornell.cpp: a C++ program using host/RayComputeManager directly (scene, OnEnable, RenderFrame x N,
    readback).  Run against the CPU oracle it must produce the image the Python-driven manager produces."""
    exe = str(tmp_path / "render_cornell")
    src = [os.path.join(REPO, "examples", "render_cornell.cpp"), os.path.join(REPO, "ray_tracing_b200", "host", "RayComputeManager.cpp"),
           os.path.join(REPO, "ray_tracing_b200", "host", "BVH.cpp")]
    cmd = [os.environ.get("CXX", "g++"), "-std=c++17", "-O1", "-ffp-contract=off", "-I", os.path.join(REPO, "include"),
           "-I", os.path.join(REPO, "ray_tracing_b200", "host")] + src + ["-ldl", "-pthread", "-o", exe]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe, oracle_path, "2"], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr + r.stdout
    m = re.search(r"numAccumulatedFrames=(\d+) alpha=([\d.]+) mean_rgb=([\d.eE+-]+)", r.stdout)
    assert m and int(m.group(1)) == 3 and float(m.group(2)) == 2.0
    _, accum = render(oracle_path, scenes.cornell_spheres(256, 256, 4, 1), frames=2)
    assert abs(float(m.group(3)) - accum[..., :3].astype(np.float64).sum() / (3.0 * 256 * 256 * 2)) < 1e-6
    # and it refuses to run without a GPU instead of falling back
    if not os.path.exists("/dev/nvidiactl"):
        r = subprocess.run([exe, CUDA_LIB, "1"], capture_output=True, text=True, timeout=120)
        assert r.returncode == 2 and "no CPU path" in r.stderr


def test_manager_error_paths_and_rebuild(oracle_path):
    m = scenes.knot_mesh(nu=30, nv=6)
    mgr = rt.RayComputeManager(oracle_path)
    mgr.set_screen(24, 16)
    mgr.set_camera(60.0, np.eye(4))
    mid = mgr.add_mesh(m.vertices, m.indices, m.normals)
    mgr.add_model(mid, *scenes.trs((0, 0, 6), (0, 0, 0), (0.5, 0.5, 0.5)), scenes.material(emission=(1, 1, 1), emissionStrength=1.0))
    mgr.OnEnable(); mgr.RenderFrame()
    first = mgr.raytraceFrameTex
    assert first[..., :3].sum() > 0 and len(mgr.bvh_stats()) == 1
    # adding a model later invalidates the BVH: the next frame rebuilds and uploads both (RayComputeManager.cs:143-161)
    mgr.add_model(mid, *scenes.trs((1.5, 1.0, 7), (0, 45, 0), (0.4, 0.4, 0.4)), scenes.material(emission=(1, 1, 1), emissionStrength=2.0))
    mgr.RenderFrame()
    assert mgr.raytraceFrameTex[..., :3].sum() > first[..., :3].sum()
    # a mesh with an out-of-range index is refused by the builder and reported through the manager, not crashed on
    bad = rt.RayComputeManager(oracle_path)
    bad.set_screen(8, 8)
    bad.set_camera(60.0, np.eye(4))
    mid = bad.add_mesh(m.vertices[:10], m.indices, m.normals[:10])
    bad.add_model(mid, np.eye(4), np.eye(4), scenes.material())
    with pytest.raises(capi.RtError) as e:
        bad.OnEnable()
    assert "index out of range" in str(e.value)
    with pytest.raises(capi.RtError):
        mgr.add_model(99, np.eye(4), np.eye(4), scenes.material())


def test_csharp_binding_declares_every_entry_point_of_the_header():
    """host_csharp/RtB200.cs (shipped as source: no C# toolchain here) must bind every function include/rt_b200.h declares."""
    import re
    header = open(os.path.join(REPO, "include", "rt_b200.h")).read()
    declared = set(re.findall(r"^(?:int|const char\*)\s+(rt[A-Z]\w*)\s*\(", header, flags=re.M))
    assert len(declared) >= 27
    cs = open(os.path.join(REPO, "host_csharp", "RtB200.cs")).read()
    bound = set(re.findall(r"static extern \w+ (rt[A-Z]\w*)\(", cs))
    assert declared <= bound, f"not bound in RtB200.cs: {sorted(declared - bound)}"
    m = re.search(r"public struct Stats \{([^}]*)\}", cs)
    fields = re.findall(r"(\w+)[,;]", m.group(1))
    assert [f for f in fields if f not in ("ulong", "double", "public")] == ["rays", "boxTests", "triTests", "sphereTests", "dispatches", "kernelMs", "sphereBoxTests", "exchangeMs"]


def test_abi_header_is_plain_c(tmp_path):
    """include/rt_b200.h promises plain C (no torch / CUDA types in any signature): gcc -std=c99 -pedantic must accept it."""
    src = tmp_path / "h.c"
    src.write_text('#include "rt_b200.h"\nint main(void) { return rtGetVersion() == RT_B200_VERSION ? 0 : 1; }\n')
    r = subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(REPO, "include"), "-fsyntax-only", str(src)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def test_bench_reference_arm_prints_the_contract_line():
    """bench.py --impl reference (the CPU arm: the oracle on this box's cores, no GPU): one JSON line with the contract's keys, the same
    `config` the GPU arm prints for the workload, and e2e = value with zero copy bytes."""
    import json
    r = subprocess.run([sys.executable, os.path.join(REPO, "bench.py"), "--impl", "reference", "--workload", "cornell64", "--steps", "1", "--warmup", "0"],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    line = json.loads(r.stdout.strip().splitlines()[-1])
    sys.path.insert(0, REPO)
    import bench
    assert line["impl"] == "reference" and line["unit"] == "Mrays/s" and line["higher_is_better"] is True and line["vs_baseline"] is None
    assert line["config"] == bench.workload_config("cornell64", bench.WORKLOADS["cornell64"])
    assert line["cpu_baseline"]["kind"] == "port" and line["cpu_baseline"]["cores"] >= 1 and line["cpu_baseline"]["value"] == line["value"] > 0
    assert line["e2e"] == {"value": line["value"], "unit": "Mrays/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert bench.DEFAULT_WORKLOAD == "knot256" and bench.WORKLOADS["knot256"]["spp"] == 256 and (bench.WORKLOADS["knot256"]["width"], bench.WORKLOADS["knot256"]["height"]) == (1920, 1080)
    # the algorithmic bytes are the SURVEY 8(d) formula
    st = {"boxTests": 10, "sphereBoxTests": 2, "triTests": 3, "rays": 5, "sphereTests": 7}
    assert bench.algorithmic_bytes(st, 4, 8, 2, 3) == 32 * 12 + 72 * 3 + 224 * 5 * 4 + 104 * 7 + 48 * 8 * 2 * 3
