"""GPU parity of everything written after the last GPU session of round 1: the round-2 options (pair order, grid fit, L2 window), the
device BVH build, the forced RandomValue draws, the TLAS over the models, the golden mesh fixture, and the regressions of the three
defects the randomised searches found (model boxes and distant ray origins, zero signs / non-finite input in the device BVH build).  All of
it is bit-exact on the SIMT interpreter build (tests/test_simt_kernels.py runs these bodies too); this file sorts after
test_gpu_parity.py so that `pytest -x -m gpu` reaches it after everything already validated on the GPU."""
import pytest

from conftest import CUDA_LIB, ORACLE_LIB, assert_bit_equal, render
from ray_tracing_b200 import scenes

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("order", [1, 3])
def test_pair_record_order_is_layout_only_on_gpu(order):
    sc = scenes.knot_room(160, 90, max_bounces=5, rays_per_pixel=2, nu=200, nv=12, glass=True)
    fo, ao, so = render(ORACLE_LIB, sc, frames=1, want_stats=True)
    for kernel, smem in ((2, 0), (2, 500), (1, 0)):
        fg, ag, sg = render(CUDA_LIB, sc, frames=1, options={"kernel": kernel, "pairOrder": order, "smemNodes": smem, "countStats": 1}, want_stats=True)
        assert_bit_equal(fg, fo, f"pairOrder={order} kernel={kernel} smemNodes={smem}")
        assert all(sg[k] == so[k] for k in ("rays", "boxTests", "triTests"))


@pytest.mark.parametrize("kernel", [1, 2])
def test_grid_fit_is_schedule_only_on_gpu(kernel):
    """A frame small enough that a 132-SM H100 gets about two pixels per persistent lane, so the fitted grid differs from the full one."""
    sc = scenes.cornell_spheres(640, 360, 6, 4) if kernel == 1 else scenes.knot_room(640, 360, max_bounces=5, rays_per_pixel=2, nu=120, nv=10)
    fo, ao = render(CUDA_LIB, sc, frames=2, options={"kernel": kernel})
    fg, ag = render(CUDA_LIB, sc, frames=2, options={"kernel": kernel, "gridFit": 1})
    assert_bit_equal(ag, ao, f"gridFit kernel={kernel}")


def _bvh_production_meshes():
    """The meshes the renders build: the 87k-triangle knot, the 871k-triangle cluster (one mesh) and the 900k-triangle mesh of the
    1M-triangle soup (the bench's big scene)."""
    biggest = lambda sc: max(sc.meshes, key=lambda m: m.triangle_count)          # noqa: E731
    return [("knot 87k", scenes.knot_mesh()), ("cluster 871k", biggest(scenes.knot_cluster(64, 36, 2, 1))),
            ("soup 900k", biggest(scenes.random_soup(16, 16, 2, 1)))]


def test_device_bvh_build_equals_the_host_builder_on_gpu():
    """rtBuildBVH on the H100 against the oracle's single-threaded restatement of the reference's recursion (oracle/rt_oracle.cpp), and
    host/BVH.cpp at all threads against the same: Nodes and Triangles byte for byte.  The production meshes, and the large adversarial
    meshes of tests/test_host.py (16,383 to 100,003 triangles: the host's multi-threaded path, empty leaves from non-finite vertices and
    overflowing extents) at all three qualities."""
    import numpy as np
    import ray_tracing_b200 as rt
    from ray_tracing_b200 import capi
    from test_host import large_adversarial_meshes
    same = lambda a, b: len(a) == len(b) and np.array_equal(a.view(np.uint8), b.view(np.uint8))    # noqa: E731
    gpu, orc = capi.RtLib(CUDA_LIB).create(0), capi.RtLib(ORACLE_LIB).create(0)
    rt.set_build_threads(0)
    cases = [(name, m, (1, 0)) for name, m in _bvh_production_meshes()] + [(name, m, (1, 0, 2)) for name, m in large_adversarial_meshes()]
    for name, m, qualities in cases:
        for q in qualities:
            to, no = orc.build_bvh(m.vertices, m.indices, m.normals, q)
            th, nh, _ = rt.build_bvh(m.vertices, m.indices, m.normals, q)
            tg, ng = gpu.build_bvh(m.vertices, m.indices, m.normals, q)
            assert same(nh, no) and same(th, to), f"host vs oracle: {name} q={q}"
            assert same(ng, no), f"device nodes vs oracle: {name} q={q} ({len(ng)} vs {len(no)} nodes)"
            assert same(tg, to), f"device triangle order vs oracle: {name} q={q}"
    gpu.destroy(); orc.destroy()


def test_device_bvh_build_through_the_manager_on_an_infinite_vertex_knot():
    """buildBVHOnDevice = 1 on the 38,400-triangle knot room with one vertex at +inf (a tree with empty leaves): the manager's frames
    are those of the host-built tree, on the H100 and through the oracle."""
    sc = scenes.knot_room(32, 18, 2, 1, nu=400, nv=48)
    knot = max(range(len(sc.meshes)), key=lambda i: sc.meshes[i].triangle_count)
    sc.meshes[knot].vertices = sc.meshes[knot].vertices.copy()
    sc.meshes[knot].vertices[1234, 0] = float("inf")

    def run(lib, on_device):
        import ray_tracing_b200 as rt
        mgr = rt.RayComputeManager(lib)
        scenes.apply(sc, mgr)
        mgr.buildBVHOnDevice = on_device
        mgr.OnEnable(); mgr.RenderFrame(); mgr.RenderFrame()
        out = mgr.accumulatedResult.copy()
        mgr.OnDestroy()
        return out

    ref = run(ORACLE_LIB, 0)
    assert_bit_equal(run(CUDA_LIB, 0), ref, "host-built tree")
    assert_bit_equal(run(CUDA_LIB, 1), ref, "device-built tree")


def test_l2_persistence_window_changes_nothing_but_caching():
    sc = scenes.knot_room(160, 90, max_bounces=5, rays_per_pixel=2, nu=200, nv=12)
    fo, ao = render(CUDA_LIB, sc, frames=2)
    fg, ag = render(CUDA_LIB, sc, frames=2, options={"l2Persist": 1})
    assert_bit_equal(ag, ao, "l2Persist")


def test_random_value_exactly_zero_and_exactly_one_on_gpu():
    """Quirk Q4 forced by seed construction (see tests/test_simt_kernels.py::test_simt_random_value_exactly_zero_and_exactly_one): log(0) in
    Box-Muller and a roulette draw of exactly 1.0, on the H100, all three kernels."""
    from conftest import seed_forcing_draw as _seed_forcing_draw
    W, H, x, y = 48, 32, 5, 7
    sc = scenes.cornell_spheres(W, H, 4, 1)
    sc.settings["useSky"] = True
    for post_state, draw in ((0, 7), (515875080, 12)):
        sc.settings["renderSeed"] = _seed_forcing_draw(post_state, draw, y * W + x)
        fo, _ = render(ORACLE_LIB, sc)
        for kernel in (0, 1, 2):
            fg, _ = render(CUDA_LIB, sc, options={"kernel": kernel})
            assert_bit_equal(fg, fo, f"forced draw {draw} kernel {kernel}")


# ---- TLAS over the models (SURVEY 8f #3): option "tlas" -----------------------------------------------------------------------------

def _tlas_scene(instances, width=96, height=54, bounces=5, spp=2):
    return scenes.instanced_knots(width, height, max_bounces=bounces, rays_per_pixel=spp, instances=instances)


@pytest.mark.parametrize("kernel", [1, 2])
def test_tlas_many_models_bitwise(kernel):
    """152 Model components (instancing of one mesh + room + light): above 128 models the TLAS is used automatically; forced on, forced
    off and automatic must all give the oracle's bits (the oracle walks every model like the reference)."""
    sc = _tlas_scene(150)
    fo, ao = render(ORACLE_LIB, sc, frames=2)
    for tlas in (-1, 1, 0):
        fg, ag = render(CUDA_LIB, sc, frames=2, options={"kernel": kernel, "tlas": tlas})
        assert_bit_equal(ag, ao, f"kernel {kernel} tlas {tlas}")


@pytest.mark.parametrize("kernel", [1, 2])
def test_tlas_forced_on_for_few_models(kernel):
    """The TLAS kernels with a root that is a leaf (3 models) and with a two-level tree (14 models); also together with the image split
    into row bands (rank 1 of 3)."""
    for sc in (scenes.knot_room(96, 54, max_bounces=5, rays_per_pixel=2, nu=90, nv=8, glass=True), _tlas_scene(12)):
        fo, ao = render(ORACLE_LIB, sc, frames=2)
        fg, ag = render(CUDA_LIB, sc, frames=2, options={"kernel": kernel, "tlas": 1})
        assert_bit_equal(ag, ao, f"{sc.name} kernel {kernel}")
    ft, at = render(CUDA_LIB, sc, frames=2, options={"kernel": kernel, "tlas": 1}, tile=(1, 3, 8))
    rows = [y for y in range(sc.height) if (y // 8) % 3 == 1]
    assert_bit_equal(at[rows], ao[rows], "row bands of rank 1 of 3")


@pytest.mark.parametrize("kernel", [1, 2])
def test_tlas_follows_per_frame_model_updates(kernel):
    """The reference re-sends ModelInfo every frame (RayComputeManager.cs:192-204): models move, change scale and material between
    frames, one leaves the scene's old bounds — the TLAS is rebuilt with the model records."""
    import numpy as np
    import ray_tracing_b200 as rt

    def run(lib, options):
        sc = _tlas_scene(80, 80, 48, 4, 1)
        rng = np.random.RandomState(3)
        mgr = rt.RayComputeManager(lib)
        scenes.apply(sc, mgr)
        for k, v in options.items():
            mgr.context.set_option(k, v)
        mgr.OnEnable()
        for frame in range(3):
            mgr.RenderFrame()
            for m in rng.choice(np.arange(2, 82), 12, replace=False):
                pos = (rng.uniform(-2.2, 2.2), rng.uniform(0.4, 3.4), rng.uniform(-1.5, 2.2)) if m % 5 else (rng.uniform(8, 12), 1.0, rng.uniform(8, 12))
                mgr.set_model_transform(int(m), *scenes.trs(position=pos, euler_deg=tuple(rng.uniform(0, 360, 3)), scale=tuple(rng.uniform(0.07, 0.3, 3))))
            mgr.set_model_material(int(rng.randint(2, 82)), scenes.material(flag=scenes.MAT_GLASS, ior=1.45, smoothness=0.9, specularProbability=0.9))
        mgr.RenderFrame()
        out = mgr.accumulatedResult.copy()
        mgr.OnDestroy()
        return out

    ref = run(ORACLE_LIB, {})
    assert_bit_equal(run(CUDA_LIB, {"kernel": kernel}), ref, "automatic TLAS, 82 models, four frames")
    assert_bit_equal(run(CUDA_LIB, {"kernel": kernel, "tlas": 0}), ref, "linear model test")


@pytest.mark.parametrize("kernel", [1, 2])
def test_tlas_with_sphere_accelerator_and_a_model_without_world_bounds(kernel):
    """70 models + 300 spheres (sphere accelerator and TLAS in one launch) + one model whose two matrices are not inverses of each
    other: the ray test only uses worldToLocal, so its world box comes from the inverse of that matrix, not from localToWorld.  Then
    the same with a second model whose worldToLocal is singular (it squashes space onto a plane): nothing can be said about where
    rays meet it, ray origins cannot be bounded any more, and no model is skipped at all."""
    import numpy as np
    sc = _tlas_scene(68)
    rng = np.random.RandomState(21)
    sph = np.zeros(300, dtype=scenes.SPHERE_DTYPE)
    for i in range(300):
        sph[i] = scenes._sphere((rng.uniform(-2.4, 2.4), rng.uniform(0.2, 3.6), rng.uniform(-1.5, 2.4)), rng.uniform(0.03, 0.12),
                                scenes.material(diffuse=tuple(rng.uniform(0.2, 0.9, 3)), specularProbability=0.3, smoothness=0.6) if i % 4 else
                                scenes.material(flag=scenes.MAT_GLASS, ior=1.5, smoothness=1.0, specularProbability=1.0))
    sc.spheres = sph
    l2w, _ = scenes.trs(position=(0.5, 1.0, 0.5), scale=(0.2, 0.2, 0.2))
    _, w2l = scenes.trs(position=(-0.8, 2.2, 0.3), euler_deg=(20, 40, 60), scale=(0.25, 0.2, 0.3))       # where the rays really meet it
    sc.models[5] = scenes.ModelDesc(0, l2w, w2l, sc.models[5].material)
    fo, ao = render(ORACLE_LIB, sc, frames=2)
    for tlas in (-1, 0):
        fg, ag = render(CUDA_LIB, sc, frames=2, options={"kernel": kernel, "tlas": tlas})
        assert_bit_equal(ag, ao, f"kernel {kernel} tlas {tlas}")
    flat = w2l.copy()
    flat[1, :] = 0.0                                                                              # local y = 0 for every world point
    sc.models[9] = scenes.ModelDesc(0, l2w, flat, sc.models[9].material)
    fo, ao = render(ORACLE_LIB, sc, frames=1)
    fg, ag = render(CUDA_LIB, sc, frames=1, options={"kernel": kernel})
    assert_bit_equal(ag, ao, f"kernel {kernel}, singular worldToLocal")


def test_golden_soup_fixture_on_the_kernels():
    """The committed mesh-path fixture (tests/golden/soup_small.json, written by the oracle): all three kernels reproduce its hashes, and
    the instrumented launches its traversal counters."""
    import hashlib
    import json
    import os
    import sys
    from conftest import GOLDEN
    sys.path.insert(0, GOLDEN)
    from make_golden import soup_scene
    fix = json.load(open(os.path.join(GOLDEN, "soup_small.json")))
    for kernel in (0, 1, 2):
        frame, accum, st = render(CUDA_LIB, soup_scene(), frames=2, options={"kernel": kernel, "countStats": 1}, want_stats=True)
        assert hashlib.sha256(accum.tobytes()).hexdigest() == fix["accum_sha256"], f"kernel {kernel}"
        assert hashlib.sha256(frame.tobytes()).hexdigest() == fix["frame_sha256"], f"kernel {kernel}"
        assert all(st[k] == fix[k] for k in ("rays", "boxTests", "triTests")), f"kernel {kernel}"


def test_tlas_at_the_capacity_of_the_candidate_mask():
    """4,096 models is what the per-lane candidate mask holds (128 words): the TLAS is used; 4,097 models fall back to the linear
    per-model test.  Small quads scattered in a room, every tenth one glass; both counts must give the oracle's bits."""
    import numpy as np
    rng = np.random.RandomState(77)
    meshes = [scenes.quad_mesh((-0.5, 0, -0.5), (0.5, 0, -0.5), (0.5, 0, 0.5), (-0.5, 0, 0.5)), scenes.room_mesh()]
    room = scenes.ModelDesc(1, np.eye(4), np.eye(4), scenes.material(diffuse=(0.75, 0.75, 0.75), specularProbability=0.0))
    quads = []
    for i in range(4096):
        l2w, w2l = scenes.trs(position=(rng.uniform(-2.5, 2.5), rng.uniform(0.2, 3.8), rng.uniform(-2.5, 2.5)), euler_deg=tuple(rng.uniform(0, 360, 3)),
                              scale=tuple(rng.uniform(0.05, 0.25, 3)))
        mat = (scenes.material(flag=scenes.MAT_GLASS, ior=1.4, smoothness=0.9, specularProbability=0.9) if i % 10 == 0 else
               scenes.material(diffuse=tuple(rng.uniform(0.2, 0.9, 3)), emission=(1, 1, 1), emissionStrength=float(i % 7 == 0) * 4.0, specularProbability=0.1))
        quads.append(scenes.ModelDesc(0, l2w, w2l, mat))
    for models in ([room] + quads[:4095], [room] + quads):
        sc = scenes.Scene(name="quads", width=64, height=36, meshes=meshes, models=models, cam_local_to_world=scenes.trs(position=(0, 1.9, -5.67))[0],
                          fov=54.5, settings=dict(maxBounceCount=4, numRaysPerPixel=2))
        fo, ao = render(ORACLE_LIB, sc, frames=1)
        for kernel in (2, 1):
            fg, ag = render(CUDA_LIB, sc, frames=1, options={"kernel": kernel})
            assert_bit_equal(ag, ao, f"{len(models)} models kernel {kernel}")


@pytest.mark.parametrize("kernel", [1, 2])
def test_model_skipping_stays_exact_for_a_distant_camera(kernel):
    """Regression: 1,500 two-to-eight-centimetre models seen from 100,000 and 400,000 units away.  Where such a ray 'passes' is blurred
    by a few ulp of its origin's coordinates in the reference's own arithmetic (world -> local transform, Moeller-Trumbore), so the
    padding of the models' world boxes must grow with the extent of the region ray origins come from (buildModels, rt_repack.cuh);
    with the fixed padding of the first version 36 and 156 values of these two frames differed from the oracle.  Linear box test and TLAS."""
    import numpy as np
    rng = np.random.RandomState(77)
    meshes = [scenes.quad_mesh((-0.5, 0, -0.5), (0.5, 0, -0.5), (0.5, 0, 0.5), (-0.5, 0, 0.5))]
    quads = []
    for i in range(1500):
        l2w, w2l = scenes.trs(position=(rng.uniform(-2.5, 2.5), rng.uniform(0.2, 3.8), rng.uniform(-2.5, 2.5)), euler_deg=tuple(rng.uniform(0, 360, 3)),
                              scale=tuple(rng.uniform(0.02, 0.08, 3)))
        quads.append(scenes.ModelDesc(0, l2w, w2l, scenes.material(diffuse=(0.8, 0.8, 0.8), emission=(1, 1, 1), emissionStrength=1.0)))
    for dist, fov in ((100000.0, 0.0032), (400000.0, 0.0008)):
        sc = scenes.Scene(name="quads_from_afar", width=160, height=90, meshes=meshes, models=quads, cam_local_to_world=scenes.trs(position=(0, 1.9, -dist))[0],
                          fov=fov, settings=dict(maxBounceCount=1, numRaysPerPixel=2, divergeStrength=0.0))
        fo, ao = render(ORACLE_LIB, sc, frames=1)
        assert np.count_nonzero(np.any(fo[..., :3] > 0, axis=2)) > 200
        for tlas in ((0, 1) if kernel == 1 else (1,)):          # (kept short for the interpreter run of the pooled kernel)
            fg, ag = render(CUDA_LIB, sc, frames=1, options={"kernel": kernel, "tlas": tlas})
            assert_bit_equal(fg, fo, f"camera at {dist} kernel {kernel} tlas {tlas}")
        if kernel == 2:
            break


def test_moving_the_camera_out_of_the_padded_region_rebuilds_the_model_boxes():
    """The padding is computed for a region of ray origins (camera + geometry, with a quarter of its size as room); a camera that leaves
    it must trigger a rebuild of the model records although ModelInfo was not re-sent."""
    import ray_tracing_b200 as rt

    def run(lib, options):
        sc = _tlas_scene(40, 80, 48, 3, 1)
        mgr = rt.RayComputeManager(lib)
        scenes.apply(sc, mgr)
        for k, v in options.items():
            mgr.context.set_option(k, v)
        mgr.OnEnable()
        mgr.RenderFrame()
        mgr.set_camera(0.02, scenes.trs(position=(0.0, 1.9, -30000.0))[0])          # far outside: the boxes built for the first frame are too tight now
        mgr.ResetAccumulatedRender()
        for _ in range(2):
            mgr.RenderFrame()
        out = mgr.accumulatedResult.copy()
        mgr.OnDestroy()
        return out

    ref = run(ORACLE_LIB, {})
    for kernel in (1, 2):
        assert_bit_equal(run(CUDA_LIB, {"kernel": kernel}), ref, f"kernel {kernel}")


def test_model_free_device_bvh_build_on_degenerate_and_non_finite_input():
    """rtBuildBVH against the oracle's restatement of the reference's recursion (and host/BVH.cpp against the same), byte for byte, where
    a level-synchronous build can go wrong (all found by tools/simt_fuzz_bvh.py): bounds that see +0 and -0 (the reference's sequential
    strict comparison keeps the first), NaN vertices (never replace a running bound), an infinite vertex and extents whose surface area
    overflows FP32 (every candidate costs inf, ChooseSplit returns its defaults 'axis 0, position 0' and Split still splits — the first
    version of the device build never finished on that).  Small meshes only: tests/test_simt_kernels.py runs this body on the
    interpreter; the large ones are in test_device_bvh_build_equals_the_host_builder_on_gpu."""
    import numpy as np
    import ray_tracing_b200 as rt
    from ray_tracing_b200 import capi
    gpu, orc = capi.RtLib(CUDA_LIB).create(0), capi.RtLib(ORACLE_LIB).create(0)
    rng = np.random.RandomState(4)
    cases = []
    cases.append(rng.choice([-1.0, -0.0, 0.0, 1.0, 0.5], (300, 3, 3)))                                        # exact zeros of both signs
    soup = rng.uniform(-1, 1, (200, 1, 3)) + rng.uniform(-0.05, 0.05, (200, 3, 3))
    for special in (np.nan, np.inf, -np.inf):
        t = soup.copy(); t[17, 1, 0] = special; t[90, 2, 2] = special
        cases.append(t)
    cases.append(soup * 1e20)                                                                                   # area overflows to inf
    k = 16; gx, gy = np.meshgrid(np.arange(k), np.arange(k))
    cases.append(np.stack([gx.ravel(), gy.ravel(), np.zeros(k * k)], 1)[:, None, :] + np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], dtype=np.float64)[None])   # equal costs
    for tri in cases:
        v = np.ascontiguousarray(tri.reshape(-1, 3), dtype=np.float32)
        idx = np.arange(len(v), dtype=np.int32)
        nrm = np.ascontiguousarray(rng.uniform(-1, 1, v.shape), dtype=np.float32)
        for q in (1, 0, 2):
            to, no = orc.build_bvh(v, idx, nrm, q)
            th, nh, _ = rt.build_bvh(v, idx, nrm, q)
            tg, ng = gpu.build_bvh(v, idx, nrm, q)
            assert len(nh) == len(no) and np.array_equal(nh.view(np.uint8), no.view(np.uint8)) and np.array_equal(th.view(np.uint8), to.view(np.uint8))
            assert len(ng) == len(no) and np.array_equal(ng.view(np.uint8), no.view(np.uint8)) and np.array_equal(tg.view(np.uint8), to.view(np.uint8))
    # a tree with more than 2n + 1 nodes (chains of empty children below an infinite box): every builder refuses, none hangs
    t = soup[:20].copy(); t[17, 1, 0] = np.inf
    v = np.ascontiguousarray(t.reshape(-1, 3), dtype=np.float32); idx = np.arange(len(v), dtype=np.int32)
    with pytest.raises(ValueError):
        rt.build_bvh(v, idx, v, 1)
    with pytest.raises(capi.RtError):
        orc.build_bvh(v, idx, v, 1)
    with pytest.raises(capi.RtError):
        gpu.build_bvh(v, idx, v, 1)
    gpu.destroy(); orc.destroy()
