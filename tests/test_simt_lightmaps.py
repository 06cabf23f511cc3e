"""The rtBakeLightmap tests of tests/test_gpu_lightmaps.py, pointed at the SIMT interpreter build of the kernels (see
tests/test_simt_kernels.py), so that they run in the CPU suite at smaller sizes — minus the cases that need torch CUDA tensors or
hundreds of millions of paths — plus a group context of three interpreter devices, the bake under the interpreter's other two lane
orders (RT_SIMT_ORDER), and the launch rule read off the interpreter's launch log: for each <STATS, EXT, TLAS> the rule can choose,
rtBakeLightmap launches exactly that k_bake_cubemaps instantiation and k_cube_sums, and equals the oracle."""
import pytest

import ray_tracing_b200 as rt
from ray_tracing_b200 import scenes
import test_gpu_kernel_matrix as KM
import test_gpu_lightmaps as G
import test_gpu_trace_rays as T
import test_simt_kernels as S
from conftest import ORACLE_LIB
from test_simt_kernel_matrix import LaunchLog

simt_lib = S.simt_lib

# left to the GPU run: two launches of 32,800-sample texels, a million texels, torch device pointers, and the cluster
_GPU_ONLY = {"test_texel_indices_across_internal_launches", "test_more_texels_than_one_host_batch",
             "test_device_form_on_the_context_stream_and_a_caller_stream", "test_vertex_texels_of_the_871k_triangle_cluster"}


@pytest.fixture(autouse=True)
def _point_lightmap_tests_at_the_interpreter(monkeypatch, simt_lib):
    monkeypatch.setattr(G, "CUDA_LIB", simt_lib)
    monkeypatch.setattr(G, "RANDOM", 2)
    monkeypatch.setattr(G, "VERTICES", 2)
    monkeypatch.setattr(G, "SAMPLES", (1, 31, 33, 65))          # one chunk short and over, three chunks padded to four
    monkeypatch.setattr(G, "BOUNCE_SAMPLES", 1024)
    monkeypatch.setattr(G, "BOUNCE_REF", 1 << 14)


for _name in sorted(dir(G)):
    if _name.startswith("test_") and _name not in _GPU_ONLY:
        globals()["test_simt_" + _name[5:]] = getattr(G, _name)


def test_simt_group_of_three_devices_bakes_like_one_context(simt_lib):
    sc = scenes.instanced_knots(24, 16, 4, 1, instances=150)
    pts = G.texel_set(sc, 18)
    one = T.open_mgr(simt_lib, sc)
    mgr = rt.RayComputeManager(simt_lib, devices=[0, 1, 2])
    scenes.apply(sc, mgr)
    mgr.OnEnable()
    for s in (33, 3):
        G.CM.assert_texels_equal(mgr.context.bake_lightmap(pts, s, 2), one.context.bake_lightmap(pts, s, 2), f"group of three, {s}")
    mgr.OnDestroy()
    one.OnDestroy()


@pytest.mark.parametrize("order", ["1", "2"])
def test_simt_bake_does_not_depend_on_the_lane_schedule(simt_lib, monkeypatch, order):
    monkeypatch.setenv("RT_SIMT_ORDER", order)
    sc = scenes.instanced_knots(24, 16, 4, 1, instances=150)
    sc.spheres = scenes.random_soup(8, 8, 1, 1, triangles=3, spheres=200).spheres
    G.check_oracle(sc, G.texel_set(sc, 19), ({"tlas": -1, "modelSkip": 1},), samples=(33,), bounces=(4,), sky=1)


@pytest.mark.parametrize("variant", KM.VARIANTS, ids=lambda v: "<%d, %d, %d>" % v)
def test_simt_launch_rule_runs_the_cube_kernels(simt_lib, variant):
    """The kernel matrix's scene and options for each <STATS, EXT, TLAS>: a bake launches exactly k_bake_cubemaps<STATS, EXT, TLAS>
    and k_cube_sums (the second bake of the session, after the scene is on the device), and equals the oracle."""
    s, x, t = variant
    opts, ext = KM._variant_options(s, x, t)
    sc = KM.matrix_scene(ext)
    pts = G.texel_set(sc, 20)
    log = LaunchLog(simt_lib)
    mgr = T.open_mgr(simt_lib, sc, opts)
    mgr.context.bake_lightmap(pts[:1], 1, 0)
    log.reset()
    mgr.context.reset_stats()
    got = mgr.context.bake_lightmap(pts, 33, 6)
    st = mgr.context.stats()
    names = {n for n, _ in log.read()}
    mgr.OnDestroy()
    want_kernel = "k_bake_cubemaps<%s, %s, %s>" % tuple(KM.B[bool(v)] for v in variant)
    assert names == {want_kernel, "k_cube_sums"}, names
    ref = T.open_mgr(ORACLE_LIB, sc, {"countStats": s} if s else {})
    ref.context.reset_stats()
    want = ref.context.bake_lightmap(pts, 33, 6)
    wst = ref.context.stats()
    ref.OnDestroy()
    G.CM.assert_texels_equal(got, want, want_kernel)
    keys = KM.COUNTS if s and len(sc.spheres) <= 64 else KM.COUNTS[:3] if s else ("rays",)
    assert all(st[k] == wst[k] for k in keys), (want_kernel, st, wst)
