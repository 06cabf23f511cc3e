"""The rtBakeCubemaps tests of tests/test_gpu_cubemaps.py, pointed at the SIMT interpreter build of the kernels (see
tests/test_simt_kernels.py), so that they run in the CPU suite at smaller sizes — minus the three cases that need torch CUDA tensors or
hundreds of millions of paths — plus a group context of three interpreter devices and the bake under the interpreter's other two lane
orders (RT_SIMT_ORDER)."""
import pytest

import ray_tracing_b200 as rt
from ray_tracing_b200 import scenes
import test_gpu_cubemaps as G
import test_gpu_probes as P
import test_gpu_trace_rays as T
import test_simt_kernels as S

simt_lib = S.simt_lib

# left to the GPU run: three launches of 32,800-sample texels, torch device pointers, and four probes on the cluster
_GPU_ONLY = {"test_texel_indices_across_internal_launches", "test_device_form_on_the_context_stream_and_a_caller_stream",
             "test_four_probes_on_the_871k_triangle_cluster"}


@pytest.fixture(autouse=True)
def _point_cubemap_tests_at_the_interpreter(monkeypatch, simt_lib):
    monkeypatch.setattr(G, "CUDA_LIB", simt_lib)
    monkeypatch.setattr(G, "PROBES", 2)
    monkeypatch.setattr(G, "CASES", ((1, 1), (1, 33), (2, 31), (2, 65), (7, 1)))    # one chunk short and over, three chunks padded to four


for _name in sorted(dir(G)):
    if _name.startswith("test_") and _name not in _GPU_ONLY:
        globals()["test_simt_" + _name[5:]] = getattr(G, _name)


def test_simt_group_of_three_devices_bakes_like_one_context(simt_lib):
    sc = scenes.instanced_knots(24, 16, 4, 1, instances=150)
    pos = P.probe_positions(sc, seed=18, n=1)
    one = T.open_mgr(simt_lib, sc)
    mgr = rt.RayComputeManager(simt_lib, devices=[0, 1, 2])
    scenes.apply(sc, mgr)
    mgr.OnEnable()
    for N, s in ((1, 33), (2, 3)):
        G.assert_texels_equal(mgr.context.bake_cubemaps(pos, N, s, 2), one.context.bake_cubemaps(pos, N, s, 2), f"group of three, {N}, {s}")
    mgr.OnDestroy()
    one.OnDestroy()


@pytest.mark.parametrize("order", ["1", "2"])
def test_simt_bake_does_not_depend_on_the_lane_schedule(simt_lib, monkeypatch, order):
    monkeypatch.setenv("RT_SIMT_ORDER", order)
    sc = scenes.instanced_knots(24, 16, 4, 1, instances=150)
    sc.spheres = scenes.random_soup(8, 8, 1, 1, triangles=3, spheres=200).spheres
    G.check_oracle(sc, P.probe_positions(sc, seed=19, n=1), ({"tlas": -1, "modelSkip": 1},), cases=((2, 33),), bounces=(4,), sky=1)
