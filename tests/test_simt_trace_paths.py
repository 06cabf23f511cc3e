"""The rtTracePaths tests of tests/test_gpu_trace_paths.py, pointed at the SIMT interpreter build of the kernels (see
tests/test_simt_kernels.py), so that they run in the CPU suite at smaller sizes — minus the 2M-path case and the torch device-pointer
case — plus a group context of three interpreter devices, the batch under the interpreter's other two lane orders (RT_SIMT_ORDER), and
the oracle's own rtTracePaths on its camera rays against its own FrameRender."""
import numpy as np
import pytest

from conftest import ORACLE_LIB, assert_bit_equal
import ray_tracing_b200 as rt
from ray_tracing_b200 import scenes
import test_gpu_trace_paths as G
import test_gpu_trace_rays as T
import test_simt_kernels as S

simt_lib = S.simt_lib

# left to the GPU run: the 2M-path case (hours of interpretation) and the one that needs torch CUDA tensors
_GPU_ONLY = {"test_two_million_camera_paths_on_the_871k_triangle_cluster", "test_device_pointer_form_on_the_context_stream_and_a_caller_stream"}


@pytest.fixture(autouse=True)
def _point_path_tests_at_the_interpreter(monkeypatch, simt_lib):
    monkeypatch.setattr(G, "CUDA_LIB", simt_lib)
    monkeypatch.setattr(G, "FRAME", (12, 8))
    monkeypatch.setattr(G, "RAYS", 32)


for _name in sorted(dir(G)):
    if _name.startswith("test_") and _name not in _GPU_ONLY:
        globals()["test_simt_" + _name[5:]] = getattr(G, _name)


def test_simt_group_of_three_devices_traces_like_one_context(simt_lib):
    sc = scenes.instanced_knots(24, 16, 4, 1, instances=150)
    rays = G.path_rays(sc, seed=17, n=24)
    one = T.open_mgr(simt_lib, sc)
    mgr = rt.RayComputeManager(simt_lib, devices=[0, 1, 2])
    scenes.apply(sc, mgr)
    mgr.OnEnable()
    for s in (1, 3):
        G.assert_radiance_equal(mgr.context.trace_paths(rays, s), one.context.trace_paths(rays, s), f"group of three, samples={s}")
    mgr.OnDestroy()
    one.OnDestroy()


@pytest.mark.parametrize("order", ["1", "2"])
def test_simt_batch_does_not_depend_on_the_lane_schedule(simt_lib, monkeypatch, order):
    monkeypatch.setenv("RT_SIMT_ORDER", order)
    sc = scenes.instanced_knots(24, 16, 4, 1, instances=150)
    sc.spheres = scenes.random_soup(8, 8, 1, 1, triangles=3, spheres=200).spheres
    G.check_rays(sc, G.path_rays(sc, seed=19, n=16), ({"tlas": -1, "modelSkip": 1}, {"countStats": 1, "modelSkip": 1}),
                 samples=(3,), bounces=(4,), sky=(1,))


@pytest.mark.parametrize("make", [lambda: scenes.cornell_spheres(24, 16, 4, 1),
                                  lambda: scenes.knot_room(24, 16, 6, 1, nu=40, nv=8, glass=True),
                                  G._soup_with_sky_and_defocus], ids=["cornell", "knot", "soup"])
@pytest.mark.parametrize("R", [1, 3])
def test_oracle_paths_on_its_camera_rays_equal_its_frame(make, R):
    """The oracle alone: its rtTracePaths over orCameraSample rays, chained sample by sample, rebuilds its own FrameRender — the
    statement that ties the path query to rtDispatch, checked without any build of the kernels."""
    sc = make()
    w, h = 20, 12
    sc.width, sc.height = w, h
    ref = G.open_frame(ORACLE_LIB, sc, R)
    assert_bit_equal(G.rebuild_frame(ref.context, ref.context, w, h, R), ref.raytraceFrameTex[..., :3], f"{sc.name} R={R}")
    ref.OnDestroy()
