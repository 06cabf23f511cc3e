"""The rtTraceRays tests of tests/test_gpu_trace_rays.py, pointed at the SIMT interpreter build of the kernels (see
tests/test_simt_kernels.py), so that they run in the CPU suite — minus the 4M-ray case and the torch device-pointer case — plus a group
context of three interpreter devices, the batch under the interpreter's other two lane orders (RT_SIMT_ORDER), and the check that the
oracle's winner-recording loop agrees with its CalculateRayCollision."""
import ctypes as C

import numpy as np
import pytest

from conftest import ORACLE_LIB
import ray_tracing_b200 as rt
from ray_tracing_b200 import capi, scenes
import test_gpu_trace_rays as G
import test_simt_kernels as S

simt_lib = S.simt_lib

# left to the GPU run: the 4M-ray case (hours of interpretation) and the one that needs torch CUDA tensors
_GPU_ONLY = {"test_four_million_rays_on_the_871k_triangle_cluster", "test_device_pointer_form_on_the_context_stream_and_a_caller_stream"}


@pytest.fixture(autouse=True)
def _point_trace_rays_tests_at_the_interpreter(monkeypatch, simt_lib):
    monkeypatch.setattr(G, "CUDA_LIB", simt_lib)
    monkeypatch.setattr(G, "RAYS", 96)


for _name in sorted(dir(G)):
    if _name.startswith("test_") and _name not in _GPU_ONLY:
        globals()["test_simt_" + _name[5:]] = getattr(G, _name)


def test_simt_group_of_three_devices_traces_like_one_context(simt_lib):
    sc = scenes.instanced_knots(24, 16, 3, 1, instances=150)
    sets = G.ray_sets(sc, seed=17, n=64)
    one = G.open_mgr(simt_lib, sc)
    mgr = rt.RayComputeManager(simt_lib, devices=[0, 1, 2])
    scenes.apply(sc, mgr)
    mgr.OnEnable()
    for name, r in sets.items():
        G.assert_hits_equal(mgr.context.trace_rays(r), one.context.trace_rays(r), f"group of three, {name}")
    mgr.OnDestroy()
    one.OnDestroy()


@pytest.mark.parametrize("order", ["1", "2"])
def test_simt_batch_does_not_depend_on_the_lane_schedule(simt_lib, monkeypatch, order):
    monkeypatch.setenv("RT_SIMT_ORDER", order)
    sc = scenes.instanced_knots(24, 16, 3, 1, instances=150)
    sc.spheres = scenes.random_soup(8, 8, 1, 1, triangles=3, spheres=200).spheres
    G.check_scene(sc, ({"tlas": -1, "modelSkip": 1}, {"countStats": 1, "modelSkip": 1}), sets=G.ray_sets(sc, seed=19, n=64), flags=(False,))


@pytest.mark.parametrize("make", [lambda: scenes.knot_room(24, 16, 3, 1, nu=40, nv=8, glass=True),
                                  lambda: scenes.random_soup(24, 16, 3, 1, triangles=400, spheres=120)], ids=["knot", "soup"])
def test_oracle_winner_loop_equals_its_calculate_ray_collision(make):
    """The oracle names the winner with a restatement of the collision loop (tests/oracle_ext/rt_oracle_trace_rays.cpp): its dst, pos,
    normal and isBackface must be CalculateRayCollision's for every ray, so that the two cannot drift apart."""
    sc = make()
    sets = G.ray_sets(sc, seed=23, n=200)
    rays = np.concatenate(list(sets.values()))
    mgr = G.open_mgr(ORACLE_LIB, sc)
    L = mgr.context._L
    L.orTraceRaysLoop.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int]
    for flags in (0, capi.RT_TRACE_NO_CULL):
        want = mgr.context.trace_rays(rays, no_cull=bool(flags))
        loop = np.zeros(len(rays), dtype=capi.RAY_HIT_DTYPE)
        assert L.orTraceRaysLoop(mgr.context.handle, rays.ctypes.data, len(rays), loop.ctypes.data, flags) == capi.RT_OK
        G.assert_hits_equal(loop, want, f"winner loop, flags {flags}")
        assert (want["kind"] != capi.RT_HIT_NONE).any()
    mgr.OnDestroy()
