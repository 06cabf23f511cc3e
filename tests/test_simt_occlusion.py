"""The rtTraceOcclusion tests of tests/test_gpu_occlusion.py, pointed at the SIMT interpreter build of the kernels (see
tests/test_simt_kernels.py), so that they run in the CPU suite — minus the 4M-segment case and the torch device-pointer case — plus a
group context of three interpreter devices, the batch under the interpreter's other two lane orders (RT_SIMT_ORDER), and the check
that the oracle's early-exit walk and its full loop from tMax give the same answer on every segment."""
import ctypes as C

import numpy as np
import pytest

from conftest import ORACLE_LIB
import ray_tracing_b200 as rt
from ray_tracing_b200 import capi, scenes
import test_gpu_occlusion as G
import test_gpu_trace_rays as T
import test_simt_kernels as S

simt_lib = S.simt_lib

# left to the GPU run: the 4M-segment case (hours of interpretation) and the one that needs torch CUDA tensors
_GPU_ONLY = {"test_four_million_segments_on_the_871k_triangle_cluster", "test_device_pointer_form_on_the_context_stream_and_a_caller_stream"}


@pytest.fixture(autouse=True)
def _point_occlusion_tests_at_the_interpreter(monkeypatch, simt_lib):
    monkeypatch.setattr(G, "CUDA_LIB", simt_lib)
    monkeypatch.setattr(G, "RAYS", 64)


for _name in sorted(dir(G)):
    if _name.startswith("test_") and _name not in _GPU_ONLY:
        globals()["test_simt_" + _name[5:]] = getattr(G, _name)


def test_simt_group_of_three_devices_traces_like_one_context(simt_lib):
    sc = scenes.instanced_knots(24, 16, 3, 1, instances=150)
    sets = G.segment_sets(sc, seed=17, n=48)
    one = T.open_mgr(simt_lib, sc)
    mgr = rt.RayComputeManager(simt_lib, devices=[0, 1, 2])
    scenes.apply(sc, mgr)
    mgr.OnEnable()
    for name, s in sets.items():
        G.assert_occlusion_equal(mgr.context.trace_occlusion(s), one.context.trace_occlusion(s), f"group of three, {name}")
    mgr.OnDestroy()
    one.OnDestroy()


@pytest.mark.parametrize("order", ["1", "2"])
def test_simt_batch_does_not_depend_on_the_lane_schedule(simt_lib, monkeypatch, order):
    monkeypatch.setenv("RT_SIMT_ORDER", order)
    sc = scenes.instanced_knots(24, 16, 3, 1, instances=150)
    sc.spheres = scenes.random_soup(8, 8, 1, 1, triangles=3, spheres=200).spheres
    G.check_scene(sc, ({"tlas": -1, "modelSkip": 1}, {"countStats": 1, "modelSkip": 1}), sets=G.segment_sets(sc, seed=19, n=48),
                  flags=(False,))


@pytest.mark.parametrize("make", [lambda: scenes.knot_room(24, 16, 3, 1, nu=40, nv=8, glass=True),
                                  lambda: scenes.random_soup(24, 16, 3, 1, triangles=400, spheres=120),
                                  lambda: scenes.instanced_knots(24, 16, 3, 1, instances=40)], ids=["knot", "soup", "instances"])
def test_oracle_early_exit_equals_its_full_loop_from_tmax(make):
    """The oracle answers with a walk that stops at its first hit (tests/oracle_ext/rt_oracle_occlusion.cpp); the definition is the
    collision loop from result.dst = tMax to the end.  The two must agree on every segment, whatever order the primitives come in —
    the argument that makes the early exit exact, as a test."""
    sc = make()
    sets = G.segment_sets(sc, seed=23, n=160)
    segs = np.concatenate(list(sets.values()))
    mgr = T.open_mgr(ORACLE_LIB, sc)
    L = mgr.context._L
    L.orTraceOcclusionFull.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int]
    for flags in (0, capi.RT_TRACE_NO_CULL):
        early = mgr.context.trace_occlusion(segs, no_cull=bool(flags))
        full = np.zeros(len(segs), dtype=np.uint8)
        st = mgr.context.stats()
        assert L.orTraceOcclusionFull(mgr.context.handle, segs.ctypes.data, len(segs), full.ctypes.data, flags) == capi.RT_OK
        assert mgr.context.stats()["rays"] == st["rays"], "the test hook counts nothing"
        G.assert_occlusion_equal(early, full.astype(bool), f"early exit vs full loop, flags {flags}", segs)
        assert 0 < early.sum() < len(early)
    mgr.OnDestroy()
