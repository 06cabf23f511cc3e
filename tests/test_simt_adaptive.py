"""The rtDispatchAdaptive tests of tests/test_gpu_adaptive.py, pointed at the SIMT interpreter build of the kernels (see
tests/test_simt_kernels.py), so that they run in the CPU suite; the list-driven kernels under the interpreter's other two lane orders
(RT_SIMT_ORDER); and the quality gate: adaptive sampling against uniform sampling at an equal budget of traced pixel-frames, measured
on the oracle, whose images the kernels reproduce bit for bit."""
import numpy as np
import pytest

from conftest import ORACLE_LIB
import ray_tracing_b200 as rt
from ray_tracing_b200 import capi, scenes
import test_gpu_adaptive as G
import test_simt_kernels as S

simt_lib = S.simt_lib

# left to the GPU run: 4K (hours of interpretation) and the torch stream
_GPU_ONLY = {"test_4k_knot_cluster_against_ten_oracle_rows", "test_stream_order_on_a_caller_stream"}


@pytest.fixture(autouse=True)
def _point_adaptive_tests_at_the_interpreter(monkeypatch, simt_lib):
    monkeypatch.setattr(G, "CUDA_LIB", simt_lib)


for _name in sorted(dir(G)):
    if _name.startswith("test_") and _name not in _GPU_ONLY:
        globals()["test_simt_" + _name[5:]] = getattr(G, _name)


@pytest.mark.parametrize("order", ["1", "2"])
def test_simt_adaptive_does_not_depend_on_the_lane_schedule(simt_lib, monkeypatch, order):
    monkeypatch.setenv("RT_SIMT_ORDER", order)
    sc = scenes.knot_room(32, 16, max_bounces=5, rays_per_pixel=2, nu=40, nv=8, glass=True)
    G.check_oracle(sc, ({"kernel": 0}, {"kernel": 1}, {"kernel": 2, "countStats": 1}, {"kernel": 2, "poolSlots": 32, "sortRays": 1}),
                   session=[(0.3, 2, 6)] * 8)


# ---- quality gate ------------------------------------------------------------------------------------------------------------

def _rel_mse(x, ref):
    return float(np.mean((x[..., :3].astype(np.float64) - ref[..., :3]) ** 2 / (ref[..., :3].astype(np.float64) ** 2 + 0.01)))


def _mean(a):
    w = a[..., 3:4]
    return np.where(w > 0, a / np.where(w > 0, w, 1), 0)


def _render(sc, adaptive, frames=0, rays_per_pixel=1, seed=None):
    mgr = rt.RayComputeManager(ORACLE_LIB)
    scenes.apply(sc, mgr)
    mgr.numRaysPerPixel = rays_per_pixel
    if seed is not None:
        mgr.renderSeed = seed
    mgr.OnEnable()
    used = 0
    if adaptive:
        while True:                     # with the managers' defaults, until nothing is active
            n = mgr.RenderFrameAdaptive()
            used += n
            if n == 0:
                break
    else:
        mgr.RenderFrames(frames)
    img = _mean(mgr.accumulatedResult)
    mgr.OnDestroy()
    return img, used


@pytest.mark.parametrize("name", ["cornell", "knot_room_glass"])
def test_adaptive_beats_uniform_at_an_equal_budget(name):
    """48 x 32, 1 spp per frame: RenderFrameAdaptive with the capi defaults until it returns 0, against uniform frames of the same
    number of traced pixel-frames (the error interpolated between the two whole frame counts around it).  Relative MSE against a
    1024-sample render of an independent seed.  DESIGN.md section 7d'''''''' records the factors."""
    W, H = 48, 32
    sc = scenes.cornell_spheres(W, H, 4, 1) if name == "cornell" else scenes.knot_room(W, H, 8, 1, glass=True)
    ref, _ = _render(sc, False, frames=64, rays_per_pixel=16, seed=977)
    img, used = _render(sc, True)
    k = used / (W * H)
    lo, hi = int(np.floor(k)), int(np.ceil(k))
    e_lo, e_hi = (_rel_mse(_render(sc, False, frames=f)[0], ref) for f in (lo, hi))
    uniform = e_lo + (e_hi - e_lo) * (k - lo) if hi > lo else e_hi
    adaptive = _rel_mse(img, ref)
    print(f"{name}: {k:.2f} frames per pixel, relative MSE adaptive {adaptive:.4f}, uniform {uniform:.4f}, factor {uniform / adaptive:.2f}")
    assert capi.ADAPTIVE_MIN_FRAMES <= k <= capi.ADAPTIVE_MAX_FRAMES
    assert adaptive < uniform
