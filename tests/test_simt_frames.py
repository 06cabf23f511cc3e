"""The rtDispatchFrames tests of tests/test_gpu_frames.py, pointed at the SIMT interpreter build of the kernels (see
tests/test_simt_kernels.py), so that they run in the CPU suite — the group context there is several interpreter 'devices' — plus
the batch kernels under the interpreter's other two lane orders (RT_SIMT_ORDER)."""
import pytest

from conftest import ORACLE_LIB, assert_bit_equal
from ray_tracing_b200 import scenes
import test_gpu_frames as G
import test_simt_kernels as S

simt_lib = S.simt_lib

# left to the GPU run: the 1080p frame (hours of interpretation)
_GPU_ONLY = {"test_1080p_knot_batch_of_16"}


@pytest.fixture(autouse=True)
def _point_frames_tests_at_the_interpreter(monkeypatch, simt_lib):
    monkeypatch.setattr(G, "CUDA_LIB", simt_lib)


for _name in sorted(dir(G)):
    if _name.startswith("test_") and _name not in _GPU_ONLY:
        globals()["test_simt_" + _name[5:]] = getattr(G, _name)


def test_simt_group_of_three_devices(simt_lib):
    """A group context of three interpreter devices: every member renders its row bands of the batch, one exchange at the end."""
    sc = scenes.knot_room(40, 30, 3, 2, nu=30, nv=6)
    b, s = G.render_both(simt_lib, sc, 3, devices=[0, 1, 2], options={"kernel": 2})
    G.assert_same(b, s, "group of three")
    ref = G.render_both(ORACLE_LIB, sc, 3)[0]
    assert_bit_equal(b["accum"], ref["accum"], "group of three vs the oracle")
    assert_bit_equal(b["frame"], ref["frame"], "group of three vs the oracle, FrameRender")


@pytest.mark.parametrize("order", ["1", "2"])
def test_simt_batch_does_not_depend_on_the_lane_schedule(simt_lib, monkeypatch, order):
    monkeypatch.setenv("RT_SIMT_ORDER", order)
    sc = scenes.knot_room(32, 16, max_bounces=5, rays_per_pixel=2, nu=40, nv=8, glass=True)
    G.check(sc, 3, ({"kernel": 0}, {"kernel": 1}, {"kernel": 2, "countStats": 1}, {"kernel": 2, "poolSlots": 32, "sortRays": 1}))
