"""The rtDispatchFeatures / rtCameraRays tests of tests/test_gpu_features.py, pointed at the SIMT interpreter build of the kernels (see
tests/test_simt_kernels.py), so that they run in the CPU suite at a smaller image size — minus the 4K case and the cases that need
torch CUDA tensors — plus a group context of three interpreter devices (refused) and the feature dispatch under the interpreter's
other two lane orders (RT_SIMT_ORDER)."""
import pytest

from ray_tracing_b200 import scenes
import test_gpu_features as F
import test_gpu_trace_paths as G
import test_simt_kernels as S

simt_lib = S.simt_lib

# left to the GPU run: the 4K case (hours of interpretation) and the ones that need torch and real devices
_GPU_ONLY = {"test_4k_features_on_the_871k_triangle_cluster_against_a_sparse_oracle_sample", "test_group_context_is_refused",
             "test_device_pointer_forms_on_the_context_stream_and_a_caller_stream"}


@pytest.fixture(autouse=True)
def _point_feature_tests_at_the_interpreter(monkeypatch, simt_lib):
    monkeypatch.setattr(F, "CUDA_LIB", simt_lib)
    monkeypatch.setattr(G, "CUDA_LIB", simt_lib)
    monkeypatch.setattr(F, "FRAME", (20, 12))


for _name in sorted(dir(F)):
    if _name.startswith("test_") and _name not in _GPU_ONLY:
        globals()["test_simt_" + _name[5:]] = getattr(F, _name)


def test_simt_group_of_three_devices_is_refused(simt_lib):
    F.check_group_refusal(simt_lib, [0, 1, 2])


@pytest.mark.parametrize("order", ["1", "2"])
def test_simt_features_do_not_depend_on_the_lane_schedule(simt_lib, monkeypatch, order):
    monkeypatch.setenv("RT_SIMT_ORDER", order)
    F.check_scene(F.checker_soup, ({"modelSkip": 1}, {"countStats": 1, "modelSkip": 1}))
    F.check_scene(lambda: scenes.instanced_knots(24, 16, 4, 1, instances=150), ({"tlas": 1, "modelSkip": 1},), frames=(1,))
