"""The named-image tests of tests/test_gpu_named_images.py, pointed at the SIMT interpreter build of the kernels (see
tests/test_simt_kernels.py), so that they run in the CPU suite; and the group of two interpreter devices."""
import pytest

import test_gpu_named_images as G
import test_simt_kernels as S

simt_lib = S.simt_lib

_GPU_ONLY = {"test_group_leader"}      # real devices; the interpreter's group is below


@pytest.fixture(autouse=True)
def _point_named_image_tests_at_the_interpreter(monkeypatch, simt_lib):
    monkeypatch.setattr(G, "CUDA_LIB", simt_lib)


for _name in sorted(dir(G)):
    if _name.startswith("test_") and _name not in _GPU_ONLY:
        globals()["test_simt_" + _name[5:]] = getattr(G, _name)


def test_simt_group_leader_of_two_devices(simt_lib):
    G.check_group_leader(simt_lib, [0, 1])
