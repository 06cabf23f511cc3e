"""Traversal stacks where they wrap, spill and fill, on the H100 (`-m gpu`): the bodies of tests/test_traversal_stacks.py against
librt_b200.so — deep combs at every ring wrap, builder-made lines of up to 2^16 triangles, deep models one after another with the
sphere accelerator and the TLAS, frame batches, the queries and the peeled sphere line, all bit for bit against the oracle."""
import pytest

from conftest import CUDA_LIB
import test_traversal_stacks as S

pytestmark = pytest.mark.gpu


def test_combs_equal_oracle_on_gpu():
    S.combs_equal_oracle(CUDA_LIB, size=(64, 36))


def test_builder_made_lines_equal_oracle_on_gpu():
    S.builder_lines_equal_oracle(CUDA_LIB)


def test_stack_state_across_models_on_gpu():
    S.stack_state_across_models(CUDA_LIB, size=(96, 54))


def test_stack_state_across_shade_phases_on_gpu():
    """An image of many pixels per resident lane, 32-slot pools and 31 tail lanes: deep rays stay in flight across shade phases."""
    sc, tree = S.multi_model_scene(depth=33, spheres=True, size=(480, 270))
    S.check_against_oracle(CUDA_LIB, sc, tree, [{"kernel": 2, "poolSlots": 32, "tailLanes": 31}, {"kernel": 2, "poolSlots": 32, "tailLanes": 31, "countStats": 1},
                                                {"kernel": 2, "poolSlots": 96, "tailLanes": 16, "sortRays": 1}, {"kernel": 2}])


def test_queries_down_the_comb_on_gpu():
    S.queries_down_the_comb(CUDA_LIB)


def test_peeled_sphere_line_on_gpu():
    S.peeled_sphere_line(CUDA_LIB)
