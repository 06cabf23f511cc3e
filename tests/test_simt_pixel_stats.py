"""The per-pixel counter tests of tests/test_gpu_pixel_stats.py, pointed at the SIMT interpreter build of the kernels (see
tests/test_simt_kernels.py), so that they run in the CPU suite; plus what only the interpreter build and the oracle can show on a
CPU: row-band tiles of three 'ranks', and known answers of scenes whose counts follow from their construction."""
import numpy as np
import pytest

from conftest import ORACLE_LIB
from ray_tracing_b200 import scenes
import test_gpu_pixel_stats as G
import test_simt_kernels as S

simt_lib = S.simt_lib

# left to the GPU run: the 640x360 frame (minutes of interpretation)
_GPU_ONLY = {"test_sparse_pixels_of_a_large_scene_against_the_oracle"}


@pytest.fixture(autouse=True)
def _point_pixel_stats_tests_at_the_interpreter(monkeypatch, simt_lib):
    monkeypatch.setattr(G, "CUDA_LIB", simt_lib)


for _name in sorted(dir(G)):
    if _name.startswith("test_") and _name not in _GPU_ONLY:
        globals()["test_simt_" + _name[5:]] = getattr(G, _name)


def test_simt_row_band_tiles_add_up_to_the_whole_image(simt_lib):
    """Three row-band 'ranks' (bands of 8 rows): each counts only its own rows, and the three images add up to one context's."""
    sc = scenes.knot_room(40, 30, 4, 2, nu=60, nv=8)
    _, _, _, whole = G.run(simt_lib, sc)
    total = {k: np.zeros(whole.shape, dtype=np.uint64) for k in G.FIELDS}
    for r in range(3):
        _, _, st, pix = G.run(simt_lib, sc, tile=(r, 3, 8))
        G.assert_sums_match(pix, st, f"rank {r}")
        rows = (np.arange(sc.height) // 8) % 3 == r
        assert not pix["rays"][~rows].any() and pix["rays"][rows].min() > 0
        for k in G.FIELDS:
            total[k] += pix[k]
    for k in G.FIELDS:
        assert np.array_equal(total[k], whole[k].astype(np.uint64)), k


def _single_leaf_models(k, n_side):
    """k small grids of 2 * n_side^2 triangles each, BVH quality Disabled (one leaf), far off-screen behind the camera."""
    v, idx = [], []
    for j in range(n_side + 1):
        for i in range(n_side + 1):
            v.append((i / n_side, j / n_side, 0.0))
    for j in range(n_side):
        for i in range(n_side):
            a = j * (n_side + 1) + i
            idx += [a, a + 1, a + n_side + 2, a, a + n_side + 2, a + n_side + 1]
    v = np.array(v, dtype=np.float32)
    mesh = scenes.MeshDesc(v, np.array(idx, dtype=np.int32), np.tile(np.float32([[0, 0, 1]]), (len(v), 1)))
    models = []
    for m in range(k):
        l2w, w2l = scenes.trs(position=(3.0 * m, 0.0, -50.0))
        models.append(scenes.ModelDesc(0, l2w, w2l, scenes.material(diffuse=(0.5, 0.5, 0.5))))
    return mesh, models


@pytest.mark.parametrize("lib_name", ["oracle", "simt"])
def test_simt_known_answers(lib_name, simt_lib):
    lib = ORACLE_LIB if lib_name == "oracle" else simt_lib
    spp = 3
    # an empty scene: every sample is one ray that tests nothing
    empty = scenes.Scene(name="empty", width=16, height=8, settings=dict(maxBounceCount=4, numRaysPerPixel=spp))
    _, _, _, pix = G.run(lib, empty)
    assert np.all(pix["rays"] == spp) and not any(pix[k].any() for k in G.FIELDS[1:])
    # MaxBounceCount = 0, k models whose BVH is one leaf of n triangles: every ray tests k * n triangles and no box
    k, side = 3, 4
    mesh, models = _single_leaf_models(k, side)
    n = 2 * side * side
    sc = scenes.Scene(name="leaves", width=16, height=8, meshes=[mesh], models=models,
                      settings=dict(maxBounceCount=0, numRaysPerPixel=spp, bvhQuality=2))
    for kernel in ((0, 1, 2) if lib_name == "simt" else (None,)):
        _, _, _, pix = G.run(lib, sc, options={} if kernel is None else {"kernel": kernel})
        assert np.all(pix["rays"] == spp) and np.all(pix["triTests"] == spp * k * n) and not pix["boxTests"].any(), (lib_name, kernel)
    # a root with two leaf children (quality Low on two far-apart triangles): two box tests per model per ray
    tri2 = scenes.MeshDesc(np.float32([[0, 0, 0], [1, 0, 0], [0, 1, 0], [40, 0, 0], [41, 0, 0], [40, 1, 0]]), np.int32([0, 1, 2, 3, 4, 5]),
                       np.tile(np.float32([[0, 0, 1]]), (6, 1)))
    sc = scenes.Scene(name="two-leaves", width=16, height=8, meshes=[tri2], models=models[:2],
                      settings=dict(maxBounceCount=0, numRaysPerPixel=spp, bvhQuality=1))
    for kernel in ((0, 1, 2) if lib_name == "simt" else (None,)):
        _, _, _, pix = G.run(lib, sc, options={} if kernel is None else {"kernel": kernel})
        assert np.all(pix["rays"] == spp) and np.all(pix["boxTests"] == spp * 2 * 2), (lib_name, kernel)
