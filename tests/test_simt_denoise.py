"""The rtDenoise tests of tests/test_gpu_denoise.py, pointed at the SIMT interpreter build of the kernels (see tests/test_simt_kernels.py),
so that they run in the CPU suite at a smaller image size — minus the cases that need torch CUDA tensors or minutes of interpretation —
plus a third restatement of the filter in numpy (independent of the oracle and the kernel) and the quality gate: the denoised image is
closer to a high-sample render than the noisy mean, by a committed factor."""
import ctypes as C
import sys

import numpy as np
import pytest

from conftest import ORACLE_LIB, REPO, assert_bit_equal
from ray_tracing_b200 import capi, scenes
import test_gpu_denoise as D
import test_gpu_features as F
import test_simt_kernels as S

sys.path.insert(0, REPO)
from oracle.py_oracle import exp_rt                                            # noqa: E402

simt_lib = S.simt_lib

_GPU_ONLY = {"test_group_context_is_refused", "test_device_pointer_and_stream_order", "test_720p_five_iterations_against_the_oracle_hook"}


def _memmove(ptr, arr):
    b = np.ascontiguousarray(arr).view(np.uint8).reshape(-1)
    C.memmove(ptr, b.ctypes.data, b.size)


@pytest.fixture(autouse=True)
def _point_denoise_tests_at_the_interpreter(monkeypatch, simt_lib):
    monkeypatch.setattr(D, "CUDA_LIB", simt_lib)
    monkeypatch.setattr(F, "CUDA_LIB", simt_lib)
    monkeypatch.setattr(F, "FRAME", (20, 12))
    monkeypatch.setattr(D, "write_device", _memmove)                          # the interpreter's "device" memory is host memory


for _name in sorted(dir(D)):
    if _name.startswith("test_") and _name not in _GPU_ONLY:
        globals()["test_simt_" + _name[5:]] = getattr(D, _name)


def test_simt_group_of_three_devices_is_refused(simt_lib):
    D.check_group_refusal(simt_lib, [0, 1, 2])


# ---- a third restatement: numpy float32, vectorised over pixels, one tap at a time in the stated order --------------------------------
F32 = np.float32
EXP_LIMIT = F32(103.972076416015625)
H5 = F32([0.0625, 0.25, 0.375, 0.25, 0.0625])


def restated(W, H, acc, colour, albedo, nf, iterations, sigma):
    """include/rt_b200.h's rtDenoise, written again from the header."""
    sc, sn, sz = (F32(v) for v in sigma)
    with np.errstate(all="ignore"):
        invC, invN, invZ = F32(1) / (sc * sc), F32(1) / (sn * sn), F32(1) / sz
        colour = colour.reshape(H, W, 4)
        if acc:
            A, L, N = colour, albedo.reshape(H, W, 4), nf.reshape(H, W, 4)
            bg = (A[..., 3] == 0) | (L[..., 3] == 0)
            c = A[..., :3] / A[..., 3:4]
            c[A[..., 3] == 0] = 0
            a = L[..., :3] / L[..., 3:4]
            n = N[..., :3] / L[..., 3:4]
            z = N[..., 3] / L[..., 3]
        else:
            f = nf.reshape(H, W)
            bg = f["object"] == -1
            c, a, n, z = colour[..., :3].copy(), f["albedo"].copy(), f["normal"].copy(), f["dst"].copy()
        m = np.maximum(a, F32(2.0 ** -8))                      # a is finite wherever it matters
        e = c / m
        bg = bg | ~np.isfinite(np.concatenate([c, a, n, z[..., None], e], axis=-1)).all(axis=-1)
        out = np.zeros((H, W, 4), F32)
        out[..., 3] = 1
        out[..., :3][bg] = c[bg]
        rz = invZ / z
        for k in range(iterations):
            s = 1 << k
            cK = invC * F32(4 ** k)
            sw, sr = np.zeros((H, W), F32), np.zeros((H, W, 3), F32)
            for j in range(-2, 3):
                for i in range(-2, 3):
                    ys, xs = np.mgrid[0:H, 0:W]
                    qy, qx = ys + s * j, xs + s * i
                    inside = (qx >= 0) & (qy >= 0) & (qx < W) & (qy < H)
                    qyc, qxc = np.clip(qy, 0, H - 1), np.clip(qx, 0, W - 1)
                    use = inside & ~bg[qyc, qxc] & ~bg
                    eq = e[qyc, qxc]
                    if i == 0 and j == 0:
                        w = np.full((H, W), F32(9 / 64), F32)
                    else:
                        de, dn = e - eq, n - n[qyc, qxc]
                        rd = F32(1) / F32(s * max(abs(i), abs(j)))
                        t = ((z - z[qyc, qxc]) * rz) * rd
                        Dv = (((de[..., 0] * de[..., 0] + de[..., 1] * de[..., 1]) + de[..., 2] * de[..., 2]) * cK
                              + ((dn[..., 0] * dn[..., 0] + dn[..., 1] * dn[..., 1]) + dn[..., 2] * dn[..., 2]) * invN) + t * t
                        w = np.zeros((H, W), F32)
                        ok = use & (Dv <= EXP_LIMIT)
                        w[ok] = [(H5[i + 2] * H5[j + 2]) * exp_rt(-d) for d in Dv[ok]]
                        use = ok & (w != 0)
                    sw = np.where(use, sw + w, sw)
                    sr = np.where(use[..., None], sr + w[..., None] * eq, sr)
            e = np.where(bg[..., None], e, sr / sw[..., None])
        out[..., :3][~bg] = (e * m)[~bg]
    return out


@pytest.mark.parametrize("acc", [1, 0])
def test_numpy_restatement_equals_the_oracle(acc):
    W, H = 24, 16
    for seed, adversarial in ((21, False), (22, True)):
        imgs = D.synthetic(W, H, seed, adversarial)
        colour = imgs["AccumulatedRender" if acc else "FrameRender"]
        albedo = imgs["AccumulatedAlbedo"] if acc else None
        nf = imgs["AccumulatedNormal"] if acc else imgs["FeatureFrame"]
        for k in range(1, capi.DENOISE_MAX_ITERATIONS + 1):
            for s in D.SIGMAS:
                rc, want = D.oracle_hook(W, H, acc, colour, albedo, nf, k, s)
                assert rc == capi.RT_OK
                assert_bit_equal(restated(W, H, acc, colour, albedo, nf, k, s), want, f"seed {seed} acc={acc} iterations={k} sigma={s}")


# ---- quality --------------------------------------------------------------------------------------------------------------------------
# relative MSE (mean of (x - ref)^2 / (ref^2 + 0.01) over pixels and channels) against a 1024-sample oracle render, at 32 x 24, with the
# managers' defaults (5 iterations, sigmas 64 / 1 / 0.1, the best of a sweep over 3-5 iterations, sigmaColour 2-256, sigmaNormal
# 0.25-1, sigmaDepth 0.1-1 by the worst of these four cases).  Measured (bit-exact, so the same on the interpreter, the oracle and the GPU):
#     cornell  1 frame: noisy 13.76, denoised 0.2056 (66.9x)     4 frames: noisy 2.422, denoised 0.2417 (10.0x)
#     knot     1 frame: noisy 37.12, denoised 0.4035 (92.0x)     4 frames: noisy 8.628, denoised 0.2864 (30.1x)
# The gate asks for a factor of 4.
QUALITY_FACTOR = 4.0


def rel_mse(x, ref):
    return float(np.mean((x[..., :3].astype(np.float64) - ref[..., :3]) ** 2 / (ref[..., :3].astype(np.float64) ** 2 + 0.01)))


def quality(lib, make, frames):
    """(noisy, denoised) relative MSE after `frames` frames of 1 sample, the feature images of every frame."""
    mgr, ctx = F.open_ctx(lib, make(), size=(32, 24))
    for f in range(1, frames + 1):
        ctx.set_int("Frame", f)
        ctx.dispatch_features()
        ctx.dispatch_full()
    acc = ctx.readback("AccumulatedRender")
    ctx.denoise(True)
    den = ctx.readback("DenoisedRender")
    mgr.OnDestroy()
    ref = reference(make)
    return rel_mse(acc[..., :3] / acc[..., 3:4], ref), rel_mse(den, ref)


_REFS = {}


def reference(make):
    name = make().name
    if name not in _REFS:
        sc = make()
        sc.settings = dict(sc.settings, numRaysPerPixel=64)
        mgr, ctx = F.open_ctx(ORACLE_LIB, sc, size=(32, 24))
        for f in range(1, 17):
            ctx.set_int("Frame", f)
            ctx.dispatch_full()
        acc = ctx.readback("AccumulatedRender")
        mgr.OnDestroy()
        _REFS[name] = acc[..., :3] / acc[..., 3:4]
    return _REFS[name]


QUALITY_SCENES = {"cornell": lambda: scenes.cornell_spheres(32, 24, 4, 1),
                  "knot": lambda: scenes.knot_room(32, 24, 6, 1, nu=60, nv=10)}


@pytest.mark.parametrize("name", sorted(QUALITY_SCENES))
@pytest.mark.parametrize("frames", [1, 4])
def test_simt_denoised_image_is_closer_to_a_high_sample_render(simt_lib, name, frames):
    noisy, den = quality(simt_lib, QUALITY_SCENES[name], frames)
    assert den * QUALITY_FACTOR <= noisy, f"{name} after {frames} frames: relative MSE noisy {noisy:.4g}, denoised {den:.4g}"
