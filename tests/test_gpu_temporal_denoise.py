"""rtDenoiseTemporal on the H100 (`-m gpu`): the temporal (SVGF) denoiser equals the oracle bit for bit after every frame, DenoisedRender
and TemporalFrame both: on six rendered scenes (model skipping on and off) along 8-frame camera paths at 1 spp with accumulate off
(still, pan, dolly, orbit, jump cut, resetHistory in mid-sequence, resize in mid-sequence), for 1, 3 and 5 iterations and two parameter
sets; and on synthetic images and cameras written through rtGetDevicePointer, against the oracle's orTemporalImages (NaN, infinite,
denormal and zero depths, points behind the previous camera, singular and non-finite matrices, sigmas at the edges of the accepted
range, 1x1 to 70x41).  Then the properties: a still camera reprojects onto itself, reset and jump cuts start over, resize discards the
history and ResetAccumulated does not, the call changes nothing else, rtDenoise and rtDenoiseTemporal do not affect each other, the
managers, and every refusal.  The same bodies run in the CPU suite against the SIMT interpreter build (tests/test_simt_temporal_denoise.py)."""
import ctypes as C
import math

import numpy as np
import pytest

from conftest import CUDA_LIB, ORACLE_LIB, assert_bit_equal
from ray_tracing_b200 import capi, scenes
import test_gpu_denoise as D
import test_gpu_features as F

pytestmark = pytest.mark.gpu

FRAME = (40, 24)                # size of the rendered images (the interpreter twin uses a smaller one)
FRAMES = 8
DEFAULT = (capi.TEMPORAL_SIGMA_LUMINANCE, capi.TEMPORAL_SIGMA_NORMAL, capi.TEMPORAL_SIGMA_DEPTH, capi.TEMPORAL_ALPHA)
PARAMS = [(k,) + p for p in (DEFAULT, (1.0, 0.3, 0.5, 0.5)) for k in (5, 1, 3)]     # PARAMS[0]: what the rendering contexts run
PATHS = ("still", "pan", "dolly", "orbit", "jump", "reset", "resize")
F32 = np.float32


# ---- cameras --------------------------------------------------------------------------------------------------------------------------
def rot_y(deg):
    c, s = math.cos(math.radians(deg)), math.sin(math.radians(deg))
    return np.array([[c, 0, s, 0], [0, 1, 0, 0], [-s, 0, c, 0], [0, 0, 0, 1]])


def translate(x, y, z):
    m = np.eye(4)
    m[:3, 3] = (x, y, z)
    return m


def camera_path(name, M0):
    """Per frame: (CamLocalToWorldMatrix, resetHistory, resize)."""
    M0 = np.asarray(M0, np.float64)
    pivot = M0 @ np.array([0.0, 0.0, 5.0, 1.0])
    around = lambda deg: translate(*pivot[:3]) @ rot_y(deg) @ translate(*-pivot[:3]) @ M0
    out = []
    for k in range(FRAMES):
        M = {"still": M0, "pan": M0 @ rot_y(1.5 * k), "dolly": M0 @ translate(0, 0, 0.15 * k), "orbit": around(2.0 * k),
             "jump": M0 if k < 4 else around(150.0), "reset": M0 @ rot_y(1.0 * k), "resize": M0 @ rot_y(-1.0 * k)}[name]
        out.append((M, name == "reset" and k == 4, name == "resize" and k == 4))
    return out


def view_params(fov, W, H):
    h = 2.0 * math.tan(math.radians(fov) / 2)
    return (h * W / H, h, 1.0)


def cam19(M, vp):
    return np.concatenate([np.asarray(M, F32).T.reshape(16), np.asarray(vp, F32)]).astype(F32)


# ---- the oracle's hook ----------------------------------------------------------------------------------------------------------------
def oracle_step(W, H, colour, feats, cur, prev, hist, params):
    """orTemporalImages: (rc, DenoisedRender, TemporalFrame, history out)."""
    L = C.CDLL(ORACLE_LIB)
    f = L.orTemporalImages
    vp = C.c_void_p
    f.argtypes = [C.c_int, C.c_int, vp, vp, vp, vp, vp, vp, C.c_int, vp, vp, vp]
    colour = np.ascontiguousarray(colour, F32)
    feats = np.ascontiguousarray(feats)
    cur = np.ascontiguousarray(cur, F32)
    prev = None if prev is None else np.ascontiguousarray(prev, F32)
    hist = None if hist is None else np.ascontiguousarray(hist, F32)
    hout = np.zeros(W * H * 12, F32)
    out, frame = np.zeros((H, W, 4), F32), np.zeros((H, W, 4), F32)
    p = np.asarray(params[1:], F32)
    rc = f(W, H, colour.ctypes.data, feats.ctypes.data, cur.ctypes.data, None if prev is None else prev.ctypes.data,
           None if hist is None else hist.ctypes.data, hout.ctypes.data, int(params[0]), p.ctypes.data, out.ctypes.data, frame.ctypes.data)
    return rc, out, frame, hout


def oracle_sequence(inputs, params):
    """The hook chained over a sequence of inputs: [(DenoisedRender, TemporalFrame)] per frame."""
    prev = hist = None
    size = None
    res = []
    for inp in inputs:
        if inp["reset"] or inp["size"] != size:
            prev = hist = None
        size = inp["size"]
        W, H = size
        rc, out, frame, hist = oracle_step(W, H, inp["FrameRender"], inp["FeatureFrame"], inp["cam"], prev, hist, params)
        assert rc == capi.RT_OK
        prev = inp["cam"]
        res.append((out, frame))
    return res


def product_sequence(lib, inputs, params):
    """The same inputs written into a blank context of the product, one rtDenoiseTemporal per frame."""
    ctx, size, res = None, None, []
    for inp in inputs:
        W, H = inp["size"]
        if ctx is None:
            ctx = D.blank_ctx(lib, W, H)
        elif inp["size"] != size:
            ctx.resize(W, H)
            ctx.set_ints("Resolution", [W, H])
        size = inp["size"]
        cam = inp["cam"]
        ctx.set_matrix("CamLocalToWorldMatrix", cam[:16].reshape(4, 4).T)
        ctx.set_vector("ViewParams", cam[16:])
        D.load_images(ctx, {"FrameRender": inp["FrameRender"], "FeatureFrame": inp["FeatureFrame"]})
        ctx.denoise_temporal(*params, reset_history=inp["reset"])
        res.append((ctx.readback("DenoisedRender"), ctx.temporal_frame()))
    return res


def assert_sequences_equal(got, want, what):
    assert len(got) == len(want)
    for k, ((go, gf), (wo, wf)) in enumerate(zip(got, want)):
        assert_bit_equal(go, wo, f"{what} frame {k}: DenoisedRender")
        assert_bit_equal(gf, wf, f"{what} frame {k}: TemporalFrame")


# ---- 1. rendered scenes along camera paths --------------------------------------------------------------------------------------------
def render_sequence(lib, make, path, options=None, size=None):
    """8 frames of 1 spp with accumulate off along the path, rtDenoiseTemporal(PARAMS[0]) after each: the inputs of every frame and
    the end-to-end results."""
    sc = make()
    mgr, ctx = F.open_ctx(lib, sc, options, size=size)
    ctx.set_bool("accumulate", False)
    inputs, res = [], []
    for k, (M, reset, resize) in enumerate(camera_path(path, sc.cam_local_to_world)):
        if resize:
            ctx.resize(ctx.width + 4, ctx.height + 2)
            ctx.set_ints("Resolution", [ctx.width, ctx.height])
        vp = view_params(sc.fov, ctx.width, ctx.height)
        ctx.set_matrix("CamLocalToWorldMatrix", M)
        ctx.set_vector("ViewParams", vp)
        ctx.set_int("Frame", k + 1)
        ctx.dispatch_full()
        ctx.dispatch_features()
        ctx.denoise_temporal(*PARAMS[0], reset_history=reset)
        inputs.append({"size": (ctx.width, ctx.height), "cam": cam19(M, vp), "reset": reset,
                       "FrameRender": ctx.readback("FrameRender"), "FeatureFrame": ctx.readback("FeatureFrame")})
        res.append((ctx.readback("DenoisedRender"), ctx.temporal_frame()))
    mgr.OnDestroy()
    return inputs, res


def check_scene(make, paths=None, size=None):
    for path in paths or PATHS:
        want_inputs, want = render_sequence(ORACLE_LIB, make, path, size=size)
        assert_sequences_equal(oracle_sequence(want_inputs, PARAMS[0]), want, f"{path}: the oracle's hook vs its context")
        if path in ("still", "pan", "dolly", "orbit"):
            assert want[-1][1][..., 2].max() > 1, f"{path}: no pixel kept its history"
        hooks = {p: oracle_sequence(want_inputs, p) for p in PARAMS[1:]}
        for skip in (1, 0):
            inputs, got = render_sequence(CUDA_LIB, make, path, {"modelSkip": skip}, size=size)
            for a, b in zip(inputs, want_inputs):
                assert_bit_equal(a["FrameRender"], b["FrameRender"], f"{path}: FrameRender")
            assert_sequences_equal(got, want, f"{make().name} {path} modelSkip={skip} params={PARAMS[0]}")
            if skip == 1:
                for p in PARAMS[1:]:
                    assert_sequences_equal(product_sequence(CUDA_LIB, inputs, p), hooks[p], f"{make().name} {path} params={p}")


def test_cornell_box():
    check_scene(lambda: scenes.cornell_spheres(24, 16, 4, 1))


def test_knot_room_with_glass():
    check_scene(lambda: scenes.knot_room(24, 16, 6, 1, nu=40, nv=8, glass=True))


def test_checker_soup_with_sky_defocus_and_spheres():
    check_scene(F.checker_soup)


def test_152_instanced_knots_with_the_tlas():
    check_scene(lambda: scenes.instanced_knots(24, 16, 4, 1, instances=150), paths=("pan", "jump", "resize"))


def test_ten_thousand_spheres():
    check_scene(lambda: scenes.random_soup(24, 16, 4, 1, triangles=300, spheres=10000), paths=("orbit", "reset"))


def test_unity_fixture():
    from test_round2_abi import load_fixture
    check_scene(lambda: load_fixture(24, 16), paths=("dolly", "still"))


# ---- 2. synthetic images and cameras through the oracle's hook -------------------------------------------------------------------------
def synthetic_inputs(W, H, seed, adversarial=True):
    """Five frames of random images under a still, moved, behind-the-camera, singular and non-finite previous camera."""
    r = np.random.RandomState(seed)
    base = np.array([[1, 0, 0, 0.5], [0, 1, 0, 1.0], [0, 0, 1, -4.0], [0, 0, 0, 1]])
    cams = [base, base, base @ rot_y(3.0) @ translate(0.1, 0, 0.2), base @ rot_y(120.0),
            np.diag([1.0, 0.0, 1.0, 1.0]), np.full((4, 4), np.nan), base @ translate(0, 0, 0.3), base]
    vp = (1.2, 0.7, 1.0)
    out = []
    for k, M in enumerate(cams):
        imgs = D.synthetic(W, H, seed * 10 + k, adversarial)
        feat = imgs["FeatureFrame"]
        feat["object"] = np.where(r.rand(H, W) < 0.1, -1, r.randint(0, 3, (H, W)))
        nn = np.float32([0.3, 0.2, -0.93]) + r.randn(H, W, 3).astype(F32) * 0.05
        feat["normal"] = nn / np.linalg.norm(nn, axis=-1, keepdims=True)
        feat["dst"] = F32(4.0) + r.rand(H, W).astype(F32) * 0.05
        if adversarial:
            bits = lambda u: np.uint32(u).view(F32)
            special = F32([np.nan, np.inf, -np.inf, 0.0, -0.0, bits(1), bits(0x007fffff), 1e30])
            m = r.rand(H, W) < 0.08
            feat["dst"][m] = r.choice(special, m.sum())
        out.append({"size": (W, H), "cam": cam19(M, vp), "reset": k == 7, "FrameRender": imgs["FrameRender"], "FeatureFrame": feat})
    return out


@pytest.mark.parametrize("W,H", [(1, 1), (1, 19), (23, 1), (37, 13), (70, 41)])
def test_synthetic_sequences_against_the_oracle_hook(W, H):
    for seed, adv in ((1, True), (2, True), (3, False)):
        inputs = synthetic_inputs(W, H, seed, adv)
        for p in PARAMS:
            assert_sequences_equal(product_sequence(CUDA_LIB, inputs, p), oracle_sequence(inputs, p), f"{W}x{H} seed {seed} {p}")


def test_sub_pixel_moves_against_the_oracle_hook():
    """Sideways moves of an eighth and a sixteenth of the view, and of 1e-7 either way: reprojections a fraction of a pixel off, and
    border pixels that land just inside or just outside the image."""
    W, H = 17, 9
    base = np.eye(4)
    vp = (2.0, 1.0, 1.0)
    inputs = synthetic_inputs(W, H, 4, adversarial=False)[:2]
    for k, dx in enumerate((0.125, 0.0625, 1e-7, -1e-7)):
        nxt = dict(inputs[-1], cam=cam19(base @ translate(dx, 0, 0), vp), reset=False)
        nxt["FeatureFrame"] = nxt["FeatureFrame"].copy()
        nxt["FeatureFrame"]["dst"] = 4.0
        inputs.append(nxt)
    inputs[0] = dict(inputs[0], cam=cam19(base, vp))
    inputs[1] = dict(inputs[1], cam=cam19(base, vp))
    for p in PARAMS[:2]:
        want = oracle_sequence(inputs, p)
        assert_sequences_equal(product_sequence(CUDA_LIB, inputs, p), want, f"edges {p}")
    fr = want[3][1]
    assert np.isfinite(fr[..., 0]).any()


def edge_inputs(W, H, tx, z):
    """Two frames: the previous camera translated by tx along x, then the identity camera with per-column depths z (ViewParams
    (1, 1, 1), so u = L.x / L.z + 0.5 and, with W - 1 = 16, prevX = 16 u)."""
    imgs = D.synthetic(W, H, 31, adversarial=False)
    feat = imgs["FeatureFrame"].copy()
    feat["object"], feat["albedo"], feat["normal"] = 0, 0.5, (0.0, 0.0, -1.0)
    feat["dst"] = 4.0
    cur = feat.copy()
    cur["dst"] = np.broadcast_to(np.asarray(z, F32), (H, W))
    vp = (1.0, 1.0, 1.0)
    return [{"size": (W, H), "cam": cam19(translate(tx, 0, 0), vp), "reset": False, "FrameRender": imgs["FrameRender"], "FeatureFrame": feat},
            {"size": (W, H), "cam": cam19(np.eye(4), vp), "reset": False, "FrameRender": imgs["FrameRender"], "FeatureFrame": cur}]


def edge_depths(W, H, tx, target):
    """Per column, the depth (bisected over its binary32 encodings with the oracle's hook) whose reprojection lands on `target`, or
    the nearest on the far side of it: prevX grows with the depth for tx > 0 and shrinks for tx < 0."""
    lo, hi = np.full(W, int(np.float32(1e-3).view(np.int32)), np.int64), np.full(W, int(np.float32(1e6).view(np.int32)), np.int64)
    for _ in range(40):
        mid = (lo + hi) // 2
        inputs = edge_inputs(W, H, tx, mid.astype(np.int32).view(F32))
        px = oracle_sequence(inputs, PARAMS[0])[1][1][0, :, 0]
        past = (px >= target) if tx > 0 else (px <= target)
        hi, lo = np.where(past, mid, hi), np.where(past, lo, mid)
    return hi.astype(np.int32).view(F32)


def test_reprojections_onto_the_image_edges_and_one_step_outside():
    """Depths chosen so that border reprojections land exactly on -1, 0, W - 1 and W (the limits of the footprint test and of the
    image) and on the nearest representable results on either side of them, against the oracle's hook; each value must occur."""
    W, H = 17, 2
    def around(r0):
        """prevX = 16 (r + 0.5) for r = L.x / L.z at r0 and at the nearest r on either side that changes the result."""
        out = [F32(16) * (F32(r0) + F32(0.5))]
        for d in (-np.inf, np.inf):
            r = F32(r0)
            while F32(16) * (r + F32(0.5)) == out[0]:
                r = np.nextafter(r, F32(d))
            out.append(F32(16) * (r + F32(0.5)))
        return out
    left = around(-0.5625) + around(-0.5)                  # prevX = -1 and 0, and one step to either side
    right = around(0.5) + around(0.5625)                   # prevX = W - 1 and W
    for tx, targets in ((0.25, left), (-0.25, right)):
        for target in targets:
            inputs = edge_inputs(W, H, tx, edge_depths(W, H, tx, target))
            for p in PARAMS[:2]:
                want = oracle_sequence(inputs, p)
                assert_sequences_equal(product_sequence(CUDA_LIB, inputs, p), want, f"edge {target!r} {p}")
            px = want[1][1][..., 0]
            assert (px == target).any(), f"no reprojection landed on {target!r}: {px[0]}"


def test_sigmas_at_the_edges_of_the_accepted_range():
    W, H = 33, 17
    inputs = synthetic_inputs(W, H, 5)
    tiny = float(np.float32(2.0 ** -63))
    for p in ((5, tiny * 16, 1.0, 1.0, 0.2), (1, 1.0, tiny, 1.0, 1.0), (3, 1.0, 1.0, float(np.float32(2.0 ** -126) * 4), 2.0 ** -24),
              (5, 3e38, 3e38, 3e38, 0.5)):
        assert_sequences_equal(product_sequence(CUDA_LIB, inputs, p), oracle_sequence(inputs, p), f"edge sigmas {p}")


# ---- 3. properties -------------------------------------------------------------------------------------------------------------------
def still_inputs(W, H, frames):
    one = synthetic_inputs(W, H, 6, adversarial=False)[0]
    return [dict(one, reset=False) for _ in range(frames)]


def test_a_still_camera_reprojects_onto_itself_and_counts_its_history():
    W, H = 9, 7
    frames = capi.TEMPORAL_MAX_HISTORY + 3
    inputs = still_inputs(W, H, frames)
    got = product_sequence(CUDA_LIB, inputs, PARAMS[0])
    fg = inputs[0]["FeatureFrame"]["object"] != -1
    ys, xs = np.mgrid[0:H, 0:W]
    for k, (_, fr) in enumerate(got):
        if k == 0:
            assert np.isnan(fr[..., :2]).all()
        else:
            assert (fr[..., 0][fg] == xs[fg]).all() and (fr[..., 1][fg] == ys[fg]).all()
        assert (fr[..., 2][fg] == min(k + 1, capi.TEMPORAL_MAX_HISTORY)).all(), k
    assert_sequences_equal(got, oracle_sequence(inputs, PARAMS[0]), "still")


def test_reset_and_jump_cut_start_over_as_a_fresh_context():
    W, H = 16, 12
    inputs = synthetic_inputs(W, H, 7, adversarial=False)
    with_reset = [dict(i, reset=(k == 3)) for k, i in enumerate(inputs[:4])]
    got = product_sequence(CUDA_LIB, with_reset, PARAMS[0])
    fresh = product_sequence(CUDA_LIB, with_reset[3:], PARAMS[0])
    assert_sequences_equal(got[3:], fresh, "resetHistory = 1 vs a fresh context")
    fg = inputs[3]["FeatureFrame"]["object"] != -1
    assert (got[3][1][..., 2][fg] == 1).all()
    # a jump cut (the camera turned away): no tap survives, every pixel starts over
    jump = [dict(inputs[0], reset=False), dict(inputs[1], cam=cam19(np.asarray(rot_y(180.0)), (1.2, 0.7, 1.0)), reset=False)]
    got = product_sequence(CUDA_LIB, jump, PARAMS[0])
    fg = jump[1]["FeatureFrame"]["object"] != -1
    assert (got[1][1][..., 2][fg] == 1).all()


def test_resize_discards_the_history_and_reset_accumulated_does_not():
    for lib in (ORACLE_LIB, CUDA_LIB):
        mgr, ctx = F.open_ctx(lib, F.checker_soup())
        ctx.set_bool("accumulate", False)
        lens = []
        for k in range(4):
            ctx.set_int("Frame", k + 1)
            ctx.dispatch_full()
            ctx.dispatch_features()
            if k == 2:
                ctx.dispatch_full(capi.RT_KERNEL_RESET_ACCUMULATED)
            ctx.denoise_temporal()
            lens.append(ctx.temporal_frame()[..., 2].max())
        assert lens == [1, 2, 3, 4], (lib, lens)
        w, h = ctx.width, ctx.height
        ctx.resize(w + 8, h)
        ctx.set_ints("Resolution", [w + 8, h])
        fr = ctx.temporal_frame()
        assert fr.shape == (h, w + 8, 4) and not fr.any(), f"{lib}: a resize zeroes TemporalFrame"
        ctx.dispatch_full()
        ctx.dispatch_features()
        ctx.denoise_temporal()
        assert ctx.temporal_frame()[..., 2].max() == 1, f"{lib}: a resize discards the history"
        mgr.OnDestroy()


def test_the_call_changes_nothing_else_and_rt_denoise_is_independent():
    make = F.checker_soup
    results, den = [], []
    for with_temporal in (False, True):
        mgr, ctx = F.open_ctx(CUDA_LIB, make(), {"countStats": 1})
        ctx.reset_stats()
        for f in range(1, 4):
            mgr.RenderFeatures()
            mgr.RenderFrame()
            if with_temporal:
                before = {n: ctx.readback(n) for n in D.INPUTS}
                st, pix, frame_no = ctx.stats(), ctx.pixel_stats(), mgr.numAccumulatedFrames
                ctx.denoise_temporal()
                for n in D.INPUTS:
                    assert ctx.readback(n).tobytes() == before[n].tobytes(), f"{n} changed by rtDenoiseTemporal"
                assert ctx.stats() == st and ctx.pixel_stats().tobytes() == pix.tobytes() and mgr.numAccumulatedFrames == frame_no
            ctx.denoise(True, 3)
            den.append(ctx.readback("DenoisedRender"))
        results.append({n: ctx.readback(n) for n in D.INPUTS})
        mgr.OnDestroy()
    for n in D.INPUTS:
        assert results[1][n].tobytes() == results[0][n].tobytes(), f"{n}: later dispatches render other bits after rtDenoiseTemporal"
    for a, b in zip(den[:3], den[3:]):
        assert_bit_equal(b, a, "rtDenoise with rtDenoiseTemporal interleaved")


def test_temporal_history_does_not_depend_on_interleaved_rt_denoise_and_repeats():
    inputs = synthetic_inputs(20, 12, 8, adversarial=False)[:4]
    plain = product_sequence(CUDA_LIB, inputs, PARAMS[0])
    ctx, res = D.blank_ctx(CUDA_LIB, 20, 12), []
    for inp in inputs:
        cam = inp["cam"]
        ctx.set_matrix("CamLocalToWorldMatrix", cam[:16].reshape(4, 4).T)
        ctx.set_vector("ViewParams", cam[16:])
        D.load_images(ctx, {"FrameRender": inp["FrameRender"], "FeatureFrame": inp["FeatureFrame"]})
        ctx.denoise(False, 4, 0.5, 0.3, 0.2)
        ctx.denoise_temporal(*PARAMS[0])
        res.append((ctx.readback("DenoisedRender"), ctx.temporal_frame()))
        ctx.denoise(True, 2)
    assert_sequences_equal(res, plain, "rtDenoise interleaved")
    assert_sequences_equal(product_sequence(CUDA_LIB, inputs, PARAMS[0]), plain, "repeated")


def test_a_refused_call_leaves_the_history_and_the_previous_camera():
    W, H = 20, 12
    inputs = synthetic_inputs(W, H, 9, adversarial=False)[:3]
    want = product_sequence(CUDA_LIB, inputs, PARAMS[0])
    assert_sequences_equal(want, oracle_sequence(inputs, PARAMS[0]), "plain")
    ctx, res = D.blank_ctx(CUDA_LIB, W, H), []
    L, h = ctx._L, ctx.handle
    for k, inp in enumerate(inputs):
        if k > 0:                          # refused calls under another camera and other images: nothing may change
            other = synthetic_inputs(W, H, 10, adversarial=False)[2]
            ctx.set_matrix("CamLocalToWorldMatrix", other["cam"][:16].reshape(4, 4).T)
            D.load_images(ctx, {"FrameRender": other["FrameRender"]})
            assert L.rtDenoiseTemporal(h, 5, 4.0, 1.0, 0.1, 1.5, 0) == capi.RT_E_INVALID
            assert L.rtDenoiseTemporal(h, 5, 4.0, 1.0, 0.1, 0.1, 2) == capi.RT_E_INVALID
            ctx.set_ints("Resolution", [W - 1, H])
            assert L.rtDenoiseTemporal(h, 5, 4.0, 1.0, 0.1, 0.1, 0) == capi.RT_E_STATE
            ctx.set_ints("Resolution", [W, H])
        cam = inp["cam"]
        ctx.set_matrix("CamLocalToWorldMatrix", cam[:16].reshape(4, 4).T)
        ctx.set_vector("ViewParams", cam[16:])
        D.load_images(ctx, {"FrameRender": inp["FrameRender"], "FeatureFrame": inp["FeatureFrame"]})
        ctx.denoise_temporal(*PARAMS[0])
        res.append((ctx.readback("DenoisedRender"), ctx.temporal_frame()))
    assert_sequences_equal(res, want, "refused calls in between")


def test_managers_equal_the_raw_context():
    make = lambda: scenes.knot_room(24, 16, 4, 1, nu=40, nv=8, glass=True)
    for lib in (ORACLE_LIB, CUDA_LIB):
        got = []
        for via_mgr in (True, False):
            mgr, ctx = F.open_ctx(lib, make())
            mgr.accumulate = False
            for _ in range(3):
                mgr.RenderFeatures()
                mgr.RenderFrame()
                if via_mgr:
                    mgr.DenoiseTemporal()
                    got.append(mgr.denoised_result)
                else:
                    ctx.denoise_temporal()
                    got.append(ctx.readback("DenoisedRender"))
            mgr.OnDestroy()
        for k in range(3):
            assert_bit_equal(got[k], got[k + 3], f"{lib}: DenoiseTemporal() vs rtDenoiseTemporal, frame {k}")


def test_every_refusal_and_state():
    sc = scenes.knot_room(16, 12, 3, 1, nu=30, nv=6)
    for lib in (ORACLE_LIB, CUDA_LIB):
        mgr = F.T.open_mgr(lib, sc, enable=False)
        ctx, L, h = mgr.context, mgr.context._L, mgr.context.handle
        ok = (3, 1.0, 0.5, 0.25, 0.2, 0)
        assert L.rtDenoiseTemporal(h, *ok) == capi.RT_E_STATE                  # before rtResize
        mgr.OnEnable()
        assert L.rtDenoiseTemporal(h, *ok) == capi.RT_E_STATE                  # before the first rtDispatchFeatures
        with pytest.raises(capi.RtError) as e:
            ctx.temporal_frame()
        assert e.value.code == capi.RT_E_STATE, lib
        if lib == CUDA_LIB:
            with pytest.raises(capi.RtError) as e:
                ctx.device_pointer("TemporalFrame")
            assert e.value.code == capi.RT_E_STATE
        ctx.dispatch_features()
        inf, nan = float("inf"), float("nan")
        assert L.rtDenoiseTemporal(None, *ok) == capi.RT_E_INVALID
        for bad in ((0, 1.0, 0.5, 0.25, 0.2, 0), (6, 1.0, 0.5, 0.25, 0.2, 0), (3, 0.0, 0.5, 0.25, 0.2, 0), (3, -1.0, 0.5, 0.25, 0.2, 0),
                    (3, inf, 0.5, 0.25, 0.2, 0), (3, nan, 0.5, 0.25, 0.2, 0), (3, 1.0, 0.0, 0.25, 0.2, 0), (3, 1.0, inf, 0.25, 0.2, 0),
                    (3, 1.0, 0.5, -0.0, 0.2, 0), (3, 1.0, 0.5, nan, 0.2, 0), (3, 1.0, 2.0 ** -64, 0.25, 0.2, 0),
                    (3, 1.0, 0.5, 2.0 ** -140, 0.2, 0), (3, 2.0 ** -140, 0.5, 0.25, 0.2, 0),
                    (3, 1.0, 0.5, 0.25, 0.0, 0), (3, 1.0, 0.5, 0.25, -0.1, 0), (3, 1.0, 0.5, 0.25, 1.5, 0), (3, 1.0, 0.5, 0.25, nan, 0),
                    (3, 1.0, 0.5, 0.25, 0.2, 2), (3, 1.0, 0.5, 0.25, 0.2, -1)):
            assert L.rtDenoiseTemporal(h, *bad) == capi.RT_E_INVALID, (lib, bad)
        assert L.rtDenoiseTemporal(h, 3, 1.0, 0.5, 0.25, 1.0, 1) == capi.RT_OK
        out = np.zeros(16 * 12 * 5, np.float32)
        assert L.rtReadback(h, b"TemporalFrame", out.ctypes.data, out.nbytes) == capi.RT_E_INVALID
        ctx.set_ints("Resolution", [8, 12])
        assert L.rtDenoiseTemporal(h, *ok) == capi.RT_E_STATE
        ctx.set_ints("Resolution", [16, 12])
        ctx.set_tile(0, 2, 4)
        assert L.rtDenoiseTemporal(h, *ok) == capi.RT_E_STATE
        ctx.set_tile(0, 1, 1)
        assert L.rtDenoiseTemporal(h, *ok) == capi.RT_OK
        mgr.OnDestroy()


# ---- 4. GPU only ----------------------------------------------------------------------------------------------------------------------
def test_group_context_is_refused():
    torch = pytest.importorskip("torch")
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import ray_tracing_b200 as rt
    mgr = rt.RayComputeManager(CUDA_LIB, devices=[0, 1])
    scenes.apply(scenes.knot_room(16, 12, 3, 1, nu=30, nv=6), mgr)
    mgr.OnEnable()
    with pytest.raises(capi.RtError) as e:
        mgr.context.denoise_temporal()
    assert e.value.code == capi.RT_E_STATE and "group" in str(e.value)
    mgr.OnDestroy()


def test_device_pointer_and_stream_order():
    """rtDenoiseTemporal on a caller's stream, TemporalFrame and DenoisedRender copied on that stream right after it."""
    torch = pytest.importorskip("torch")
    W, H = 64, 40
    inputs = synthetic_inputs(W, H, 11)[:3]
    want = oracle_sequence(inputs, PARAMS[0])
    ctx = D.blank_ctx(CUDA_LIB, W, H)
    stream = torch.cuda.Stream()
    ctx.set_stream(stream.cuda_stream)
    for inp, (wo, wf) in zip(inputs, want):
        cam = inp["cam"]
        ctx.set_matrix("CamLocalToWorldMatrix", cam[:16].reshape(4, 4).T)
        ctx.set_vector("ViewParams", cam[16:])
        D.load_images(ctx, {"FrameRender": inp["FrameRender"], "FeatureFrame": inp["FeatureFrame"]})
        ctx.denoise_temporal(*PARAMS[0])
        copies = []
        for name in ("DenoisedRender", "TemporalFrame"):
            ptr, nbytes = ctx.device_pointer(name)
            assert nbytes == W * H * 16

            class _Dev:
                __cuda_array_interface__ = {"shape": (nbytes // 4,), "typestr": "<f4", "data": (ptr, False), "version": 3, "strides": None}
            with torch.cuda.stream(stream):
                copies.append(torch.as_tensor(_Dev(), device="cuda").clone())
        stream.synchronize()
        assert_bit_equal(copies[0].cpu().numpy().reshape(H, W, 4), wo, "DenoisedRender on a caller stream")
        assert_bit_equal(copies[1].cpu().numpy().reshape(H, W, 4), wf, "TemporalFrame on a caller stream")
    ctx.set_stream(0)


def test_720p_against_the_oracle_hook():
    W, H = 1280, 720
    inputs = synthetic_inputs(W, H, 13)[:3]
    assert_sequences_equal(product_sequence(CUDA_LIB, inputs, PARAMS[0]), oracle_sequence(inputs, PARAMS[0]), "720p")
