"""The arithmetic contract (DESIGN.md section 2), primitive by primitive, on the GPU: every device routine the path uses, compiled
with the product's flags into the probe library tests/gpu_probe/rt_probe.cu, against the oracle's restatement (orProbe) bit for bit
and against float64 references.

Whole-frame parity only reaches the inputs that some pixel happens to produce; here the scalar routines see every one of the 2^32
input patterns (or the whole domain the path feeds them), and the intersection and shading primitives see seeded adversarial
classes: axis-aligned rays, origins on slab planes, edges and vertices, the culling threshold, tangent rays, total internal
reflection, special values.  A NaN must be a NaN on both sides; its sign and payload are not compared (conftest.assert_bit_equal).

The same tests run on the CPU, on the SIMT interpreter build of the same probe source, over every 4,096th pattern and 10^5 cases
per primitive (tests/test_simt_arith_contract.py).  Run with -s (or -rP) to see the per-routine report: inputs compared, worst
float64 error and where it occurred.
"""
import importlib.util
import json
import os

import numpy as np
import pytest

from conftest import GOLDEN, ORACLE_LIB, REPO

pytestmark = pytest.mark.gpu


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


probe_build = _load("gpu_probe_build", os.path.join(REPO, "tests", "gpu_probe", "build.py"))
P = _load("gpu_probe_lib", os.path.join(REPO, "tests", "gpu_probe", "probe_lib.py"))

# SunFocus of the path: the manager's default, the committed Unity fixture, and the five shipped scenes (their manager blocks, read
# once from the reference's scene files: every one says `sunFocus: 500`).  GetEnvironmentLight raises to 1000 / SunFocus.
SUN_FOCUS = {"default": 500.0, "fixture": 400.0, "Glass Dragon": 500.0, "Glass Balls": 500.0, "Sphere Refract": 500.0, "Splash": 500.0, "Text": 500.0}
POW_EXPONENTS = sorted({0.35, 0.41666666} | {float(np.float32(1000.0) / np.float32(f)) for f in SUN_FOCUS.values()})
TWO_PI_BITS = int(P.f32bits(6.2831852)[()])          # the largest angle the path feeds sin / cos (6.2831852 * RandomValue <= 6.2831852)
ONE_BITS = 0x3F800000
E5_BITS = int(P.f32bits(1e5)[()])


@pytest.fixture(scope="module")
def libs():
    # RT_PROBE_LIB: test a probe built with other code-generation flags (probe_build.build_gpu(flags=..., out=...))
    return P.Lib(os.environ.get("RT_PROBE_LIB") or probe_build.build_gpu(), oracle=False), P.Lib(ORACLE_LIB, oracle=True)


@pytest.fixture(scope="module")
def scale():
    """GPU: every pattern, 10^7 cases per primitive, 10^8 RNG states and random pow pairs."""
    return dict(start=0, stride=1, chunk=1 << 26, cases=10 ** 7, batch=10 ** 6, states=10 ** 8, pairs=10 ** 8)


def _span(lo, hi, sc):
    """(start, count) of the scan over bit patterns lo..hi with the scale's stride."""
    start = lo + (sc["start"] % sc["stride"] if sc["stride"] > 1 else 0)
    return start, (hi - start) // sc["stride"] + 1


def _full(sc):
    return sc["start"], (1 << 32) // sc["stride"]


def _report(what, n, extra="", vs_oracle=True):
    head = f"{n:,} inputs compared bitwise with the oracle, 0 differ" if vs_oracle else f"{n:,} cases"
    print(f"\n[arith] {what}: {head}{'; ' + extra if extra else ''}", flush=True)


def _at(x):
    return f"x = {np.uint32(x).view(np.float32)!r} ({int(x):#010x})" if x is not None else "-"


# ---- section 2: the scalar routines over every input pattern --------------------------------------------------------------------------

def _special_inputs():
    """Special values and the edges of every routine's domain, with their float neighbours."""
    base = np.array([0.0, 1e-45, 1.1754942e-38, 1.17549435e-38, 3.4028235e38, np.inf, np.nan, 1.0, 0.5, 2.0, 0.0031308, 0.04045,
                     88.72283935546875, 103.972076416015625, 1e5, 6.2831852, 3.1415927, 1.5707964, 0.7853982, 1.41421354, 0.70710677,
                     33554432.0, 4294967296.0, 4294967040.0, 255.5, 1e-8, 1e30], dtype=np.float32)
    v = np.concatenate([base, -base])
    v = np.concatenate([v, np.nextafter(v, np.float32(np.inf)), np.nextafter(v, np.float32(-np.inf))])
    bits = np.concatenate([P.f32bits(v), np.array([0x7fc00000, 0xffc00000, 0x7f800001, 0x7fa12345, 0xffffffff, 0x80000000], dtype=np.uint32)])
    return np.unique(bits)


def test_scalar_routines_on_special_values(libs):
    """Every one-argument scalar routine on +-0, subnormals, +-inf, NaNs with payloads and the edges of each domain (the sin/cos
    domain +-1e5, exp's overflow / underflow thresholds, the sRGB knee, 2^32 for the float -> uint conversion) and their neighbours."""
    dev, orc = libs
    x = _special_inputs()
    for name in ("log", "exp", "sin", "cos", "sincos", "saturate", "f2uint_rz", "display_encode"):
        P.compare_cases(dev, orc, name, x[:, None])
    _report("special values of log exp sin cos sincos saturate f2uint_rz display_encode", len(x))


def test_log_and_exp_every_pattern_bitwise_and_within_one_ulp(libs, scale):
    """log_rt and exp_rt against orc::log / orc::exp on every input pattern; log < 1 ulp of float64 log on every positive float, exp
    < 1 ulp of float64 exp wherever float64 exp rounded to binary32 is finite (subnormal results included; an early overflow to inf
    counts as an infinite error)."""
    dev, orc = libs
    for name, ref, domain in (("log", np.log, lambda x: (x > 0) & np.isfinite(x)), ("exp", np.exp, lambda x: np.isfinite(x))):
        worst = P.Worst()

        def analyse(xb, out, ref=ref, domain=domain, worst=worst):
            x = xb.view(np.float32)
            y = out[:, 0].view(np.float32)
            with np.errstate(all="ignore"):
                r = ref(x.astype(np.float64))
                err = np.abs(y.astype(np.float64) - r) / P.ulp32(r)
                m = domain(x) & np.isfinite(r.astype(np.float32))     # where the correctly rounded result is finite, whatever the device returned
            err[~m] = 0.0
            worst.add(err, xb, int(np.count_nonzero(m)))

        lim = 0x7F800000 if name == "log" else 0x42D00000
        n = P.scan(dev, orc, name, *_full(scale), stride=scale["stride"], chunk=scale["chunk"], analyse=analyse,
                   arrays_for=lambda a, b, lim=lim: (a & 0x7FFFFFFF) < lim or (b & 0x7FFFFFFF) < lim or scale["stride"] > 1)
        _report(f"{name}_rt", n, f"worst error {worst.err:.3f} ulp of float64 {name} at {_at(worst.at)} over {worst.n:,} inputs with a finite result")
        assert worst.n > 0 and worst.err < 1.0


def test_sin_and_cos_every_pattern_bitwise_domain_and_accuracy(libs, scale):
    """sin_rt and cos_rt against orc::sin / orc::cos on every input pattern; NaN exactly outside [-1e5, 1e5] (and for NaN); within
    1.5e-7 of float64 on [0, 2pi], the angles the path feeds them (special values and the neighbours of +-1e5: the test above).  The worst error on (2pi, 1e5] is reported, not asserted."""
    dev, orc = libs
    for name, ref in (("sin", np.sin, ), ("cos", np.cos)):
        path, beyond, nan_wrong = P.Worst(), P.Worst(), []

        def analyse(xb, out, ref=ref, path=path, beyond=beyond, nan_wrong=nan_wrong):
            x = xb.view(np.float32)
            y = out[:, 0].view(np.float32)
            nan_wrong.append(int(np.count_nonzero(np.isnan(y) != ~(np.abs(x) <= 1e5))))
            with np.errstate(all="ignore"):
                err = np.abs(y.astype(np.float64) - ref(x.astype(np.float64)))
            for w, m in ((path, xb <= TWO_PI_BITS), (beyond, (xb > TWO_PI_BITS) & (xb <= E5_BITS))):
                w.add(np.where(m, err, 0.0), xb, int(np.count_nonzero(m)))

        # arrays (and the NaN-ness check) for the chunks of [0, 1e5] and the one holding -1e5; everywhere else the bit equality with
        # orc::sin / orc::cos, which return NaN outside [-1e5, 1e5], decides it
        n = P.scan(dev, orc, name, *_full(scale), stride=scale["stride"], chunk=scale["chunk"], analyse=analyse,
                   arrays_for=lambda a, b: scale["stride"] > 1 or a <= E5_BITS or a <= (E5_BITS | 0x80000000) <= b)
        _report(f"{name}_rt", n, f"worst |error| {path.err:.3e} on [0, 2pi] at {_at(path.at)}; {beyond.err:.3e} on (2pi, 1e5] at {_at(beyond.at)}")
        assert sum(nan_wrong) == 0, f"{name}_rt: {sum(nan_wrong)} inputs where NaN-ness does not match the domain [-1e5, 1e5]"
        assert path.n > 0 and path.err < 1.5e-7


def test_sincos_equals_the_oracle_and_the_devices_own_sin_and_cos(libs, scale):
    """sincos_rt (RandomPointInCircle) on every pattern: the oracle's separate sin and cos, and the device's own sin_rt / cos_rt, give
    the same bits (compared through the per-output digests of the same scan)."""
    dev, orc = libs
    start, count = _full(scale)
    done = 0
    while done < count:
        m = min(scale["chunk"], count - done)
        base = (start + done * scale["stride"]) & 0xFFFFFFFF
        kw = dict(n=m, base=base, stride=scale["stride"], arrays=False)
        _, dsc = dev.run("sincos", **kw)
        _, osc = orc.run("sincos", **kw)
        _, ds = dev.run("sin", **kw)
        _, dc = dev.run("cos", **kw)
        assert np.array_equal(dsc, osc), f"sincos_rt differs from the oracle's sin / cos in the chunk at {base:#x}"
        assert dsc[0] == ds[0] and dsc[1] == dc[0], f"sincos_rt differs from the device's sin_rt / cos_rt in the chunk at {base:#x}"
        done += m
    _report("sincos_rt (vs the oracle, vs sin_rt / cos_rt)", done)


MINMAX_PARTNERS = np.array([0x00000000, 0x80000000, 0x00000001, 0x80000001, 0x007FFFFF, 0x807FFFFF, 0x3F800000, 0xBF800000,
                            0x7F800000, 0xFF800000, 0x7FC00000, 0x7FA12345], dtype=np.uint32)


def test_saturate_fmin_fmax_every_pattern(libs, scale):
    """saturate1 on every pattern, and fminf / fmaxf of every pattern with each partner of the special set (+-0, +-smallest and
    largest subnormal, +-1, +-inf, a quiet NaN, a NaN with payload) against orc::min / orc::max: NaN-ignoring, -0 below +0.  In the
    product saturate1 is lowered to max/min in most places and to cvt.sat.f32.f32 in k_display and one pooled kernel
    (test_ptx_contract.py), so this is where both lowerings meet the contract."""
    dev, orc = libs
    n = P.scan(dev, orc, "saturate", *_full(scale), stride=scale["stride"], chunk=scale["chunk"])
    _report("saturate1", n)
    for name in ("fmin", "fmax"):
        for p in MINMAX_PARTNERS:
            n = P.scan(dev, orc, name, *_full(scale), stride=scale["stride"], partner=int(p), chunk=scale["chunk"])
        _report(f"{name}f x {len(MINMAX_PARTNERS)} partners", n * len(MINMAX_PARTNERS))


def test_min_max_saturate_contract_on_special_pairs(libs):
    """All ordered pairs of the special set through fminf / fmaxf (operand order must not matter), and the contract stated
    explicitly: min(-0, +0) = -0, max(-0, +0) = +0 in either order, a NaN operand is ignored, saturate(-0) = saturate(NaN) = +0."""
    dev, orc = libs
    s = np.unique(np.concatenate([MINMAX_PARTNERS, _special_inputs()]))
    pairs = np.stack(np.meshgrid(s, s, indexing="ij"), axis=-1).reshape(-1, 2)
    lo = P.compare_cases(dev, orc, "fmin", pairs)[:, 0]
    hi = P.compare_cases(dev, orc, "fmax", pairs)[:, 0]
    swapped = pairs[:, ::-1]
    for name, got in (("fmin", lo), ("fmax", hi)):
        other = P.compare_cases(dev, orc, name, swapped)[:, 0]
        assert not np.any((got != other) & ~np.isnan(got.view(np.float32))), f"{name}f depends on the operand order"
    z = np.array([[0x80000000, 0x00000000], [0x00000000, 0x80000000]], dtype=np.uint32)
    assert list(P.compare_cases(dev, orc, "fmin", z)[:, 0]) == [0x80000000, 0x80000000]
    assert list(P.compare_cases(dev, orc, "fmax", z)[:, 0]) == [0x00000000, 0x00000000]
    nan1 = np.array([[0x7FC00000, 0x3F800000], [0x3F800000, 0x7FA12345]], dtype=np.uint32)
    assert list(P.compare_cases(dev, orc, "fmin", nan1)[:, 0]) == [0x3F800000, 0x3F800000]
    sat = P.compare_cases(dev, orc, "saturate", np.array([[0x80000000], [0x7FC00000], [0xFFC00000], [0xBF800000], [0x7F800000]], dtype=np.uint32))[:, 0]
    assert list(sat) == [0x00000000, 0x00000000, 0x00000000, 0x00000000, 0x3F800000]
    _report("fminf / fmaxf / saturate1 on special pairs, both operand orders", 2 * len(pairs))


def _srgb_code(v: np.ndarray) -> np.ndarray:
    """IEC 61966-2-1 in float64, rounded to 8 bits."""
    e = np.where(v <= 0.0031308, 12.92 * v, 1.055 * np.power(v, 1.0 / 2.4) - 0.055)
    return np.floor(np.clip(e, 0.0, 1.0) * 255.0 + 0.5)


def test_float_to_uint_and_display_encode_every_pattern(libs, scale):
    """__float2uint_rz against orc::f2uint_rz and DisplayEncode against the oracle's, on every pattern; the display code is within one
    of the float64 sRGB transfer function for every float in (0, 1] (the off-by-one count is reported)."""
    dev, orc = libs
    n = P.scan(dev, orc, "f2uint_rz", *_full(scale), stride=scale["stride"], chunk=scale["chunk"])
    _report("__float2uint_rz", n)
    worst, off_by_one = P.Worst(), []

    def analyse(xb, out):
        x = xb.view(np.float32)
        m = (x > 0) & (x <= 1)
        with np.errstate(all="ignore"):
            d = np.abs(out[:, 0].astype(np.float64) - _srgb_code(x.astype(np.float64)))
        d[~m] = 0.0
        off_by_one.append(int(np.count_nonzero(d == 1)))
        worst.add(d, xb, int(np.count_nonzero(m)))

    n = P.scan(dev, orc, "display_encode", *_full(scale), stride=scale["stride"], chunk=scale["chunk"], analyse=analyse,
               arrays_for=lambda a, b: a <= ONE_BITS or scale["stride"] > 1)
    _report("DisplayEncode", n, f"worst {worst.err:.0f} code(s) from float64 sRGB over {worst.n:,} inputs in (0, 1]; {sum(off_by_one)} off by one")
    assert worst.n > 0 and worst.err <= 1


def test_rng_every_state_and_known_answers(libs, scale):
    """NextRandom and RandomValue (__uint2float_rn(r) * 2^-32 against (float)r / 4294967296.0f) for every state, i.e. every
    NextRandom output (the step is a bijection); NextRandom against tests/golden/pcg_kat.json and a Python-integer restatement."""
    dev, orc = libs
    for name in ("next_random", "random_value"):
        n = P.scan(dev, orc, name, *_full(scale), stride=scale["stride"], chunk=scale["chunk"])
        _report(name, n)
    kat = json.load(open(os.path.join(GOLDEN, "pcg_kat.json")))
    for entry in kat:
        st = entry["seed"] & 0xFFFFFFFF
        for draw in entry["draws"]:
            r, v = dev.run("next_random", np.array([[st]], dtype=np.uint32))[0][0], dev.run("random_value", np.array([[st]], dtype=np.uint32))[0][0]
            assert (int(r[0]), int(r[1]), int(v[0])) == (draw["result"], draw["state"], draw["value_bits"])
            st = draw["state"]
    seeds = np.random.default_rng(7).integers(0, 1 << 32, min(10 ** 6, scale["states"]), dtype=np.uint64).astype(np.uint32)
    got = P.compare_cases(dev, orc, "next_random", seeds[:, None])
    s = (seeds.astype(np.uint64) * P.A + P.C_INC) & 0xFFFFFFFF
    res = (((s >> ((s >> 28) + 4)) ^ s) * 277803737) & 0xFFFFFFFF
    res = (res >> 22) ^ res
    assert np.array_equal(got[:, 0], res.astype(np.uint32)) and np.array_equal(got[:, 1], s.astype(np.uint32))
    assert all(P.pcg_python(int(x))[0] == int(y) for x, y in zip(seeds[:1000], got[:1000, 0]))
    _report("NextRandom known answers + Python-integer restatement", len(kat) + len(seeds))


def test_pow_on_the_paths_domain(libs, scale):
    """pow_rt(x, y) for every float x in [0, 1] with the exponents the path uses (0.35 sky gradient, 0.41666666 display encode,
    1000 / SunFocus for the default, the fixture and the five shipped scenes), and random (x, y) pairs."""
    dev, orc = libs
    for y in POW_EXPONENTS:
        n = P.scan(dev, orc, "pow", *_span(0, ONE_BITS, scale), stride=scale["stride"], partner=int(P.f32bits(y)), chunk=scale["chunk"])
        _report(f"pow_rt(x in [0, 1], {y})", n)
    rng = np.random.default_rng(11)
    done = 0
    while done < scale["pairs"]:
        m = min(scale["batch"] * 10, scale["pairs"] - done)
        x = rng.integers(0, ONE_BITS + 1, m, dtype=np.uint64).astype(np.uint32)
        y = P.f32bits(np.float32(10.0) ** rng.uniform(-3, 3, m).astype(np.float32))
        raw = rng.random(m) < 0.05                                  # and some arbitrary bit patterns as exponents
        y[raw] = rng.integers(0, 1 << 32, int(raw.sum()), dtype=np.uint64).astype(np.uint32)
        P.compare_cases(dev, orc, "pow", np.stack([x, y], axis=1))
        done += m
    _report("pow_rt on random (x in [0, 1], y in [1e-3, 1e3]) pairs", done)


def test_normal_draws_directions_and_points_in_circle(libs, scale):
    """RandomValueNormalDistribution, RandomDirection and RandomPointInCircle over 10^8 RNG states (outputs and the advanced state),
    and the states that force a draw to be exactly 0 (log(0) in Box-Muller) or exactly 1.0 at each of the draws they consume."""
    dev, orc = libs
    for name, draws in (("random_normal", 2), ("random_direction", 6), ("random_point_in_circle", 2)):
        n = P.scan(dev, orc, name, 0x2545F491, scale["states"], stride=0x9E3779B1, chunk=scale["chunk"] // 4)
        forced = P.forced_states(draws)
        out = P.compare_cases(dev, orc, name, forced[:, None])
        _report(f"{name} (+ {len(forced)} forced states)", n + len(forced))
        if name == "random_normal":
            assert np.any(~np.isfinite(out[:, 0].view(np.float32))), "a forced zero draw reaches log(0)"


# ---- section 3: intersection and shading primitives on adversarial classes -------------------------------------------------------------

def _batches(scale, seed):
    n, b = scale["cases"], scale["batch"]
    for k in range((n + b - 1) // b):
        yield np.random.default_rng(seed * 1000 + k), min(b, n - k * b)


def _f64(rec, a, b):
    return rec[:, a:b].view(np.float32).astype(np.float64)


def test_ray_box(libs, scale):
    """RayBoundingBoxDst (invDir = 1 / dir as the kernels form it) on generic rays, axis-aligned rays (invDir = +-inf), origins on a
    slab plane (0 * inf = NaN), inverted and flat boxes, coordinates up to 1e30, special values.  Float64 check on the generic class:
    each slab distance (b - p) * (1 / d) carries at most 3 roundings, |error| <= 3 * 2^-24 (|b| + |p|) / |d| (1 + 2^-23); hit / miss must
    agree with the float64 slab test unless tFar - tNear is inside twice that band, and dst within it."""
    dev, orc = libs
    worst, total = 0.0, 0
    for rng, m in _batches(scale, 1):
        rec, cls = P.box_cases(rng, m)
        got = P.compare_cases(dev, orc, "ray_box", rec)[:, 0].view(np.float32)
        total += m
        g = cls == 0
        pos, d, lo, hi = _f64(rec[g], 0, 3), _f64(rec[g], 3, 6), _f64(rec[g], 6, 9), _f64(rec[g], 9, 12)
        t1, t2 = (lo - pos) / d, (hi - pos) / d
        tn, tf = np.minimum(t1, t2).max(axis=1), np.maximum(t1, t2).min(axis=1)
        band = (3 * 2.0 ** -24 * (1 + 2.0 ** -23) * (np.abs(np.stack([lo, hi])).max(axis=0) + np.abs(pos)) / np.abs(d)).max(axis=1)
        hit64 = (tf >= tn) & (tf > 0)
        clear = (np.abs(tf - tn) > 2 * band) & (np.abs(tf) > band)
        hit = np.isfinite(got[g])
        assert np.all(hit[clear] == hit64[clear]), f"{np.count_nonzero(hit[clear] != hit64[clear])} box hit / miss decisions differ from float64"
        both = clear & hit & hit64
        err = np.abs(got[g][both] - np.maximum(tn[both], 0)) / band[both]
        worst = max(worst, float(err.max(initial=0)))
    _report("RayBoundingBoxDst", total, f"worst |dst - float64| = {worst:.3f} of the derived band")
    assert worst <= 1.0


def test_ray_triangle_through_the_upload_repack(libs, scale):
    """k_repack_tris then RayTriangleCore + TriangleSmoothNormal, as the kernels run them: hit flag, back-face flag, dst and normal
    bitwise.  Rays through edges and vertices (u, v or w exactly 0 where representable), |det| at 1e-8 and one ulp either side,
    axis-aligned rays, coordinates up to 1e30, special values.  Float64 check on the generic classes, aimed inside and aimed outside
    the triangle: with |det| far from 1e-8 and every float64 barycentric weight >= 1e-3 the ray must hit (dst > 0 by construction);
    with one weight <= -1e-3 it must miss; back faces under culling must miss.  Band: dst = dot(AO, N) / -dot(D, N), every term a
    short IEEE sum, relative error <= 2^-20 * cond, cond = (|AO| |N| / |dot(AO, N)|) + (|D| |N| / |dot(D, N)|); the weights carry the
    same kind of error, far below 1e-3 for cond < 1e4."""
    dev, orc = libs
    worst, total = 0.0, 0
    checked_miss = 0
    for rng, m in _batches(scale, 2):
        rec, cls = P.triangle_cases(rng, m)
        got = P.compare_cases(dev, orc, "ray_triangle", rec)
        total += m
        pos, d, A, B, Cc = (_f64(rec, 3 * k, 3 * k + 3) for k in range(5))
        N = np.cross(B - A, Cc - A)
        ao = pos - A
        dn = -(d * N).sum(axis=1)
        t = (ao * N).sum(axis=1) / np.where(dn == 0, 1, dn)
        cond = np.linalg.norm(ao, axis=1) * np.linalg.norm(N, axis=1) / np.maximum(np.abs((ao * N).sum(axis=1)), 1e-300) + \
            np.linalg.norm(d, axis=1) * np.linalg.norm(N, axis=1) / np.maximum(np.abs(dn), 1e-300)
        perp = np.cross(ao, d)
        u = (((Cc - A) * perp).sum(axis=1)) / np.where(dn == 0, 1, dn)
        v = -(((B - A) * perp).sum(axis=1)) / np.where(dn == 0, 1, dn)
        w = 1 - u - v
        cull = rec[:, 24] != 0
        gen = np.isin(cls, (0, 6)) & (cond < 1e4) & (np.abs(dn) > 1e-6) & (np.abs(t) > 1e-3)
        wmin = np.minimum(np.minimum(u, v), w)
        g = gen & (wmin > 1e-3) & np.where(cull, dn > 0, True) & (t > 0)
        miss = gen & ((wmin < -1e-3) | (cull & (dn < 0)) | (t < 0))
        flags = got[:, 0]
        assert np.all(flags[g] & 1), f"{np.count_nonzero((flags[g] & 1) == 0)} clear triangle hits missed"
        assert not np.any(flags[miss] & 1), f"{np.count_nonzero(flags[miss] & 1)} clear triangle misses hit"
        checked_miss += int(np.count_nonzero(miss))
        dst = got[g, 1].view(np.float32).astype(np.float64)
        err = np.abs(dst - t[g]) / (np.abs(t[g]) * 2.0 ** -20 * cond[g])
        worst = max(worst, float(err.max(initial=0)))
    _report("RayTriangleCore + TriangleSmoothNormal (through k_repack_tris)", total, f"worst |dst - float64| = {worst:.3f} of the derived band; "
            f"{checked_miss:,} clear misses agree with float64")
    assert worst <= 1.0 and checked_miss > 0


def test_ray_sphere_and_the_sphere_padding_bound(libs, scale):
    """RaySphereCore with r*r from rt_repack.cuh sphereR2, as buildSpheres forms it (the dstFar >= 0 <=> numFar >= 0 shortcut and
    div_cold included): hit, inside and dst bitwise on near-tangent and grazing rays, origins on the surface, r*r in {0, subnormal,
    inf}, zero and subnormal directions, far origins, special values.
    Against the product's padded boxes: for every hit the reference computes on the generic, near-tangent, on-surface and far classes,
    the box paddedSphereBox (rt_repack.cuh, the one buildSpheres uses) returns for an origin box holding the ray origin and the sphere
    must contain the hit point (float64 pos + dir * dst), or the accelerator could skip it.  The distance of the hit point from the
    exact sphere over the padding of that box (the smallest distance from the sphere's own box to the padded one) must stay below
    0.5, so that a tightening of the padding that eats the margin fails here.  Also reported: the same distance over 2.5e-7 (D^2 + r^2)
    / r, the estimate the padding was derived from."""
    dev, orc = libs
    worst_claim, worst_pad, total, counted = 0.0, 0.0, 0, 0
    for rng, m in _batches(scale, 3):
        rec, cls = P.sphere_cases(rng, m)
        got = P.compare_cases(dev, orc, "ray_sphere", rec)
        total += m
        g = np.isin(cls, (0, 1, 2, 5)) & ((got[:, 0] & 1) == 1)
        pos32, c32, r32 = rec[g, 0:3].view(np.float32), rec[g, 6:9].view(np.float32), rec[g, 9].view(np.float32)
        origin = np.concatenate([np.minimum(pos32, c32 - r32[:, None]), np.maximum(pos32, c32 + r32[:, None])], axis=1)
        inside, off_pad, off_claim = _sphere_hit_in_padded_box(dev, rec[g], got[g], origin)
        assert np.all(inside), f"{np.count_nonzero(~inside)} sphere hit points outside the padded box of their sphere"
        worst_pad = max(worst_pad, float(off_pad.max(initial=0)))
        worst_claim = max(worst_claim, float(off_claim.max(initial=0)))
        counted += int(np.count_nonzero(g))
    _report("RaySphereCore", total, f"{counted:,} hit points inside the product's padded sphere boxes; distance off the sphere: worst "
            f"{worst_pad:.3f} of the padding ({worst_claim:.3f} of the 2.5e-7 (D^2+r^2)/r estimate)")
    assert counted > 0 and worst_pad < 0.5


def _sphere_hit_in_padded_box(dev, rec, got, origin):
    """For ray_sphere hits (rec, got rows) and origin boxes (n, 6): whether the float64 hit point pos + dir * dst lies in the box
    paddedSphereBox gives the sphere, its distance off the exact sphere over the padding of that box, and over the 2.5e-7 (D^2 + r^2)
    / r estimate the padding was derived from."""
    c32, r32 = rec[:, 6:9].view(np.float32), rec[:, 9].view(np.float32)
    blo, bhi = dev.sphere_boxes(np.concatenate([c32, r32[:, None]], axis=1), origin)
    pos, d, c = _f64(rec, 0, 3), _f64(rec, 3, 6), _f64(rec, 6, 9)
    r = np.abs(r32.astype(np.float64))
    p = pos + d * got[:, 1].view(np.float32).astype(np.float64)[:, None]
    inside = np.all((p >= blo) & (p <= bhi), axis=1)
    off = np.abs(np.linalg.norm(p - c, axis=1) - r)
    pad = np.minimum((c - r[:, None]) - blo, bhi - (c + r[:, None])).min(axis=1)
    D2 = ((pos - c) ** 2).sum(axis=1)
    return inside, off / pad, off / (2.5e-7 * (D2 + r * r) / r)


SPHERE_GATE_CLASSES = ("aimed inside", "near-tangent", "from the surface", "from inside the origin box")


def test_sphere_padding_over_the_query_gates_domain(libs, scale):
    """The padding bound above over the domain in which the queries use the sphere accelerator: direction lengths log-uniform over
    the gate's 2^-10 .. 2^10 with both bounds, ray origins aimed from up to 8 units, near-tangent, on the surface (a bounce), and
    anywhere in an origin box reaching 1e5 units out.  RaySphereCore bitwise against the oracle; per class, every hit point inside
    the product's padded box and at most 0.5 of the padding off the sphere."""
    dev, orc = libs
    n_cls = len(SPHERE_GATE_CLASSES)
    worst, counted, total = np.zeros(n_cls), np.zeros(n_cls, int), 0
    for rng, m in _batches(scale, 10):
        rec, cls, origin = P.sphere_gate_cases(rng, m)
        got = P.compare_cases(dev, orc, "ray_sphere", rec)
        g = (got[:, 0] & 1) == 1
        inside, off_pad, _ = _sphere_hit_in_padded_box(dev, rec[g], got[g], origin[g])
        assert np.all(inside), f"{np.count_nonzero(~inside)} sphere hit points outside the padded box, classes {sorted(set(cls[g][~inside].tolist()))}"
        for c in range(n_cls):
            s = cls[g] == c
            worst[c] = max(worst[c], float(off_pad[s].max(initial=0)))
            counted[c] += int(np.count_nonzero(s))
        total += m
    _report("RaySphereCore over the query gate's domain", total,
            "; ".join(f"{name}: {counted[c]:,} hits, worst {worst[c]:.3f} of the padding" for c, name in enumerate(SPHERE_GATE_CLASSES)))
    assert counted.min() > 0 and worst.max() < 0.5, f"worst margins {dict(zip(SPHERE_GATE_CLASSES, worst.round(3)))}"


# Found by sphere_gate_cases with |dir| = 1e-21 (below the gate): a sphere of radius 0.19, 11.9 units from the ray origin.
# dot(dir, dir) ~ 1e-42 is subnormal, the discriminant is mostly rounding, and the reference reports a hit at dst = 1.16e22, 0.20
# units off the sphere (128 times the padding) and outside the box paddedSphereBox gives it: the accelerator would prune a hit the
# reference draws.
BELOW_GATE_SPHERE_CASE = [0xc0c6fcb7, 0xc08321d5, 0xc11e5cff, 0x1c54e618, 0x1bc1efc9, 0x1c3f59c8, 0x400daa36, 0xbe813338, 0xc016e4f8, 0x3e4486f3]
BELOW_GATE_SPHERE_ORIGIN_BOX = [-6.218348979949951, -4.097879886627197, -9.897704124450684, 8.591245651245117, 2.244865655899048, -2.165803909301758]


def test_sphere_hit_below_the_gate_lies_outside_its_padded_box(libs):
    """Why the queries use the sphere accelerator only for 2^-20 <= dot(dir, dir) <= 2^20: below that the padding bound does not hold.
    The pinned case: the device and the oracle agree bit for bit on a hit whose point lies outside the sphere's padded box."""
    dev, orc = libs
    rec = np.array([BELOW_GATE_SPHERE_CASE], dtype=np.uint32)
    got = P.compare_cases(dev, orc, "ray_sphere", rec)
    d = rec[0, 3:6].view(np.float32)
    assert np.float32(np.float32(d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]) < np.float32(2.0 ** -20), "the case lies inside the gate"
    assert got[0, 0] & 1, "the reference's arithmetic no longer reports the hit"
    inside, off_pad, _ = _sphere_hit_in_padded_box(dev, rec, got, np.array([BELOW_GATE_SPHERE_ORIGIN_BOX], dtype=np.float32))
    assert not inside[0], f"the hit point lies inside the padded box ({off_pad[0]:.3g} of the padding off the sphere)"
    _report("RaySphereCore below the gate (|dir| = 1e-21)", 1, f"hit {off_pad[0]:.3g} x the padding off the sphere, outside its padded box")


def test_model_skipping_keeps_every_hit_the_reference_finds(libs, scale):
    """The padding of the models' world boxes (rt_repack.cuh paddedModelBox, as buildModels applies it to the image of the mesh's
    geometry box under the inverse of worldToLocal) against the reference's own arithmetic: single-triangle models 1e-3 .. 100 in size,
    rotated, non-uniformly scaled and mirrored, up to 1e5 from the origin, rays from up to 1e5 away aimed at the interior, the edges and
    vertices, and just outside.  For every hit the reference finds (the ray transformed with mul_rm, RayTriangleCore on the repacked
    triangle, and the slab test of the geometry box passed), WorldBoxOutOfReach on the product's padded world box must not skip the
    model at bestDst = nextafter(dst, +inf).  The distance of the world hit point (float64 pos + dir * dst) outside the exact world
    box, over that axis's padding, must stay below 0.5, so that a tightening that eats the margin fails here.  Device only: the
    reference has no model skipping to compare with.  Hits outside the geometry box, which the reference's slab test discards for an
    inner root, are counted and must not be skipped either.
    Grazing rays are the exception, and a known defect: when the ray meets the triangle's plane at |cos| < GRAZING_COS, the float32
    transform of a distant origin into model space moves the reference's hit along the ray by far more than the padding (its
    Moeller-Trumbore can even report a hit the exact ray misses), so WorldBoxOutOfReach can skip a hit the reference finds.  Those
    hits are counted and reported here, and test_model_skipping_loses_a_grazing_hit pins one such case."""
    dev, _ = libs
    worst, counted, outside_box, total, grazing, grazing_skipped = 0.0, 0, 0, 0, 0, 0
    for rng, m in _batches(scale, 7):
        case = P.model_cases(rng, m)
        r = _model_hit(dev, *case)
        assert r["placed"].all()
        grazing += int(np.count_nonzero(r["hit"] & r["graze"]))
        grazing_skipped += int(np.count_nonzero(r["hit"] & r["graze"] & r["skipped"]))
        hit = r["hit"] & ~r["graze"]
        assert not np.any(hit & r["skipped"]), f"{np.count_nonzero(hit & r['skipped'])} model hits skipped by WorldBoxOutOfReach"
        outside_box += int(np.count_nonzero(hit & ~r["in_box"]))
        worst = max(worst, float(r["margin"].max(initial=0)))
        counted += int(np.count_nonzero(hit & r["in_box"]))
        total += m
    _report("model skipping (mul_rm + RayTriangleCore + WorldBoxOutOfReach)", total,
            f"{counted:,} hits the reference finds, none skipped; worst distance outside the exact world box {worst:.3f} of the padding; "
            f"{outside_box:,} hits outside the geometry box, none skipped; {grazing:,} grazing hits (|cos| < {GRAZING_COS}), "
            f"{grazing_skipped} of them skipped (known defect)", vs_oracle=False)
    assert counted > 0 and worst < 0.5


def _model_hit(dev, w2l, tri, geo, pos, d, origin, cull):
    """model_hit on the product's padded world boxes of a batch of model_cases: per case `placed` (worldBoxOfModel accepted the
    matrix; otherwise the box is infinite), `hit` (the reference finds it), `skipped` (WorldBoxOutOfReach skips the model), `graze`
    (|cos| < GRAZING_COS), `in_box` (the local ray reaches the geometry box) and `margin`: for a non-grazing hit inside the geometry
    box of a placed model, the largest distance of the world hit point outside the exact world box over that axis's padding (else 0)."""
    m = len(pos)
    exact, padded, _ = dev.model_boxes(w2l, geo, origin)
    rows = w2l.reshape(m, 4, 4).transpose(0, 2, 1)[:, :3, :].reshape(m, 12)
    rec = np.concatenate([P.f32bits(pos), P.f32bits(d), P.f32bits(tri), np.zeros((m, 9), np.uint32), P.f32bits(rows), P.f32bits(geo),
                          padded.view(np.uint32), cull[:, None]], axis=1)
    out, _ = dev.run("model_hit", rec)
    f = out[:, 0]
    A = rows.reshape(m, 3, 4)[:, :, :3].astype(np.float64)
    ld = np.einsum("nij,nj->ni", A, d.astype(np.float64))
    t3 = tri.reshape(m, 3, 3).astype(np.float64)
    N = np.cross(t3[:, 1] - t3[:, 0], t3[:, 2] - t3[:, 0])
    with np.errstate(all="ignore"):
        cos = np.abs((ld * N).sum(axis=1)) / (np.linalg.norm(ld, axis=1) * np.linalg.norm(N, axis=1))
    r = dict(placed=np.isfinite(padded).all(axis=1), hit=(f & 1) == 1, skipped=(f & 4) == 4, graze=cos < GRAZING_COS, in_box=(f & 2) == 2)
    g = r["hit"] & ~r["graze"] & r["in_box"] & r["placed"]
    p = pos[g].astype(np.float64) + d[g].astype(np.float64) * out[g, 1].view(np.float32).astype(np.float64)[:, None]
    lo, hi = exact[g, :3], exact[g, 3:]
    need = np.maximum(np.maximum(lo - p, p - hi), 0.0)
    pad = np.minimum(lo - padded[g, :3], padded[g, 3:] - hi)
    r["margin"] = np.zeros(m)
    r["margin"][g] = (need / pad).max(axis=1, initial=0)
    return r


MODEL_GATE_CLASSES = ("R S R, from afar", "sheared, from afar", "R S R, from inside the origin box", "sheared, from inside the origin box",
                      "R S R, from the triangle", "sheared, from the triangle")


def test_model_skipping_over_the_query_gates_domain(libs, scale):
    """The check above over the whole domain in which the queries (rtTraceRays, rtTraceOcclusion, every bounce of rtTracePaths) use
    model skipping and the TLAS: worldToLocal with singular values 1e-3 .. 1e3, rotation x scale x rotation and sheared products of
    two of them (a rotated child of a non-uniformly scaled parent); direction lengths log-uniform over the gate's 2^-10 .. 2^10 with
    both bounds; ray origins from afar, anywhere in the origin box, and on the triangle itself (a bounce).  Per class: no non-grazing
    hit skipped, worst distance outside the exact world box below 0.5 of the padding.  Matrices worldBoxOfModel refuses get an
    infinite box (never skipped) and are counted.  Also reported, not asserted: skipped hits with |dir| below the gate (1e-23 ..
    2^-10), where the queries take the linear loop."""
    dev, _ = libs
    n_cls = len(MODEL_GATE_CLASSES)
    worst, counted, refused, grazing, total = np.zeros(n_cls), np.zeros(n_cls, int), 0, 0, 0
    for rng, m in _batches(scale, 8):
        *case, cls = P.model_gate_cases(rng, m)
        r = _model_hit(dev, *case)
        hit = r["hit"] & ~r["graze"]
        bad = hit & r["skipped"]
        assert not bad.any(), f"{np.count_nonzero(bad)} model hits skipped by WorldBoxOutOfReach, classes {sorted(set(cls[bad].tolist()))}"
        for c in range(n_cls):
            s = cls == c
            worst[c] = max(worst[c], float(r["margin"][s].max(initial=0)))
            counted[c] += int(np.count_nonzero(hit[s] & r["placed"][s]))
        refused += int(np.count_nonzero(~r["placed"]))
        grazing += int(np.count_nonzero(r["hit"] & r["graze"]))
        total += m
    below, below_hits, below_skipped = 0, 0, 0
    for rng, m in _batches(dict(scale, cases=scale["cases"] // 10), 9):
        *case, _ = P.model_gate_cases(rng, m, lengths=np.exp(rng.uniform(np.log(1e-23), np.log(P.GATE_LEN_MIN), m)))
        r = _model_hit(dev, *case)
        hit = r["hit"] & ~r["graze"]
        below_hits += int(np.count_nonzero(hit))
        below_skipped += int(np.count_nonzero(hit & r["skipped"]))
        below += m
    _report("model skipping over the query gate's domain", total,
            "; ".join(f"{name}: {counted[c]:,} hits, worst {worst[c]:.3f} of the padding" for c, name in enumerate(MODEL_GATE_CLASSES)) +
            f"; {refused:,} matrices refused by worldBoxOfModel (infinite box); {grazing:,} grazing hits left out.  Below the gate "
            f"(|dir| 1e-23 .. 2^-10): {below:,} cases, {below_hits:,} hits, {below_skipped} skipped", vs_oracle=False)
    assert counted.min() > 0 and worst.max() < 0.5, f"worst margins {dict(zip(MODEL_GATE_CLASSES, worst.round(3)))}"


def test_tlas_marks_every_model_its_own_box_keeps(libs, scale):
    """TlasCollect (rt_device.cuh) on the tree the host's planTlas builds: a model is left out of the mask only if WorldBoxOutOfReach
    rejects a TLAS box that encloses its box, and that must imply the same test rejects the model's own box, at the same bestDst.
    Trees of 1 .. 4,096 boxes (generic, grid cells sharing faces, flat, bounds at +-0, NaN bounds, the infinite box of a singular
    model); rays generic, axis-aligned (invDir = +-inf), on a slab plane or one ulp inside it and parallel to it (0 x inf = NaN), from
    box corners, direction lengths over the query gate's range; bestDst +inf, a box corner's distance, +-0, tiny, huge, NaN.  Every
    model whose own box test keeps it must be marked.  Device only: the reference has no TLAS."""
    dev, _ = libs
    trees = 40
    per_tree = max(scale["cases"] // trees, 1)
    rng = np.random.default_rng(12)
    kept, rays, models = 0, 0, 0
    for t in range(trees):
        n = P.TLAS_SIZES[t] if t < len(P.TLAS_SIZES) else int(np.exp(rng.uniform(0, np.log(4096))))
        boxes = P.tlas_boxes(rng, n)
        for done in range(0, per_tree, scale["batch"]):
            r = P.tlas_rays(rng, boxes, min(scale["batch"], per_tree - done))
            out = dev.tlas_check(boxes, r)
            bad = np.flatnonzero(out[:, 1])
            assert len(bad) == 0, (f"{len(bad)} rays:TlasCollect leaves out a model its own box keeps; first: {n} models, "
                                   f"ray {r[bad[0]].tolist()}, model {out[bad[0], 2]} box {boxes[out[bad[0], 2]].tolist()}")
            kept += int(out[:, 0].sum())
            rays += len(r)
        models += n
    _report("TlasCollect on planTlas trees", rays, f"{trees} trees, {models:,} model boxes; {kept:,} (ray, model) pairs kept by the "
            "model's own box, every one marked", vs_oracle=False)
    assert kept > 0


GRAZING_COS = 1e-2
# Found by the test above on the H100 and reproduced on the SIMT build: a 0.25-unit triangle 1.8 units from the world origin, the ray
# from (16827.8, -2967.3, -4582.9), 17,693 units away, meeting the triangle's plane at |cos| = 5e-4.  The exact ray misses the triangle
# (v = -1.75); the reference's float32 arithmetic reports a hit at dst = 17692.277, 0.76 short of where the ray crosses the plane, and
# the world box, padded by 0.34, is entered beyond that: the product skips the model and loses a hit the reference draws.
GRAZING_CASE = [0x4683779a, 0xc5397538, 0xc58f3740, 0xbf738174, 0x3e2bcf03, 0x3e849b2d, 0x3e76c811, 0xbda3a141, 0x3cb1cb17, 0xbb8e29d5,
                0xbd37b73f, 0x3e00dcf0, 0x3e408065, 0xbdf70fa6, 0x3bd9401d] + [0] * 9 + \
               [0xbfaffb82, 0xbe76f02b, 0xbf585e06, 0xc0114b1a, 0xbf1d1c50, 0xbe7d2c43, 0x3f94402e, 0xbe3b0621, 0xbda96475, 0x3f22f3fb,
                0x3f09c7d2, 0xbf11620d, 0xbb8e29d5, 0xbdf70fa6, 0x3bd9401d, 0x3e76c811, 0xbd37b73f, 0x3e00dcf0, 0xc0049797, 0x3f42c292,
                0xbf6b5607, 0xbf98e3c6, 0x3fd77fbc, 0xbdefdfaa, 0x00000000]


@pytest.mark.xfail(strict=True, reason="known defect: model skipping can lose a hit of a far grazing ray (DESIGN.md section 5)")
def test_model_skipping_loses_a_grazing_hit(libs):
    """Regression case of the defect described at test_model_skipping_keeps_every_hit_the_reference_finds: the reference finds the hit
    (flags 1 and 2), and WorldBoxOutOfReach on the product's padded box must not skip it (flag 4).  Expected to fail until the skip
    test accounts for the error of a grazing hit; strict, so that a fix shows up here."""
    dev, _ = libs
    out, _ = dev.run("model_hit", np.array([GRAZING_CASE], dtype=np.uint32))
    assert out[0, 0] & 3 == 3, "the reference's arithmetic no longer finds the grazing hit"
    assert not out[0, 0] & 4, "WorldBoxOutOfReach skips a hit the reference finds"


def test_reflectance_refract_reflect(libs, scale):
    """CalculateReflectance, Refract and Reflect on glass-like inputs, total internal reflection at sinSqr == 1 exactly and next to it,
    ior in {0, 1, negative, -0} and special values.  Float64: for physical inputs (unit vectors, iors in [1, 2.5]) the reflectance lies
    in [0, 1] and matches the float64 evaluation of the reference's own expression (the duplicated denominator included).  Band:
    about 30 roundings each <= 2^-24 relative, amplified by 1 / denominator and by squaring terms <= 1, give 2^-16; near total internal
    reflection cosAngleOfRefraction = sqrt(1 - sinSqr) magnifies the <= 4 ulp error of sinSqr (<= rr^2 2^-22) by 1 / (2 cos), and the
    quotients carry it with weight (iorA + iorB) / den: band = 2^-16 + 2^-23 rr^2 (iorA + iorB) / (cos den)."""
    dev, orc = libs
    worst, total = 0.0, 0
    for rng, m in _batches(scale, 4):
        rec, cls = P.shading_cases(rng, m)
        refl = P.compare_cases(dev, orc, "reflectance", rec)[:, 0].view(np.float32)
        P.compare_cases(dev, orc, "refract", rec)
        P.compare_cases(dev, orc, "reflect", rec[:, :6])
        total += m
        g = cls == 0
        d, nrm, a, b = _f64(rec[g], 0, 3), _f64(rec[g], 3, 6), _f64(rec[g], 6, 7)[:, 0], _f64(rec[g], 7, 8)[:, 0]
        rr = a / b
        ci = -(d * nrm).sum(axis=1)
        s2 = rr * rr * (1 - ci * ci)
        ct = np.sqrt(np.maximum(1 - s2, 0))
        den = a * ci + b * ct
        ref = np.where((s2 >= 1) | (den < 1e-8), 1.0, 0.5 * (((a * ci - b * ct) / den) ** 2 + ((b * ci - a * ct) / den) ** 2))
        r = refl[g].astype(np.float64)
        assert np.all((r >= 0) & (r <= 1)), "reflectance outside [0, 1] for a physical input"
        clear = (s2 < 1 - 1e-6) & (den > 1e-6)
        band = 2.0 ** -16 + 2.0 ** -23 * rr * rr * (a + b) / (np.maximum(ct, 1e-300) * np.maximum(den, 1e-300))
        worst = max(worst, float((np.abs(r - ref) / band)[clear].max(initial=0)))
    _report("CalculateReflectance / Refract / Reflect", total, f"worst |reflectance - float64| = {worst:.3f} of the derived band")
    assert worst <= 1.0


def test_material_colour_on_checker_cell_boundaries(libs, scale):
    """GetMaterialColour on checkered and plain materials at positions on, and one ulp either side of, the cell boundaries (multiples
    of 1 / 1.5), with normals whose components tie (the projection-plane choice)."""
    dev, orc = libs
    total = 0
    for rng, m in _batches(scale, 5):
        rec, _ = P.checker_cases(rng, m)
        P.compare_cases(dev, orc, "material_colour", rec)
        total += m
    _report("GetMaterialColour", total)


def test_environment_light_around_the_horizon(libs, scale):
    """GetEnvironmentLight with dir.y at and around +-0 and the -0.01 edge of the ground blend, the sun direction itself, the SunFocus
    values of the path and special values."""
    dev, orc = libs
    total = 0
    for rng, m in _batches(scale, 6):
        rec, _ = P.sky_cases(rng, m, sorted(set(SUN_FOCUS.values())))
        P.compare_cases(dev, orc, "environment_light", rec)
        total += m
    _report("GetEnvironmentLight", total)
