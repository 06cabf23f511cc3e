"""TEST INFRASTRUCTURE ONLY.  ctypes side of the primitive probe (rt_probe.cu) and of the oracle's orProbe: function codes, record
shapes, exhaustive scans compared by digest, batched case comparison, and the seeded generator of adversarial primitive inputs."""
from __future__ import annotations

import ctypes as C
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np

# name: (code, words in, words out, mask of the output words that are floats); the codes are rt_probe.cu's ProbeFn
FN = {
    "log": (0, 1, 1, 0b1), "exp": (1, 1, 1, 0b1), "sin": (2, 1, 1, 0b1), "cos": (3, 1, 1, 0b1), "sincos": (4, 1, 2, 0b11),
    "pow": (5, 2, 1, 0b1), "saturate": (6, 1, 1, 0b1), "fmin": (7, 2, 1, 0b1), "fmax": (8, 2, 1, 0b1), "f2uint_rz": (9, 1, 1, 0b0),
    "display_encode": (10, 1, 1, 0b0), "next_random": (11, 1, 2, 0b00), "random_value": (12, 1, 2, 0b01),
    "random_normal": (13, 1, 2, 0b01), "random_direction": (14, 1, 4, 0b0111), "random_point_in_circle": (15, 1, 3, 0b011),
    "ray_box": (20, 12, 1, 0b1), "ray_triangle": (21, 25, 5, 0b11110), "ray_sphere": (22, 10, 2, 0b10),
    "reflectance": (23, 8, 1, 0b1), "refract": (24, 8, 3, 0b111), "reflect": (25, 6, 3, 0b111),
    "material_colour": (26, 17, 3, 0b111), "environment_light": (27, 11, 3, 0b111),
    "model_hit": (28, 49, 2, 0b10),                                 # device only
}

THREADS = os.cpu_count() or 4


class Lib:
    """One side of the comparison: the device probe (rtpRun) or the oracle (orProbe)."""

    def __init__(self, path: str, oracle: bool):
        self.lib = C.CDLL(path)
        self.oracle = oracle
        args = [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32, C.c_size_t, C.c_void_p]
        self.fn = self.lib.orProbe if oracle else self.lib.rtpRun
        self.fn.argtypes = args + ([C.c_int] if oracle else [])
        self.fn.restype = C.c_int

    def sphere_boxes(self, centre_radius, origin_box):
        """The sphere accelerator's padded boxes (rt_repack.cuh paddedSphereBox) for (n, 4) centre + radius, (n, 6) origin boxes."""
        cr, ob = np.ascontiguousarray(centre_radius, dtype=np.float32), np.ascontiguousarray(origin_box, dtype=np.float32)
        lo, hi = np.empty((len(cr), 3), dtype=np.float32), np.empty((len(cr), 3), dtype=np.float32)
        self.lib.rtpSphereBoxes(C.c_void_p(cr.ctypes.data), C.c_void_p(ob.ctypes.data), C.c_void_p(lo.ctypes.data), C.c_void_p(hi.ctypes.data), C.c_size_t(len(cr)))
        return lo, hi

    def model_boxes(self, w2l_colmajor, geo, origin_box):
        """(exact world box (n, 6) float64, padded world box (n, 6) float32) of models as buildModels computes them."""
        w, g, ob = (np.ascontiguousarray(a, dtype=np.float32) for a in (w2l_colmajor, geo, origin_box))
        exact, padded = np.empty((len(w), 6)), np.empty((len(w), 6), dtype=np.float32)
        self.lib.rtpModelBoxes.restype = C.c_int
        placed = self.lib.rtpModelBoxes(C.c_void_p(w.ctypes.data), C.c_void_p(g.ctypes.data), C.c_void_p(ob.ctypes.data), C.c_void_p(exact.ctypes.data),
                                        C.c_void_p(padded.ctypes.data), C.c_size_t(len(w)))
        return exact, padded, placed

    def tlas_check(self, boxes, rays):
        """TlasCollect over the TLAS planTlas builds for the (n, 6) model boxes, for (m, 7) rays (pos, dir, bestDst): (m, 3) int32 rows
        (models WorldBoxOutOfReach keeps on their own box, how many of those the TLAS mask lacks, the first of them or -1)."""
        b, r = np.ascontiguousarray(boxes, dtype=np.float32), np.ascontiguousarray(rays, dtype=np.float32)
        out = np.empty((len(r), 3), dtype=np.int32)
        self.lib.rtpTlasCheck.restype = C.c_int
        rc = self.lib.rtpTlasCheck(C.c_void_p(b.ctypes.data), C.c_int(len(b)), C.c_void_p(r.ctypes.data), C.c_size_t(len(r)), C.c_void_p(out.ctypes.data))
        assert rc == 0, f"rtpTlasCheck returned {rc}"
        return out

    def run(self, name, cases=None, n=None, base=0, stride=1, partner=0, arrays=True):
        """cases: (n, nin) uint32, or None for index mode over n cases.  Returns (outputs (n, nout) uint32 or None, digest (nout,))."""
        code, nin, nout, fmask = FN[name]
        if cases is not None:
            cases = np.ascontiguousarray(cases, dtype=np.uint32).reshape(-1, nin)
            n = len(cases)
        out = np.empty((n, nout), dtype=np.uint32) if arrays else None
        dig = np.zeros(nout, dtype=np.uint64)
        extra = (0,) if self.oracle else ()
        rc = self.fn(code, nin, nout, None if cases is None else cases.ctypes.data, base & 0xffffffff, stride & 0xffffffff, partner & 0xffffffff,
                     None if out is None else out.ctypes.data, fmask, n, dig.ctypes.data, *extra)
        assert rc == 0, f"{'orProbe' if self.oracle else 'rtpRun'}({name}) returned {rc}"
        return out, dig


def first_difference(name, dev, orc, inputs):
    """Report of the NaN-aware bitwise comparison of two (n, nout) output arrays (None when equal)."""
    fmask = FN[name][3]
    bad = dev != orc
    for j in range(dev.shape[1]):
        if (fmask >> j) & 1:
            bad[:, j] &= ~(np.isnan(dev[:, j].view(np.float32)) & np.isnan(orc[:, j].view(np.float32)))
    rows = np.flatnonzero(bad.any(axis=1))
    if len(rows) == 0:
        return None
    i = rows[0]
    return (f"{name}: {len(rows)} of {len(dev)} cases differ; first: input words {[hex(int(w)) for w in inputs[i]]} -> device "
            f"{[hex(int(w)) for w in dev[i]]}, oracle {[hex(int(w)) for w in orc[i]]}")


def compare_cases(dev: Lib, orc: Lib, name, cases):
    """Evaluates the cases on both sides; asserts bit equality (NaN = NaN); returns the device outputs."""
    d, _ = dev.run(name, cases)
    o, _ = orc.run(name, cases)
    msg = first_difference(name, d, o, np.asarray(cases, dtype=np.uint32).reshape(len(d), -1))
    assert msg is None, msg
    return d


def scan(dev: Lib, orc: Lib, name, start, count, stride=1, partner=0, chunk=1 << 26, analyse=None, arrays_for=None):
    """Index-mode scan of `count` inputs start, start + stride, ... (mod 2^32), compared chunk by chunk by digest; a chunk whose digests
    differ is evaluated again with arrays and reported.  analyse(x_bits, dev_out) runs in a thread pool on the device outputs of every
    chunk for which arrays_for(first, last) is true (default: all).  Returns the number of inputs compared."""
    pool = ThreadPoolExecutor(THREADS) if analyse else None
    futures = []
    done = 0
    while done < count:
        m = min(chunk, count - done)
        base = (start + done * stride) & 0xffffffff
        want = analyse is not None and (arrays_for is None or arrays_for(base, (base + (m - 1) * stride) & 0xffffffff))
        d, dd = dev.run(name, n=m, base=base, stride=stride, partner=partner, arrays=want)
        _, od = orc.run(name, n=m, base=base, stride=stride, partner=partner, arrays=False)
        if not np.array_equal(dd, od):
            d, _ = dev.run(name, n=m, base=base, stride=stride, partner=partner)
            o, _ = orc.run(name, n=m, base=base, stride=stride, partner=partner)
            x = (base + np.arange(m, dtype=np.uint64) * stride).astype(np.uint32)
            cols = [x] + [np.full(m, partner, dtype=np.uint32)] * (FN[name][1] - 1)
            msg = first_difference(name, d, o, np.stack(cols, axis=1))
            raise AssertionError(msg or f"{name}: digests differ at chunk base {base:#x} but no output word does")
        if want:
            x = (base + np.arange(m, dtype=np.uint64) * stride).astype(np.uint32)
            futures.append(pool.submit(analyse, x, d))
            if len(futures) >= THREADS:
                futures.pop(0).result()            # bounds the chunks held in memory
        done += m
    for f in futures:
        f.result()
    if pool:
        pool.shutdown()
    return done


def ulp32(ref: np.ndarray) -> np.ndarray:
    """Spacing of binary32 numbers at the (float64) value ref: 2^(e-24) for |ref| in [2^(e-1), 2^e), 2^-149 below 2^-126."""
    _, e = np.frexp(np.abs(ref))
    return np.ldexp(1.0, np.maximum(e - 24, -149))


class Worst:
    """Running maximum of an error measure and the input where it occurred (shared by the analysis threads of a scan)."""

    def __init__(self):
        self.err, self.at, self.n = 0.0, None, 0
        import threading
        self.lock = threading.Lock()

    def add(self, err: np.ndarray, x: np.ndarray, n=None):
        """err: errors of the inputs x (0 where not measured); n: how many were measured (default all)."""
        with self.lock:
            self.n += err.size if n is None else n
            if err.size:
                err = np.where(np.isnan(err), np.inf, err)          # a NaN error is the worst error, never a silent one
                i = int(np.argmax(err))
                if err[i] > self.err:
                    self.err, self.at = float(err[i]), x[i]


def f32bits(v) -> np.ndarray:
    return np.asarray(v, dtype=np.float32).view(np.uint32)


# ---- PCG (RayCommon.hlsl:127-133) as Python integers, and states that force a draw ----------------------------------------------------

A, C_INC, M32 = 747796405, 2891336453, 1 << 32
A_INV = pow(A, -1, M32)


def pcg_python(state: int):
    state = (state * A + C_INC) % M32
    result = (((state >> ((state >> 28) + 4)) ^ state) * 277803737) % M32
    return (result >> 22) ^ result, state


def state_before(post_step_state: int, draws: int) -> int:
    """The state whose `draws`-th NextRandom leaves the generator in post_step_state (the inverse LCG, as conftest.seed_forcing_draw)."""
    st = post_step_state
    for _ in range(draws):
        st = ((st - C_INC) * A_INV) % M32
    return st


# post-step states whose draw is exactly 0 (output 0) and exactly 1.0 (output >= 2^32 - 128, rounds to 2^32); test_oracle.py uses them too
FORCED_POST_STATES = (0, 515875080)


def forced_states(max_draw: int) -> np.ndarray:
    return np.array([state_before(p, k) for p in FORCED_POST_STATES for k in range(1, max_draw + 1)], dtype=np.uint32)


# ---- adversarial primitive inputs ------------------------------------------------------------------------------------------------------

SPECIAL = np.array([0.0, -0.0, 1.0, -1.0, np.inf, -np.inf, np.nan, 1e-45, -1e-45, 1.1754942e-38, -1.1754942e-38, 1.17549435e-38,
                    3.4028235e38, -3.4028235e38, 1e30, -1e30, 0.5, 1e-8, 2.0, 1e5], dtype=np.float32)


def _vec(rng, n, scale=1.0):
    return (rng.standard_normal((n, 3)) * scale).astype(np.float32)


def _unit(rng, n):
    v = rng.standard_normal((n, 3))
    return (v / np.linalg.norm(v, axis=1, keepdims=True)).astype(np.float32)


def _sprinkle(rng, a: np.ndarray, frac: float):
    """Replaces a fraction of the float components with special values (NaN, +-inf, +-0, subnormals, huge)."""
    f = a.view(np.float32)
    mask = rng.random(f.shape) < frac
    f[mask] = rng.choice(SPECIAL, size=int(mask.sum()))
    return a


def _axis_aligned(rng, d: np.ndarray):
    """Zeroes one or two components of each direction, with either sign of zero (invDir = +-inf)."""
    n = len(d)
    k = rng.integers(0, 3, n)
    d[np.arange(n), k] = np.where(rng.random(n) < 0.5, np.float32(0.0), np.float32(-0.0))
    two = rng.random(n) < 0.3
    k2 = (k + 1) % 3
    d[np.flatnonzero(two), k2[two]] = np.float32(-0.0)
    return d


def box_cases(rng, n):
    """pos, dir, boxMin, boxMax.  Classes: generic; axis-aligned directions; origin on a slab plane (0 * inf); min > max and zero
    extent; huge coordinates; special values anywhere."""
    lo = _vec(rng, n, 4.0)
    hi = lo + np.abs(_vec(rng, n, 2.0))
    pos = _vec(rng, n, 8.0)
    d = _unit(rng, n)
    cls = rng.integers(0, 6, n)
    s = cls == 1
    d[s] = _axis_aligned(rng, d[s])
    s = cls == 2                                                   # origin exactly on a slab plane, direction parallel to it
    ax = rng.integers(0, 3, n)
    idx = np.flatnonzero(s)
    pos[idx, ax[idx]] = np.where(rng.random(len(idx)) < 0.5, lo[idx, ax[idx]], hi[idx, ax[idx]])
    d[idx, ax[idx]] = np.where(rng.random(len(idx)) < 0.5, np.float32(0.0), np.float32(-0.0))
    s = cls == 3                                                   # inverted or flat boxes
    idx = np.flatnonzero(s)
    flat = rng.random(len(idx)) < 0.5
    hi[idx[flat], ax[idx[flat]]] = lo[idx[flat], ax[idx[flat]]]
    lo[idx[~flat]], hi[idx[~flat]] = hi[idx[~flat]].copy(), lo[idx[~flat]].copy()
    s = cls == 4                                                   # far away: coordinates up to 1e30, distances up to 1e5
    big = np.float32(10.0) ** rng.uniform(3, 30, (int(s.sum()), 1)).astype(np.float32)
    lo[s] *= big; hi[s] *= big; pos[s] *= np.float32(10.0) ** rng.uniform(0, 5, (int(s.sum()), 1)).astype(np.float32)
    rec = np.concatenate([pos, d, lo, hi], axis=1)
    s = cls == 5
    rec[s] = _sprinkle(rng, rec[s], 0.15)
    return rec.view(np.uint32), cls


def triangle_cases(rng, n):
    """pos, dir, A, B, C, nA, nB, nC, cull.  Rays aimed at a chosen barycentric point; classes: 0 generic; 1 through an edge or a vertex
    (a weight 0 in float64; the float32 rounding of the ray leaves u, v or w within a few ulp of 0); 2 |determinant| near the 1e-8
    culling threshold (the edges scaled in float64 so that |det| is 1e-8 or its float32 neighbours, then rounded to float32, which
    moves it by a few ulp); 3 axis-aligned directions; 4 huge coordinates; 5 special values anywhere; 6 generic, aimed outside."""
    A = _vec(rng, n, 2.0)
    B = A + _vec(rng, n, 1.0)
    Cc = A + _vec(rng, n, 1.0)
    bary = rng.dirichlet((1.0, 1.0, 1.0), n)
    cls = rng.integers(0, 7, n)
    s = np.flatnonzero(cls == 6)                                   # aimed outside: one weight negative
    bary[s, rng.integers(0, 3, len(s))] = -rng.uniform(0.002, 0.5, len(s))
    bary[s] /= bary[s].sum(axis=1, keepdims=True)
    s = np.flatnonzero(cls == 1)                                   # on an edge (one weight 0) or a vertex (two weights 0)
    k = rng.integers(0, 3, len(s))
    bary[s, k] = 0.0
    vert = rng.random(len(s)) < 0.3
    bary[s[vert], (k[vert] + 1) % 3] = 0.0
    bary[s] /= bary[s].sum(axis=1, keepdims=True)
    target = (bary[:, :1] * A + bary[:, 1:2] * B + bary[:, 2:] * Cc).astype(np.float32)
    d = _unit(rng, n)
    pos = (target - d * np.float32(5.0)).astype(np.float32)
    s = np.flatnonzero(cls == 2)                                   # |det| = 1e-8 and its neighbours: scale the face vector
    N = np.cross(B.astype(np.float64) - A, Cc.astype(np.float64) - A)
    det = -(d[s].astype(np.float64) * N[s]).sum(axis=1)
    want = np.float32(1e-8) * rng.choice(np.array([-1, 1], dtype=np.float32), len(s))
    want = np.where(rng.random(len(s)) < 0.33, np.nextafter(want, np.float32(np.inf)), np.where(rng.random(len(s)) < 0.5, np.nextafter(want, np.float32(-np.inf)), want))
    f = np.sqrt(np.abs(want.astype(np.float64) / np.where(det == 0, 1.0, det)))[:, None]
    B[s] = (A[s] + (B[s] - A[s]) * f).astype(np.float32)
    Cc[s] = (A[s] + (Cc[s] - A[s]) * f).astype(np.float32)
    s = cls == 3
    d[s] = _axis_aligned(rng, d[s])
    s = cls == 4
    big = np.float32(10.0) ** rng.uniform(2, 30, (int(s.sum()), 1)).astype(np.float32)
    for v in (A, B, Cc, pos):
        v[s] *= big
    nA, nB, nC = _unit(rng, n), _unit(rng, n), _unit(rng, n)
    cull = (rng.random(n) < 0.5).astype(np.uint32)
    rec = np.concatenate([pos, d, A, B, Cc, nA, nB, nC], axis=1).view(np.uint32)
    s = cls == 5
    rec[s] = _sprinkle(rng, rec[s].copy(), 0.1).view(np.uint32)
    return np.concatenate([rec, cull[:, None]], axis=1), cls


def sphere_cases(rng, n):
    """pos, dir, centre, radius.  Classes: generic; near-tangent rays (offset r, r (1 +- 1e-7), r (1 + 1e-6) from the centre in float64,
    so the float32 discriminant is near 0, not exactly 0); origin on the surface (up to rounding); radius with
    r*r = 0, subnormal or inf; zero or subnormal direction; far away (D up to 1e5); special values anywhere."""
    cen = _vec(rng, n, 4.0)
    r = np.abs(rng.standard_normal(n)).astype(np.float32) + np.float32(0.05)
    d = _unit(rng, n)
    pos = _vec(rng, n, 8.0)
    cls = rng.integers(0, 7, n)
    s = np.flatnonzero(cls == 1)                                   # tangent: offset perpendicular to dir by exactly r (up to rounding)
    perp = np.cross(d[s], _unit(rng, len(s)))
    perp /= np.linalg.norm(perp, axis=1, keepdims=True)
    graze = 1.0 + rng.choice(np.array([0.0, 1e-7, -1e-7, 1e-6]), len(s))
    pos[s] = (cen[s] + perp * (r[s] * graze)[:, None] - d[s] * np.float32(3.0)).astype(np.float32)
    s = np.flatnonzero(cls == 2)                                   # origin on the surface
    pos[s] = (cen[s] + _unit(rng, len(s)) * r[s][:, None]).astype(np.float32)
    s = np.flatnonzero(cls == 3)                                   # r*r = 0, subnormal, inf
    r[s] = rng.choice(np.array([0.0, -0.0, 1e-23, 1e-20, 3e-39, 2e19, 1e30, np.inf], dtype=np.float32), len(s))
    s = np.flatnonzero(cls == 4)                                   # zero / subnormal direction: a = 0 or subnormal
    d[s] = (d[s] * rng.choice(np.array([0.0, 1e-23, 1e-20, 1e-40], dtype=np.float32), len(s))[:, None]).astype(np.float32)
    s = cls == 5
    far = np.float32(10.0) ** rng.uniform(2, 5, (int(s.sum()), 1)).astype(np.float32)
    pos[s] = (pos[s] * far).astype(np.float32)
    rec = np.concatenate([pos, d, cen, r[:, None]], axis=1)
    s = cls == 6
    rec[s] = _sprinkle(rng, rec[s], 0.15)
    return rec.view(np.uint32), cls


def sphere_gate_cases(rng, n, lengths=None):
    """sphere_cases over the query gate's domain: pos, dir, centre, radius and an origin box (n, 6) that holds the ray origin and the
    sphere.  Classes: 0 aimed at a point inside the sphere from up to 8 units away; 1 near-tangent, as sphere_cases; 2 from the surface
    (up to rounding) in any direction, as a bounce leaves it; 3 from anywhere in a box that holds the sphere and a point up to 1e5
    away, aimed at a point inside the sphere.  Direction lengths log-uniform over the gate's [2^-10, 2^10] with both bounds
    (gate_lengths), or `lengths` (n,)."""
    cen = rng.standard_normal((n, 3)) * 4.0
    r = np.abs(rng.standard_normal(n)) + 0.05
    pos = rng.standard_normal((n, 3)) * 8.0
    aim = cen + _unit(rng, n) * (r * rng.random(n))[:, None]
    cls = rng.integers(0, 4, n)
    far = cen + _unit(rng, n) * (10.0 ** rng.uniform(0, 5, n))[:, None]
    lo, hi = np.minimum(far, cen - r[:, None]), np.maximum(far, cen + r[:, None])
    s = np.flatnonzero(cls == 3)
    pos[s] = lo[s] + rng.random((len(s), 3)) * (hi[s] - lo[s])
    d = aim - pos
    s = np.flatnonzero(cls == 1)                                   # tangent: offset perpendicular to dir by r (1 + {0, +-1e-7, 1e-6})
    u = _unit(rng, len(s)).astype(np.float64)
    perp = np.cross(u, _unit(rng, len(s)))
    perp /= np.linalg.norm(perp, axis=1, keepdims=True)
    pos[s] = cen[s] + perp * (r[s] * (1.0 + rng.choice(np.array([0.0, 1e-7, -1e-7, 1e-6]), len(s))))[:, None] - u * 3.0
    d[s] = u
    s = np.flatnonzero(cls == 2)                                   # on the surface, any direction
    pos[s] = cen[s] + _unit(rng, len(s)) * r[s][:, None]
    d[s] = rng.standard_normal((len(s), 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    d *= (gate_lengths(rng, n) if lengths is None else np.asarray(lengths, dtype=np.float64))[:, None]
    pos32, c32, r32 = pos.astype(np.float32), cen.astype(np.float32), r.astype(np.float32)
    origin = np.concatenate([np.minimum(np.minimum(lo, pos32), c32 - r32[:, None]), np.maximum(np.maximum(hi, pos32), c32 + r32[:, None])], axis=1)
    rec = np.concatenate([pos32, d.astype(np.float32), c32, r32[:, None]], axis=1)
    return rec.view(np.uint32), cls, origin.astype(np.float32)


TLAS_SIZES = (1, 2, 4, 5, 17, 129, 4096)


def tlas_boxes(rng, n):
    """n padded model boxes (n, 6: min xyz, max xyz) as planTlas receives them.  Classes: generic boxes scattered over 10 .. 1e4
    units; cells of a grid, which share faces exactly; flat boxes (min = max on an axis); bounds at +-0; a NaN bound; the infinite
    box of a model worldBoxOfModel cannot place."""
    spread = 10.0 ** rng.uniform(1, 4)
    c = rng.uniform(-1, 1, (n, 3)) * spread
    h = np.exp(rng.uniform(np.log(1e-4), np.log(0.3), (n, 3))) * spread
    lo, hi = c - h, c + h
    cls = rng.integers(0, 6, n)
    s = np.flatnonzero(cls == 1)                                    # grid cells: neighbours share a face
    cell = spread / 8
    g = rng.integers(-4, 4, (len(s), 3)).astype(np.float64)
    lo[s], hi[s] = g * cell, (g + rng.integers(1, 3, (len(s), 3))) * cell
    s = np.flatnonzero(cls == 2)                                    # flat on one axis
    ax = rng.integers(0, 3, len(s))
    hi[s, ax] = lo[s, ax]
    s = np.flatnonzero(cls == 3)                                    # a bound at +-0
    ax = rng.integers(0, 3, len(s))
    lo[s, ax] = np.minimum(lo[s, ax], -1.0)
    hi[s, ax] = np.where(rng.random(len(s)) < 0.5, 0.0, -0.0)
    flip = rng.random(len(s)) < 0.5
    lo[s[flip], ax[flip]] = np.where(rng.random(int(flip.sum())) < 0.5, 0.0, -0.0)
    hi[s[flip], ax[flip]] = np.abs(hi[s[flip], ax[flip]]) + 1.0
    box = np.concatenate([lo, hi], axis=1).astype(np.float32)
    s = np.flatnonzero(cls == 4)                                    # a NaN bound
    box[s, rng.integers(0, 6, len(s))] = np.nan
    s = np.flatnonzero((cls == 5) & (rng.random(n) < 0.1))          # the infinite box of a singular model (rare: it marks every ray)
    box[s, :3], box[s, 3:] = -np.inf, np.inf
    return box


def tlas_rays(rng, boxes, m):
    """(m, 7) rays pos, dir, bestDst against `boxes`.  Directions: generic, axis-aligned (+-0 components, invDir = +-inf), lengths over
    the query gate's range.  Origins: anywhere around the boxes, on a slab plane of some box (with the direction parallel to it: 0 x inf),
    at a box corner.  bestDst: +inf, the distance to some box's corner, 0, -0, a tiny or huge value, NaN."""
    fin = np.where(np.isfinite(boxes), boxes, 0.0).astype(np.float64)
    span = max(float(np.abs(fin).max()), 1.0)
    pos = rng.uniform(-1.2, 1.2, (m, 3)) * span
    d = rng.standard_normal((m, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    d *= gate_lengths(rng, m)[:, None]
    d = d.astype(np.float32)
    cls = rng.integers(0, 4, m)
    pick = rng.integers(0, len(boxes), m)
    s = np.flatnonzero(cls == 1)
    d[s] = _axis_aligned(rng, d[s])
    s = np.flatnonzero(cls == 2)                                    # on a slab plane of a box or one ulp inside it, parallel to it
    ax = rng.integers(0, 3, len(s))
    side = rng.integers(0, 2, len(s))
    face = fin[pick[s], ax + 3 * side].astype(np.float32)
    inward = np.where(side == 0, np.float32(np.inf), np.float32(-np.inf))
    pos[s, ax] = np.where(rng.random(len(s)) < 0.5, face, np.nextafter(face, inward))
    d[s, ax] = np.where(rng.random(len(s)) < 0.5, np.float32(0.0), np.float32(-0.0))
    s = np.flatnonzero(cls == 3)                                    # at a corner, axis-aligned half of the time
    pos[s] = np.where(rng.random((len(s), 3)) < 0.5, fin[pick[s], :3], fin[pick[s], 3:])
    half = s[rng.random(len(s)) < 0.5]
    d[half] = _axis_aligned(rng, d[half])
    corner = np.where(rng.random((m, 3)) < 0.5, fin[pick, :3], fin[pick, 3:])
    best = (np.linalg.norm(corner - pos, axis=1) / np.maximum(np.linalg.norm(d.astype(np.float64), axis=1), 1e-30)).astype(np.float32)
    kind = rng.random(m)
    best = np.where(kind < 0.3, np.float32(np.inf), best)
    special = np.array([0.0, -0.0, 1e-30, 1e-6, 3.4028235e38, np.nan], dtype=np.float32)
    best = np.where(kind > 0.85, rng.choice(special, m), best).astype(np.float32)
    return np.concatenate([pos.astype(np.float32), d, best[:, None]], axis=1)


def shading_cases(rng, n):
    """inDir, normal, iorA, iorB.  Classes: generic glass (one ior 1, the other in [1, 2.5]); total internal reflection at sinSqr == 1
    exactly (grazing incidence with equal iors) and around it; ior in {0, 1, negative}; special values anywhere."""
    nrm = _unit(rng, n)
    d = _unit(rng, n)
    d = np.where(((d * nrm).sum(axis=1) > 0)[:, None], -d, d).astype(np.float32)
    glass = rng.uniform(1.0, 2.5, n).astype(np.float32)
    inside = rng.random(n) < 0.5
    iorA = np.where(inside, glass, np.float32(1.0)).astype(np.float32)
    iorB = np.where(inside, np.float32(1.0), glass).astype(np.float32)
    cls = rng.integers(0, 4, n)
    s = np.flatnonzero(cls == 1)                                   # cosAngleIn = 0 with equal iors: sinSqr = 1 exactly
    t = np.cross(nrm[s], _unit(rng, len(s)))
    t = (t / np.linalg.norm(t, axis=1, keepdims=True)).astype(np.float32)
    exact = rng.random(len(s)) < 0.5
    d[s[exact]] = np.array([1.0, 0.0, 0.0], dtype=np.float32)
    nrm[s[exact]] = np.array([0.0, 1.0, 0.0], dtype=np.float32)
    d[s[~exact]] = t[~exact]
    iorA[s] = iorB[s] = rng.choice(np.array([1.0, 1.5, 1.0000001], dtype=np.float32), len(s))
    s = np.flatnonzero(cls == 2)
    iorA[s] = rng.choice(np.array([0.0, 1.0, -1.5, -0.0], dtype=np.float32), len(s))
    iorB[s] = rng.choice(np.array([0.0, 1.0, -1.0, 1.5], dtype=np.float32), len(s))
    rec = np.concatenate([d, nrm, iorA[:, None], iorB[:, None]], axis=1)
    s = cls == 3
    rec[s] = _sprinkle(rng, rec[s], 0.15)
    return rec.view(np.uint32), cls


def checker_cases(rng, n):
    """pos, normal, isSpecularBounce, flag, diffuse, emission, specular.  Positions on and next to checker-cell boundaries (multiples of
    1/1.5), all three projection planes and normals with tied components, both material flags."""
    cell = rng.integers(-20, 20, (n, 3)).astype(np.float64) / 1.5
    pos = cell.astype(np.float32)
    jitter = rng.choice(np.array([0, 1, -1, 2]), (n, 3))
    pos = np.where(jitter == 1, np.nextafter(pos, np.float32(np.inf)), np.where(jitter == -1, np.nextafter(pos, np.float32(-np.inf)),
                   np.where(jitter == 2, (pos + rng.uniform(-0.5, 0.5, (n, 3))).astype(np.float32), pos))).astype(np.float32)
    nrm = _unit(rng, n)
    tie = rng.random(n) < 0.3
    nrm[tie] = rng.choice(np.array([0.0, -0.0, 0.5, -0.5, 1.0], dtype=np.float32), (int(tie.sum()), 3))
    spec = (rng.random(n) < 0.3).astype(np.uint32)
    flag = np.where(rng.random(n) < 0.8, 1, rng.integers(0, 3, n)).astype(np.uint32)
    cols = rng.random((n, 9)).astype(np.float32)
    return np.concatenate([pos.view(np.uint32), nrm.view(np.uint32), spec[:, None], flag[:, None], cols.view(np.uint32)], axis=1), None


def sky_cases(rng, n, sun_focus):
    """dir, SunFocus, SunIntensity, dirToSun, SunColour: dir.y around +-0 and the -0.01 edge of the ground blend, the sun direction
    itself and directions next to it."""
    d = _unit(rng, n)
    cls = rng.integers(0, 4, n)
    s = np.flatnonzero(cls == 1)
    d[s, 1] = rng.choice(np.array([0.0, -0.0, -0.01, 0.4, 1e-45, -1e-45], dtype=np.float32), len(s))
    d[s, 1] = np.where(rng.random(len(s)) < 0.3, np.nextafter(d[s, 1], np.float32(np.inf)), d[s, 1])
    d[s, 1] = np.where(rng.random(len(s)) < 0.3, np.nextafter(d[s, 1], np.float32(-np.inf)), d[s, 1])
    sun = _unit(rng, n)
    s = np.flatnonzero(cls == 2)
    d[s] = sun[s]
    focus = rng.choice(np.asarray(sun_focus, dtype=np.float32), n)
    inten = rng.choice(np.array([0.0, 1.0, 10.0, 8.0], dtype=np.float32), n)
    col = rng.random((n, 3)).astype(np.float32)
    rec = np.concatenate([d, focus[:, None], inten[:, None], sun, col], axis=1)
    s = cls == 3
    rec[s] = _sprinkle(rng, rec[s], 0.1)
    return rec.view(np.uint32), cls


def model_cases(rng, n):
    """One single-triangle model per case, the triangle local size 1e-3 .. 100, worldToLocal = rotation x non-uniform scale (0.3 .. 3,
    mirrored in a third of the cases) x rotation + translation, models up to 1e5 from the origin, rays from up to 1e5 away aimed at
    the triangle's interior, at its edges and vertices (weights 0 or +-1e-7) and just outside (weight -1e-5).
    Returns (worldToLocal column-major (n, 16) float32, triangle (n, 9) local A B C, geometry box (n, 6), ray pos (n, 3), dir (n, 3),
    origin box (n, 6), cull (n,))."""
    scale = rng.uniform(0.3, 3.0, (n, 3)) * np.where(rng.random((n, 3)) < 0.1, -1.0, 1.0)
    A = _rotations(rng, n) @ (scale[:, :, None] * _rotations(rng, n))         # x_local = A x_world + t
    return _model_records(rng, n, A)


def _rotations(rng, k):
    q = rng.standard_normal((k, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    w, x, y, z = q.T
    return np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                     2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                     2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], axis=1).reshape(k, 3, 3)


# the query gate of rt_kernel_query.cuh: model skipping, the TLAS and the sphere accelerator are used for 2^-20 <= dot(dir, dir) <= 2^20
GATE_LEN_MIN, GATE_LEN_MAX = 2.0 ** -10, 2.0 ** 10


def gate_lengths(rng, n, lo=GATE_LEN_MIN, hi=GATE_LEN_MAX):
    """Direction lengths log-uniform over [lo, hi], the bounds themselves in a tenth of the cases."""
    L = np.exp(rng.uniform(np.log(lo), np.log(hi), n))
    edge = rng.random(n)
    return np.where(edge < 0.05, lo, np.where(edge < 0.1, hi, L))


def model_gate_cases(rng, n, lengths=None):
    """model_cases over the query gate's domain.  worldToLocal: rotation x scale x rotation with singular values log-uniform in
    1e-3 .. 1e3 (class bit 0 clear), or the product of two rotation x scale pairs (a rotated child of a non-uniformly scaled parent:
    sheared, singular values spread over about the same range; bit 0 set).  Rays (class >> 1): 0 from up to 1e5 away aimed at the
    triangle, as model_cases; 1 from anywhere in an origin box that holds the geometry and a point up to 1e5 away, aimed at the
    triangle; 2 from a point of the triangle itself in any direction, as a bounce leaves a surface.  Direction lengths log-uniform
    over the gate's [2^-10, 2^10] with both bounds (gate_lengths), or `lengths` (n,).  Returns model_cases' tuple and the class."""
    shear = rng.random(n) < 0.5
    s1 = np.exp(rng.uniform(np.log(1e-3), np.log(1e3), (n, 3))) * np.where(rng.random((n, 3)) < 0.1, -1.0, 1.0)
    A = _rotations(rng, n) @ (s1[:, :, None] * _rotations(rng, n))
    s2 = np.exp(rng.uniform(np.log(10 ** -1.5), np.log(10 ** 1.5), (n, 2, 3)))
    B = (s2[:, 0, :, None] * _rotations(rng, n)) @ (s2[:, 1, :, None] * _rotations(rng, n))
    A[shear] = B[shear]
    origin_cls = rng.integers(0, 3, n)
    L = gate_lengths(rng, n) if lengths is None else np.asarray(lengths, dtype=np.float64)
    return _model_records(rng, n, A, origin_cls, L) + (shear.astype(int) + 2 * origin_cls,)


def _model_records(rng, n, A, origin_cls=None, L=None):
    size = 10.0 ** rng.uniform(-3, 2, n)
    centre_local = rng.standard_normal((n, 3)) * size[:, None] * rng.uniform(0, 3, (n, 1))
    tri = centre_local[:, None, :] + rng.standard_normal((n, 3, 3)) * size[:, None, None]
    tri = tri.astype(np.float32).astype(np.float64)
    world_pos = rng.standard_normal((n, 3)) * (10.0 ** rng.uniform(0, 5, n))[:, None]
    t = -np.einsum("nij,nj->ni", A, world_pos)                      # the model sits at world_pos
    M = np.zeros((n, 4, 4))
    M[:, :3, :3], M[:, :3, 3], M[:, 3, 3] = A, t, 1.0
    w2l = M.astype(np.float32)
    A32, t32 = w2l[:, :3, :3].astype(np.float64), w2l[:, :3, 3].astype(np.float64)
    bary = rng.dirichlet((1.0, 1.0, 1.0), n)
    cls = rng.integers(0, 3, n)
    k = rng.integers(0, 3, n)
    e = np.flatnonzero(cls == 1)                                    # on an edge / vertex, up to a weight of 1e-7
    bary[e, k[e]] = rng.choice(np.array([0.0, 1e-7, -1e-7]), len(e))
    o = np.flatnonzero(cls == 2)                                    # just outside an edge
    bary[o, k[o]] = -1e-5
    bary /= bary.sum(axis=1, keepdims=True)
    target_local = np.einsum("nk,nkj->nj", bary, tri)
    target = np.linalg.solve(A32, (target_local - t32)[:, :, None])[:, :, 0]
    d = rng.standard_normal((n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    dist = 10.0 ** rng.uniform(-1, 5, n)
    pos = (target - d * dist[:, None]).astype(np.float32)
    world_tri = np.linalg.solve(A32[:, None], (tri - t32[:, None, :])[..., None])[..., 0]        # the vertices in world space
    lo = np.minimum(pos.astype(np.float64), world_tri.min(axis=1))                               # origin box: camera and geometry
    hi = np.maximum(pos.astype(np.float64), world_tri.max(axis=1))
    if origin_cls is not None:
        s = np.flatnonzero(origin_cls == 1)                         # anywhere in the origin box, aimed at the target
        p = lo[s] + rng.random((len(s), 3)) * (hi[s] - lo[s])
        pos[s] = p.astype(np.float32)
        d[s] = target[s] - pos[s]
        s = np.flatnonzero(origin_cls == 2)                         # on the triangle, any direction
        w = rng.dirichlet((1.0, 1.0, 1.0), len(s))
        pos[s] = np.einsum("nk,nkj->nj", w, world_tri[s]).astype(np.float32)
        d[s] = rng.standard_normal((len(s), 3))
        d /= np.linalg.norm(d, axis=1, keepdims=True)
        d *= L[:, None]
        lo, hi = np.minimum(lo, pos.astype(np.float64)), np.maximum(hi, pos.astype(np.float64))
    d = d.astype(np.float32)
    geo = np.concatenate([tri.min(axis=1), tri.max(axis=1)], axis=1).astype(np.float32)
    origin = np.concatenate([lo, hi], axis=1).astype(np.float32)
    cull = (rng.random(n) < 0.5).astype(np.uint32)
    return w2l.transpose(0, 2, 1).reshape(n, 16), tri.reshape(n, 9).astype(np.float32), geo, pos, d, origin, cull
