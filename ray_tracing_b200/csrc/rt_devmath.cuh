// rt_devmath.cuh — device-side FP32 arithmetic contract of the H100 path tracer.
//
// The kernels must return the same bits on the GPU as the CPU restatement of the reference shader
// does on the host, so every operation here is a single IEEE-754 binary32 op (RNE), evaluated in the
// order the HLSL writes it, and never contracted: this translation unit is compiled with -fmad=false
// (plus the default -prec-div=true -prec-sqrt=true -ftz=false).  HLSL intrinsics are pinned as
//   normalize(v) = v * (1/sqrt(dot(v,v)))      lerp(a,b,t) = a + t*(b-a)      dot: left-to-right sum
//   reflect(i,n) = i - (2*dot(n,i))*n          sign(0) = sign(NaN) = 0        min/max: NaN-ignoring
//   smoothstep(a,b,x): t = saturate((x-a)/(b-a)); t*t*(3-2t)                   (SURVEY.md §8a Q11)
// and log / exp / sin / cos / pow are polynomial routines made only of those IEEE ops (Cody–Waite
// range reduction + published minimax kernels), so they need no libdevice and are reproducible on any
// conforming FP32 machine.  Accuracy, exhaustive (DESIGN.md §2): < 1 ulp (log, exp); sin / cos < 1.5e-7 absolute on [0, 2π], the only angles the path uses (6.2831852 · RandomValue), but up to ~1e-6 on (2π, 1e5], NaN beyond ±1e5.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

// ---- build defaults of round 2 ---------------------------------------------------------------------------------------------------
// Every switch below was a compile-time candidate of round 1 and won its A/B comparison in round 2 (same image bits in every variant).
// They have not been re-tuned on the H100.  -DRT_DEFAULTS_R1 builds the round-1 kernels again (A/B runs, tools/build_variants.py "r1").
#ifndef RT_DEFAULTS_R1
#ifndef RT_VOTE_WL
#define RT_VOTE_WL 3               // cost-weighted vote of the trace phase: a leaf step is cheap and frees its lanes for the inner population
#endif
#ifndef RT_VOTE_WN
#define RT_VOTE_WN 2
#endif
#ifndef RT_SMEM_STACK
#define RT_SMEM_STACK 8            // the top 8 entries of every lane's traversal stack in a shared-memory ring (lane = bank), deeper ones spill to local memory
#endif
#ifndef RT_BRANCHLESS_POP
#define RT_BRANCHLESS_POP          // an inner step that misses both children takes the stack top by a select, not by a 2.4-lane branch
#endif
#ifndef RT_LEAF_REPEAT
#define RT_LEAF_REPEAT 2           // two leaf primitives per census
#endif
#ifndef RT_SPHERE_SAH_DEPTH
#define RT_SPHERE_SAH_DEPTH 20     // sphere accelerator: top 20 levels by the surface-area sweep ...
#endif
#ifndef RT_SPHERE_LEAF
#define RT_SPHERE_LEAF 1           // ... and one sphere per leaf (faster than leaves of 2, 4 or 8 on config 5)
#endif
#ifndef RT_PUSH_PREDICATED
#define RT_PUSH_PREDICATED         // the far child's push as two predicated ring stores; only the spill of a full ring branches
#endif
#endif

namespace rtd {

struct f2 { float x, y; };
struct f3 { float x, y, z; };

#define RT_DI __device__ __forceinline__
// out-of-line device function.  (RT_SIMT_EMU: the test-only host build of these kernels, tests/simt — never defined in the product build)
#ifdef RT_SIMT_EMU
#define RT_DNI __attribute__((noinline))
#else
#define RT_DNI __device__ __noinline__
#endif
// kernel launch: kernel<<<grid, block, smem, stream>>>(args)
#ifndef RT_SIMT_EMU
#define RT_LAUNCH(grid, block, smem, stream, kern, ...) kern<<<grid, block, smem, stream>>>(__VA_ARGS__)
#define RT_DYNAMIC_SMEM(name) extern __shared__ __align__(128) unsigned char name[]      // the CTA's dynamic shared memory
#endif

RT_DI f2 make_f2(float x, float y) { f2 r; r.x = x; r.y = y; return r; }
RT_DI f3 make_f3(float x, float y, float z) { f3 r; r.x = x; r.y = y; r.z = z; return r; }
RT_DI f3 splat3(float s) { return make_f3(s, s, s); }
RT_DI f3 load3(const float* p) { return make_f3(p[0], p[1], p[2]); }

RT_DI f3 operator+(f3 a, f3 b) { return make_f3(a.x + b.x, a.y + b.y, a.z + b.z); }
RT_DI f3 operator-(f3 a, f3 b) { return make_f3(a.x - b.x, a.y - b.y, a.z - b.z); }
RT_DI f3 operator*(f3 a, f3 b) { return make_f3(a.x * b.x, a.y * b.y, a.z * b.z); }
RT_DI f3 operator*(f3 a, float s) { return make_f3(a.x * s, a.y * s, a.z * s); }
RT_DI f3 operator*(float s, f3 a) { return make_f3(s * a.x, s * a.y, s * a.z); }
RT_DI f3 operator/(f3 a, float s) { return make_f3(a.x / s, a.y / s, a.z / s); }
RT_DI f3 operator-(f3 a) { return make_f3(-a.x, -a.y, -a.z); }
RT_DI f3 rcp3(f3 a) { return make_f3(1.0f / a.x, 1.0f / a.y, 1.0f / a.z); }

RT_DI float dot3(f3 a, f3 b) { return (a.x * b.x + a.y * b.y) + a.z * b.z; }
RT_DI f3 cross3(f3 a, f3 b) { return make_f3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }
#ifdef RT_NOINLINE_NORMALIZE
RT_DNI f3 normalize3(f3 v) { float inv = 1.0f / sqrtf(dot3(v, v)); return v * inv; }
#else
RT_DI f3 normalize3(f3 v) { float inv = 1.0f / sqrtf(dot3(v, v)); return v * inv; }
#endif
// IEEE quotient behind a call: for divisions on rarely taken paths, so the compiler cannot speculate them
RT_DNI float div_cold(float a, float b) { return a / b; }
RT_DI f3 lerp3(f3 a, f3 b, float t) { return a + t * (b - a); }
RT_DI f3 reflect3(f3 i, f3 n) { return i - (2.0f * dot3(n, i)) * n; }
RT_DI float sign1(float a) { return (a > 0.0f ? 1.0f : 0.0f) - (a < 0.0f ? 1.0f : 0.0f); }
RT_DI float saturate1(float a) { return fminf(fmaxf(a, 0.0f), 1.0f); }
RT_DI float smoothstep1(float a, float b, float x) { float t = saturate1((x - a) / (b - a)); return t * t * (3.0f - 2.0f * t); }

RT_DI float inf32() { return __uint_as_float(0x7f800000u); }
RT_DI float nan32() { return __uint_as_float(0x7fc00000u); }

// natural log: m in (sqrt2/2, sqrt2], s = f/(2+f), even/odd split minimax in s^2
RT_DI float log_rt(float x)
{
    uint32_t ix = __float_as_uint(x);
    if (x != x) return x;
    if ((ix << 1) == 0u) return -inf32();
    if (ix >> 31) return nan32();
    if (ix == 0x7f800000u) return x;
    int k = 0;
    if (ix < 0x00800000u) { x = x * 33554432.0f; ix = __float_as_uint(x); k = -25; }
    k += (int)(ix >> 23) - 127;
    float m = __uint_as_float((ix & 0x007fffffu) | 0x3f800000u);
    if (m > 1.41421354f) { m = m * 0.5f; k += 1; }
    const float f = m - 1.0f;
    const float s = f / (2.0f + f);
    const float z = s * s;
    const float w = z * z;
    const float t1 = w * (0.40000972152f + w * 0.24279078841f);
    const float t2 = z * (0.66666662693f + w * 0.28498786688f);
    const float R = t2 + t1;
    const float hfsq = (0.5f * f) * f;
    const float dk = (float)k;
    return dk * 6.9313812256e-01f - ((hfsq - (s * (hfsq + R) + dk * 9.0580006145e-06f)) - f);
}

// exp: k = round(x/ln2), r = x - k ln2 (two-constant), rational kernel, two-step power-of-two scaling
RT_DI float exp_rt(float x)
{
    if (x != x) return x;
    if (x > 88.72283935546875f) return inf32();
    if (x < -103.972076416015625f) return 0.0f;
    const float fk = x * 1.4426950216e+00f + (x < 0.0f ? -0.5f : 0.5f);
    const int k = (int)fk;
    const float t = (float)k;
    const float hi = x - t * 6.9314575195e-01f;
    const float lo = t * 1.4286067653e-06f;
    const float r = hi - lo;
    const float rr = r * r;
    const float c = r - rr * (1.6666625440e-1f + rr * -2.7667332906e-3f);
    const float y = 1.0f - ((lo - (r * c) / (2.0f - c)) - hi);
    const int k1 = k / 2, k2 = k - k1;
    return (y * __uint_as_float((uint32_t)(k1 + 127) << 23)) * __uint_as_float((uint32_t)(k2 + 127) << 23);
}

RT_DI void sincos_reduce_rt(float ax, int& q, float& r)
{
    const int n = (int)(ax * 0.636619772367581343f + 0.5f);
    const float fn = (float)n;
    r = ((ax - fn * 1.5703125f) - fn * 4.837512969970703125e-4f) - fn * 7.549789948768648e-8f;
    q = n & 3;
}
RT_DI float sin_poly_rt(float r)
{
    const float z = r * r;
    return ((((-1.9515295891e-4f * z + 8.3321608736e-3f) * z) - 1.6666654611e-1f) * z) * r + r;
}
RT_DI float cos_poly_rt(float r)
{
    const float z = r * r;
    const float y = (((2.443315711809948e-5f * z - 1.388731625493765e-3f) * z) + 4.166664568298827e-2f) * (z * z);
    return (y - 0.5f * z) + 1.0f;
}
RT_DI float sin_rt(float x)
{
    const float ax = fabsf(x);
    if (!(ax <= 100000.0f)) return nan32();
    int q; float r; sincos_reduce_rt(ax, q, r);
    float v = (q & 1) ? cos_poly_rt(r) : sin_poly_rt(r);
    if (q & 2) v = -v;
    return (x < 0.0f) ? -v : v;
}
RT_DI float cos_rt(float x)
{
    const float ax = fabsf(x);
    if (!(ax <= 100000.0f)) return nan32();
    int q; float r; sincos_reduce_rt(ax, q, r);
    float v = (q & 1) ? sin_poly_rt(r) : cos_poly_rt(r);
    if (q == 1 || q == 2) v = -v;
    return v;
}
// both at once (same reduction, same polynomials, hence the same bits as sin_rt / cos_rt)
RT_DI void sincos_rt(float x, float& s, float& c)
{
    const float ax = fabsf(x);
    if (!(ax <= 100000.0f)) { s = c = nan32(); return; }
    int q; float r; sincos_reduce_rt(ax, q, r);
    const float sp = sin_poly_rt(r), cp = cos_poly_rt(r);
    float sv = (q & 1) ? cp : sp; if (q & 2) sv = -sv;
    float cv = (q & 1) ? sp : cp; if (q == 1 || q == 2) cv = -cv;
    s = (x < 0.0f) ? -sv : sv; c = cv;
}
RT_DI float pow_rt(float x, float y) { return exp_rt(y * log_rt(x)); }

} // namespace rtd
