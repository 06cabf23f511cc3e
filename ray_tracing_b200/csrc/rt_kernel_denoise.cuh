// rt_kernel_denoise.cuh — rtDenoise: the edge-avoiding a-trous filter (Dammertz et al., HPG 2010) over the albedo-demodulated colour,
// guided by the feature images.  The arithmetic is stated bit for bit in include/rt_b200.h; this file only schedules it.
//
// k_denoise_prepare (one thread per pixel) writes three images: the demodulated colour e (float4, w unused), the guide (normal, depth)
// with a NaN depth marking background, and DenoisedRender itself, which holds (c, 1) for background and (m, 1) for the others until
// the last pass multiplies m by the filtered e.  k_denoise_pass runs one iteration: e ping-pongs between two scratch images, and the
// last pass writes DenoisedRender instead.
//
// Sub-lattice tiling: at step s the taps of pixel (x, y) are the pixels (x + s*i, y + s*j), all of the residue class (x mod s, y mod s).
// A CTA takes a 32x8 tile of ONE class's lattice (blockIdx.z = class), so its taps form a dense 5x5 stencil on that lattice and the
// tile plus a 2-point halo, 36x12 points of e and guide, is staged in shared memory once: 432 points for 256 outputs, whatever the step.
// -DRT_DENOISE_PLAIN builds the other arm of that choice (tools/build_variants.py "denoise_plain"): the same lattice order, every tap
// loaded from global memory through the read-only cache.  Both give the same bits; DESIGN.md section 7d has the measurement.
#pragma once
#include "rt_devmath.cuh"

namespace rtd {

constexpr int DN_TX = 32, DN_TY = 8, DN_HALO = 2;
constexpr int DN_SX = DN_TX + 2 * DN_HALO, DN_SY = DN_TY + 2 * DN_HALO;

struct DenoiseParams
{
    const float4* colour;                    // AccumulatedRender (useAccumulated) or FrameRender
    const float4* albedo;                    // AccumulatedAlbedo (useAccumulated)
    const float4* normal;                    // AccumulatedNormal (useAccumulated)
    const RtPixelFeatures* features;         // FeatureFrame (frame source)
    float4* e[2];                            // demodulated colour, ping-pong
    float4* guide;                           // (n, z); z = NaN: background
    float4* out;                             // DenoisedRender
    int W, H, useAccumulated;
    float invN, invZ;
};

// one iteration's constants, from the host (include/rt_b200.h)
struct DenoisePass
{
    float cK, rd1, rd2;                      // invC * 4^k, 2^-k, 2^-(k+1)
    int step, src, last;                     // s = 2^k; e[src] is read, e[src ^ 1] (or DenoisedRender when last) written
};

RT_DI bool finite1(float v) { return fabsf(v) < inf32(); }

__global__ void __launch_bounds__(256) k_denoise_prepare(const __grid_constant__ DenoiseParams P)
{
    const size_t n = (size_t)P.W * P.H;
    const size_t p = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (p >= n) return;
    f3 c, a, nn; float z; bool bg;
    if (P.useAccumulated)
    {
        const float4 A = P.colour[p], L = P.albedo[p], N = P.normal[p];
        bg = A.w == 0.0f || L.w == 0.0f;
        c = A.w == 0.0f ? splat3(0.0f) : make_f3(A.x / A.w, A.y / A.w, A.z / A.w);
        a = make_f3(L.x / L.w, L.y / L.w, L.z / L.w);
        nn = make_f3(N.x / L.w, N.y / L.w, N.z / L.w);
        z = N.w / L.w;
    }
    else
    {
        const float4 C = P.colour[p];
        const float4* f = reinterpret_cast<const float4*>(P.features + p);
        const float4 f0 = f[0], f1 = f[1];
        bg = __float_as_int(f1.w) == -1;
        c = make_f3(C.x, C.y, C.z);
        a = make_f3(f0.x, f0.y, f0.z);
        nn = make_f3(f1.x, f1.y, f1.z);
        z = f0.w;
    }
    const f3 m = make_f3(fmaxf(a.x, 0.00390625f), fmaxf(a.y, 0.00390625f), fmaxf(a.z, 0.00390625f));
    const f3 e = make_f3(c.x / m.x, c.y / m.y, c.z / m.z);
    bg = bg || !(finite1(c.x) && finite1(c.y) && finite1(c.z) && finite1(a.x) && finite1(a.y) && finite1(a.z) &&
                 finite1(nn.x) && finite1(nn.y) && finite1(nn.z) && finite1(z) && finite1(e.x) && finite1(e.y) && finite1(e.z));
    if (bg)
    {
        P.guide[p] = make_float4(0.0f, 0.0f, 0.0f, nan32());
        P.out[p] = make_float4(c.x, c.y, c.z, 1.0f);
        return;
    }
    P.guide[p] = make_float4(nn.x, nn.y, nn.z, z);
    P.e[0][p] = make_float4(e.x, e.y, e.z, 0.0f);
    P.out[p] = make_float4(m.x, m.y, m.z, 1.0f);
}

// rtDenoiseTemporal's passes (rt_kernel_temporal.cuh) run the same tiling with the variance-guided weights: e.w carries the variance
struct TemporalPassParams : DenoiseParams
{
    float4* hist;                            // the colour history: iteration 0's output
    float* gv;                               // this iteration's prefiltered variance (k_temporal_prefilter)
    float sigmaL;
};

RT_DI float luminance(float4 e) { return (0.2126f * e.x + 0.7152f * e.y) + 0.0722f * e.z; }

// One iteration of either filter: SVGF = false is rtDenoise's, true rtDenoiseTemporal's (include/rt_b200.h states both)
template <bool SVGF, class PP>
RT_DI void denoise_pass_body(const PP& P, const DenoisePass& S)
{
    const int s = S.step;
    const int rx = (int)blockIdx.z % s, ry = (int)blockIdx.z / s;             // the residue class of this CTA's lattice
    const int LW = rx < P.W ? (P.W - rx + s - 1) / s : 0, LH = ry < P.H ? (P.H - ry + s - 1) / s : 0;
    const int lx0 = (int)blockIdx.x * DN_TX, ly0 = (int)blockIdx.y * DN_TY;
    if (lx0 >= LW || ly0 >= LH) return;                                        // the whole CTA: no lattice point here
    const float4* __restrict__ eIn = P.e[S.src];
    const int tx = (int)threadIdx.x % DN_TX, ty = (int)threadIdx.x / DN_TX;

#ifndef RT_DENOISE_PLAIN
    __shared__ float4 sE[DN_SY * DN_SX], sG[DN_SY * DN_SX];
    for (int t = (int)threadIdx.x; t < DN_SY * DN_SX; t += DN_TX * DN_TY)
    {
        const int lx = lx0 - DN_HALO + t % DN_SX, ly = ly0 - DN_HALO + t / DN_SX;
        const int x = rx + lx * s, y = ry + ly * s;
        float4 g = make_float4(0.0f, 0.0f, 0.0f, nan32()), e = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        if (lx >= 0 && ly >= 0 && x < P.W && y < P.H)                          // outside the image: skipped like background
        {
            const size_t q = (size_t)y * P.W + x;
            g = __ldg(P.guide + q);
            if (g.w == g.w) e = __ldg(eIn + q);
        }
        sG[t] = g; sE[t] = e;
    }
    __syncthreads();
#define RT_DN_TAP(i, j, E, G) { const int o_ = (ty + DN_HALO + (j)) * DN_SX + tx + DN_HALO + (i); E = sE[o_]; G = sG[o_]; }
#else
#define RT_DN_TAP(i, j, E, G) { const int qx_ = x + s * (i), qy_ = y + s * (j);                                                        \
        G = make_float4(0.0f, 0.0f, 0.0f, nan32());                                                                                     \
        if (qx_ >= 0 && qy_ >= 0 && qx_ < P.W && qy_ < P.H) { const size_t q_ = (size_t)qy_ * P.W + qx_; G = __ldg(P.guide + q_);      \
                                                              if (G.w == G.w) E = __ldg(eIn + q_); } }
#endif

    const int lx = lx0 + tx, ly = ly0 + ty;
    if (lx >= LW || ly >= LH) return;
    const int x = rx + lx * s, y = ry + ly * s;
    float4 ep, gp;
    RT_DN_TAP(0, 0, ep, gp);
    if (gp.w != gp.w) return;                                                  // background: DenoisedRender already holds (c, 1)
    const float rz = P.invZ / gp.w;
    float sw = 0.0f, sr = 0.0f, sg = 0.0f, sb = 0.0f;
    float kL = 0.0f, lp = 0.0f, sv = 0.0f;
    if constexpr (SVGF)
    {
#ifdef RT_TEMPORAL_LATTICE_PREFILTER
        // build variant for the A/B of DESIGN.md section 7d''''''' (tools/build_variants.py temporal_lattice): the 3x3 Gaussian over
        // the lattice neighbours at +-s, read from the staged tile.  Not SVGF's form and not the header's: no oracle restates it.
        float gw = 0.0f, gv = 0.0f;
#pragma unroll
        for (int j = -1; j <= 1; j++)
        {
#pragma unroll
            for (int i = -1; i <= 1; i++)
            {
                float4 eq = make_float4(0.0f, 0.0f, 0.0f, 0.0f), gq;
                RT_DN_TAP(i, j, eq, gq);
                if (gq.w != gq.w) continue;
                const float k = (i == 0 ? 0.5f : 0.25f) * (j == 0 ? 0.5f : 0.25f);
                gw = gw + k; gv = gv + k * eq.w;
            }
        }
        const float gvp = gv / gw;
#else
        const float gvp = P.gv[(size_t)y * P.W + x];                           // SVGF's 3x3 Gaussian over the immediate neighbours
#endif
        kL = 1.0f / (P.sigmaL * sqrtf(gvp) + RT_TEMPORAL_EPSILON);
        lp = luminance(ep);
    }
#pragma unroll
    for (int j = -2; j <= 2; j++)
    {
#pragma unroll
        for (int i = -2; i <= 2; i++)
        {
            const float hi = (i == 0 ? 0.375f : (i == 1 || i == -1) ? 0.25f : 0.0625f), hj = (j == 0 ? 0.375f : (j == 1 || j == -1) ? 0.25f : 0.0625f);
            float4 eq = make_float4(0.0f, 0.0f, 0.0f, 0.0f), gq;
            float w;
            if (i == 0 && j == 0) { eq = ep; w = 0.140625f; }
            else
            {
                RT_DN_TAP(i, j, eq, gq);
                if (gq.w != gq.w) continue;
                const float dr = ep.x - eq.x, dg = ep.y - eq.y, db = ep.z - eq.z;
                const float nx = gp.x - gq.x, ny = gp.y - gq.y, nz = gp.z - gq.z;
                const int d = (i < 0 ? -i : i) > (j < 0 ? -j : j) ? (i < 0 ? -i : i) : (j < 0 ? -j : j);
                const float t = ((gp.w - gq.w) * rz) * (d == 1 ? S.rd1 : S.rd2);
                const float D = SVGF ? (fabsf(lp - luminance(eq)) * kL + ((nx * nx + ny * ny) + nz * nz) * P.invN) + t * t
                                     : (((dr * dr + dg * dg) + db * db) * S.cK + ((nx * nx + ny * ny) + nz * nz) * P.invN) + t * t;
                if (!(D <= 103.972076416015625f)) continue;                    // exp_rt is exactly 0 there; a NaN D weighs 0 too
                w = (hi * hj) * exp_rt(-D);
                if (w == 0.0f) continue;
            }
            sw = sw + w;
            sr = sr + w * eq.x; sg = sg + w * eq.y; sb = sb + w * eq.z;
            if constexpr (SVGF) sv = sv + (w * w) * eq.w;
        }
    }
#undef RT_DN_TAP
    const size_t p = (size_t)y * P.W + x;
    const float er = sr / sw, eg = sg / sw, eb = sb / sw;
    if constexpr (SVGF) { if (s == 1) P.hist[p] = make_float4(er, eg, eb, 0.0f); }
    if (S.last)
    {
        const float4 m = P.out[p];
        P.out[p] = make_float4(er * m.x, eg * m.y, eb * m.z, 1.0f);
    }
    else P.e[S.src ^ 1][p] = make_float4(er, eg, eb, SVGF ? sv / (sw * sw) : 0.0f);
}

__global__ void __launch_bounds__(DN_TX * DN_TY) k_denoise_pass(const __grid_constant__ DenoiseParams P, const DenoisePass S)
{
    denoise_pass_body<false>(P, S);
}

__global__ void __launch_bounds__(DN_TX * DN_TY) k_temporal_pass(const __grid_constant__ TemporalPassParams P, const DenoisePass S)
{
    denoise_pass_body<true>(P, S);
}

// `iterations` filter passes of KERNEL on `stream`
template <class PP>
inline cudaError_t denoise_passes(void (*kernel)(PP, DenoisePass), const PP& P, const DenoisePass* passes, int iterations, cudaStream_t stream)
{
    cudaError_t e = cudaSuccess;
    for (int k = 0; k < iterations && e == cudaSuccess; k++)
    {
        const int s = passes[k].step;
        const unsigned LW = (unsigned)((P.W + s - 1) / s), LH = (unsigned)((P.H + s - 1) / s);
        const dim3 grid((LW + DN_TX - 1) / DN_TX, (LH + DN_TY - 1) / DN_TY, (unsigned)(s * s));
        RT_LAUNCH(grid, DN_TX * DN_TY, 0, stream, kernel, P, passes[k]);
        e = cudaGetLastError();
    }
    return e;
}

// The prepare pass and `iterations` filter passes on `stream`.  The caller has checked the arguments and computed the constants.
inline cudaError_t denoise_launch(const DenoiseParams& P, const DenoisePass* passes, int iterations, cudaStream_t stream)
{
    const size_t n = (size_t)P.W * P.H;
    RT_LAUNCH((unsigned)((n + 255) / 256), 256, 0, stream, k_denoise_prepare, P);
    cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? denoise_passes(k_denoise_pass, P, passes, iterations, stream) : e;
}

} // namespace rtd
