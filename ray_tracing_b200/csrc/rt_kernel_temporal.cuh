// rt_kernel_temporal.cuh — rtDenoiseTemporal: reprojected history and variance-guided a-trous filtering (SVGF, Schied et al., HPG 2017)
// over the albedo-demodulated colour of one frame.  The arithmetic is stated bit for bit in include/rt_b200.h; this file only schedules it.
//
// k_temporal_reproject (one thread per pixel) demodulates FrameRender, reprojects the pixel's first hit into the previous call's
// camera, validates and blends the 2x2 history footprint and writes the integrated colour (scratch e[0].rgb), the pixel's new history
// record (guide and moments), TemporalFrame.xyz and DenoisedRender's (m, 1) / (c, 1).  k_temporal_variance writes the variance into
// e[0].w and TemporalFrame.w: the moments' variance, or for a short history the 7x7 bilateral estimate.  Each iteration is
// k_temporal_prefilter (SVGF's 3x3 Gaussian of the variance over the immediate neighbours) and k_temporal_pass, rtDenoise's sub-lattice
// tiling (rt_kernel_denoise.cuh) with the variance-guided weights; e.w carries the variance through the ping-pong and iteration 0 also
// writes the colour history.
#pragma once
#include "rt_kernel_denoise.cuh"

namespace rtd {

struct TemporalParams
{
    const float4* colour;                    // FrameRender
    const RtPixelFeatures* features;         // FeatureFrame
    float4* e;                               // scratch: integrated colour (rgb) and variance (w)
    float4* out;                             // DenoisedRender: (m, 1), or (c, 1) for background
    float4* frame;                           // TemporalFrame
    float4* guide;                           // this call's history record: (n, z), z = NaN for background ...
    float4* mom;                             // ... and (m1, m2, len, object)
    const float4* prevGuide;                 // the previous call's records
    const float4* prevMom;
    const float4* prevColour;                // the previous call's colour history
    float inv[12];                           // rows of the previous camera's inverse affine map: (r00 r01 r02 b0), (r10 ...), (r20 ...)
    float prevOrigin[3];                     // the previous camera's translation
    float kx, ky;                            // VP'.z / VP'.x, VP'.z / VP'.y
    int W, H;
    int mode;                                // 0: no history, 1: reproject, 2: static camera
    float alpha, invN, invZ, invL;
};

enum { TEMPORAL_NONE = 0, TEMPORAL_REPROJECT = 1, TEMPORAL_STATIC = 2 };

RT_DI float lum3(f3 e) { return (0.2126f * e.x + 0.7152f * e.y) + 0.0722f * e.z; }

__global__ void __launch_bounds__(256) k_temporal_reproject(const __grid_constant__ TemporalParams T, const __grid_constant__ DevParams P)
{
    const size_t n = (size_t)T.W * T.H;
    const size_t p = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (p >= n) return;
    const int x = (int)(p % (size_t)T.W), y = (int)(p / (size_t)T.W);
    const float4 C = T.colour[p];
    const float4* f = reinterpret_cast<const float4*>(T.features + p);
    const float4 f0 = f[0], f1 = f[1];
    const int object = __float_as_int(f1.w);
    const f3 c = make_f3(C.x, C.y, C.z), a = make_f3(f0.x, f0.y, f0.z), nn = make_f3(f1.x, f1.y, f1.z);
    const float z = f0.w;
    const f3 m = make_f3(fmaxf(a.x, 0.00390625f), fmaxf(a.y, 0.00390625f), fmaxf(a.z, 0.00390625f));
    const f3 e = make_f3(c.x / m.x, c.y / m.y, c.z / m.z);
    const bool bg = object == -1 || !(finite1(c.x) && finite1(c.y) && finite1(c.z) && finite1(a.x) && finite1(a.y) && finite1(a.z) &&
                                      finite1(nn.x) && finite1(nn.y) && finite1(nn.z) && finite1(z) && finite1(e.x) && finite1(e.y) && finite1(e.z));
    if (bg)
    {
        T.out[p] = make_float4(c.x, c.y, c.z, 1.0f);
        T.guide[p] = make_float4(0.0f, 0.0f, 0.0f, nan32());
        T.mom[p] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        T.frame[p] = make_float4(nan32(), nan32(), 0.0f, 0.0f);
        return;
    }
    const float l = lum3(e);

    // reprojection of the pixel's first hit into the previous camera
    float px = nan32(), py = nan32(), zexp = 0.0f;
    if (T.mode == TEMPORAL_STATIC) { px = (float)x; py = (float)y; zexp = z; }
    else if (T.mode == TEMPORAL_REPROJECT)
    {
        const PixelSetup s = SetupPixel(P, (unsigned)x, (unsigned)y);
        const f3 d = normalize3(s.focusPoint - s.camOrigin);
        const f3 X = make_f3(s.camOrigin.x + d.x * z, s.camOrigin.y + d.y * z, s.camOrigin.z + d.z * z);
        const float Lx = ((T.inv[0] * X.x + T.inv[1] * X.y) + T.inv[2] * X.z) + T.inv[3];
        const float Ly = ((T.inv[4] * X.x + T.inv[5] * X.y) + T.inv[6] * X.z) + T.inv[7];
        const float Lz = ((T.inv[8] * X.x + T.inv[9] * X.y) + T.inv[10] * X.z) + T.inv[11];
        if (Lz > 0.0f)
        {
            const float u = (Lx / Lz) * T.kx + 0.5f, v = (Ly / Lz) * T.ky + 0.5f;
            const float qx = u * (float)(T.W - 1), qy = v * (float)(T.H - 1);
            const float dx = X.x - T.prevOrigin[0], dy = X.y - T.prevOrigin[1], dz = X.z - T.prevOrigin[2];
            const float ze = sqrtf((dx * dx + dy * dy) + dz * dz);
            if (finite1(X.x) && finite1(X.y) && finite1(X.z) && finite1(Lx) && finite1(Ly) && finite1(Lz) && finite1(u) && finite1(v) &&
                finite1(qx) && finite1(qy) && finite1(ze)) { px = qx; py = qy; zexp = ze; }
        }
    }

    // the bilinear 2x2 history footprint, valid taps only, in tap order
    float sw = 0.0f, sr = 0.0f, sg = 0.0f, sb = 0.0f, s1 = 0.0f, s2 = 0.0f, lenH = 0.0f;
    if (px > -1.0f && px < (float)T.W && py > -1.0f && py < (float)T.H)        // false for NaN; otherwise some tap may be inside
    {
        const float fx0 = floorf(px), fy0 = floorf(py);
        const int ix = (int)fx0, iy = (int)fy0;
        const float fx = px - fx0, fy = py - fy0;
        const float wx[2] = {1.0f - fx, fx}, wy[2] = {1.0f - fy, fy};
#pragma unroll
        for (int t = 0; t < 4; t++)
        {
            const int qx = ix + (t & 1), qy = iy + (t >> 1);
            const float w = wx[t & 1] * wy[t >> 1];
            if (w == 0.0f || qx < 0 || qy < 0 || qx >= T.W || qy >= T.H) continue;
            const size_t q = (size_t)qy * T.W + qx;
            const float4 g = T.prevGuide[q];
            if (g.w != g.w) continue;                                           // background in history
            const float4 M = T.prevMom[q];
            if (__float_as_int(M.w) != object) continue;
            if (!(fabsf(g.w - zexp) <= RT_TEMPORAL_TAU_Z * zexp)) continue;
            if (!(((nn.x * g.x + nn.y * g.y) + nn.z * g.z) >= RT_TEMPORAL_TAU_N)) continue;
            const float4 h = T.prevColour[q];
            sw = sw + w;
            sr = sr + w * h.x; sg = sg + w * h.y; sb = sb + w * h.z;
            s1 = s1 + w * M.x; s2 = s2 + w * M.y;
            lenH = fmaxf(lenH, M.z);
        }
    }

    // integration
    f3 col = e;
    float m1 = l, m2 = l * l, len = 1.0f;
    if (sw > 0.0f)
    {
        len = fminf(lenH + 1.0f, (float)RT_TEMPORAL_MAX_HISTORY);
        const float al = fmaxf(T.alpha, 1.0f / len);
        const float hr = sr / sw, hg = sg / sw, hb = sb / sw, h1 = s1 / sw, h2 = s2 / sw;
        col = make_f3(hr + al * (e.x - hr), hg + al * (e.y - hg), hb + al * (e.z - hb));
        m1 = h1 + al * (l - h1);
        m2 = h2 + al * (l * l - h2);
    }
    T.e[p] = make_float4(col.x, col.y, col.z, 0.0f);
    T.guide[p] = make_float4(nn.x, nn.y, nn.z, z);
    T.mom[p] = make_float4(m1, m2, len, __int_as_float(object));
    T.frame[p] = make_float4(px, py, len, 0.0f);
    T.out[p] = make_float4(m.x, m.y, m.z, 1.0f);
}

__global__ void __launch_bounds__(256) k_temporal_variance(const __grid_constant__ TemporalParams T)
{
    const size_t n = (size_t)T.W * T.H;
    const size_t p = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (p >= n) return;
    const float4 gp = T.guide[p];
    if (gp.w != gp.w) return;
    const float4 Mp = T.mom[p];
    float var;
    if (Mp.z >= 4.0f) var = fmaxf(Mp.y - Mp.x * Mp.x, 0.0f);
    else
    {
        // short history: the moments' bilateral 7x7 mean over non-background pixels, its variance boosted by 4 / len
        const int x = (int)(p % (size_t)T.W), y = (int)(p / (size_t)T.W);
        const float rz = T.invZ / gp.w;
        float sw = 0.0f, s1 = 0.0f, s2 = 0.0f;
        for (int j = -3; j <= 3; j++)
        {
            for (int i = -3; i <= 3; i++)
            {
                const int qx = x + i, qy = y + j;
                if (qx < 0 || qy < 0 || qx >= T.W || qy >= T.H) continue;
                const size_t q = (size_t)qy * T.W + qx;
                const float4 gq = T.guide[q];
                if (gq.w != gq.w) continue;
                const float4 Mq = T.mom[q];
                float w = 1.0f;
                if (i != 0 || j != 0)
                {
                    const float nx = gp.x - gq.x, ny = gp.y - gq.y, nz = gp.z - gq.z;
                    const float t = (gp.w - gq.w) * rz;
                    const float D = (fabsf(Mp.x - Mq.x) * T.invL + ((nx * nx + ny * ny) + nz * nz) * T.invN) + t * t;
                    if (!(D <= 103.972076416015625f)) continue;
                    w = exp_rt(-D);
                    if (w == 0.0f) continue;
                }
                sw = sw + w;
                s1 = s1 + w * Mq.x; s2 = s2 + w * Mq.y;
            }
        }
        const float a1 = s1 / sw, a2 = s2 / sw;
        var = fmaxf(a2 - a1 * a1, 0.0f) * (4.0f / Mp.z);
    }
    reinterpret_cast<float*>(T.e)[4 * p + 3] = var;
    reinterpret_cast<float*>(T.frame)[4 * p + 3] = var;
}

// SVGF's prefilter of one iteration: per non-background pixel the 3x3 Gaussian (1/4, 1/2, 1/4)^2 of the variance (e[src].w) over its
// immediate non-background neighbours, renormalised, into gv
__global__ void __launch_bounds__(256) k_temporal_prefilter(const __grid_constant__ TemporalPassParams P, const int src)
{
    const size_t n = (size_t)P.W * P.H;
    const size_t p = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (p >= n) return;
    if (P.guide[p].w != P.guide[p].w) return;
    const int x = (int)(p % (size_t)P.W), y = (int)(p / (size_t)P.W);
    float gw = 0.0f, gv = 0.0f;
    for (int j = -1; j <= 1; j++)
    {
        for (int i = -1; i <= 1; i++)
        {
            const int qx = x + i, qy = y + j;
            if (qx < 0 || qy < 0 || qx >= P.W || qy >= P.H) continue;
            const size_t q = (size_t)qy * P.W + qx;
            if (P.guide[q].w != P.guide[q].w) continue;
            const float k = (i == 0 ? 0.5f : 0.25f) * (j == 0 ? 0.5f : 0.25f);
            gw = gw + k; gv = gv + k * P.e[src][q].w;
        }
    }
    P.gv[p] = gv / gw;
}

// The reprojection, the variance and `iterations` filter passes on `stream`.  The caller has checked the arguments and computed the
// constants; Pp.e / guide / out / W / H / invN / invZ / hist / sigmaL are set for the passes.
inline cudaError_t temporal_launch(const TemporalParams& T, const DevParams& P, const TemporalPassParams& Pp, const DenoisePass* passes,
                                   int iterations, cudaStream_t stream)
{
    const size_t n = (size_t)T.W * T.H;
    RT_LAUNCH((unsigned)((n + 255) / 256), 256, 0, stream, k_temporal_reproject, T, P);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    RT_LAUNCH((unsigned)((n + 255) / 256), 256, 0, stream, k_temporal_variance, T);
    e = cudaGetLastError();
    for (int k = 0; k < iterations && e == cudaSuccess; k++)
    {
#ifndef RT_TEMPORAL_LATTICE_PREFILTER
        RT_LAUNCH((unsigned)((n + 255) / 256), 256, 0, stream, k_temporal_prefilter, Pp, passes[k].src);
        e = cudaGetLastError();
        if (e != cudaSuccess) break;
#endif
        e = denoise_passes(k_temporal_pass, Pp, passes + k, 1, stream);
    }
    return e;
}

} // namespace rtd
