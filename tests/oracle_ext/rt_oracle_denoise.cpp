/* rt_oracle_denoise.cpp — rtDenoise / rtDisplayDenoised (include/rt_b200.h) for the oracle, built around it rather than inside it.
 * Test infrastructure: ray_tracing_b200/build.py compiles THIS file into oracle/liboracle.so.  It includes the oracle with the feature
 * images (rt_oracle_features.cpp, which includes the rest) and adds the a-trous filter, restated from the header's statement with orc::
 * arithmetic, one pixel and one tap at a time in the stated order.
 *
 * orDenoiseImages is the filter on caller-supplied arrays, so that synthetic images (denormals, NaN, overflowing demodulation, ...) can
 * be compared with the product, whose input images the tests write through rtGetDevicePointer.
 *
 * Three entry points the feature layer already wraps have to reach "DenoisedRender" as well: rtDestroy, rtResize (a new size zeroes it)
 * and rtReadback (one new name).  As that layer does with the layers below it, the three wrappers it defines are declared here first
 * with an assembler name of their own (orFeat_*), and the wrappers at the end of this file get the plain symbols the ABI exports.  GCC
 * warns that the feature layer's own labels are ignored (-Wpragmas); that is the point, so the warning is silenced around the include. */
struct RtContext;
extern "C" {
int orFeatures_rtDestroy(RtContext* c) __asm__("orFeat_rtDestroy");
int orFeatures_rtResize(RtContext* c, int w, int h) __asm__("orFeat_rtResize");
int orFeatures_rtReadback(RtContext* c, const char* tex, float* dst, unsigned long bytes) __asm__("orFeat_rtReadback");
}
#pragma GCC diagnostic push
#pragma GCC diagnostic ignored "-Wpragmas"
#include "rt_oracle_features.cpp"
#pragma GCC diagnostic pop

namespace {

std::mutex g_denMutex;
std::map<const RtContext*, std::vector<float>> g_denoised;      // W*H float4 "DenoisedRender"; absent until the first rtDenoise

bool finite1(float v) { return fabsf(v) < orc::rt_inf(); }

struct DenoiseConstants { float cK[RT_DENOISE_MAX_ITERATIONS], invN, invZ; };

// The argument checks and the host constants of include/rt_b200.h
int denoiseConstants(int useAccumulated, int iterations, const float sigma[3], DenoiseConstants& k)
{
    if (useAccumulated != 0 && useAccumulated != 1) return RT_E_INVALID;
    if (iterations < 1 || iterations > RT_DENOISE_MAX_ITERATIONS) return RT_E_INVALID;
    for (int i = 0; i < 3; i++)
        if (!(sigma[i] > 0.0f) || !finite1(sigma[i])) return RT_E_INVALID;
    const float invC = 1.0f / (sigma[0] * sigma[0]);
    float fourK = 1.0f;
    for (int i = 0; i < iterations; i++) { k.cK[i] = invC * fourK; fourK = fourK * 4.0f; }
    k.invN = 1.0f / (sigma[1] * sigma[1]);
    k.invZ = 1.0f / sigma[2];
    if (!finite1(k.cK[iterations - 1]) || !finite1(k.invN) || !finite1(k.invZ)) return RT_E_INVALID;
    return RT_OK;
}

void denoise(int W, int H, int useAccumulated, const float* colour, const float* albedo, const float* normal, const RtPixelFeatures* feats,
             int iterations, const DenoiseConstants& K, float* out)
{
    const size_t n = (size_t)W * H;
    std::vector<float3> e(n), m(n), nrm(n);
    std::vector<float> z(n);
    std::vector<char> bg(n);
    for (size_t p = 0; p < n; p++)
    {
        float3 c, a;
        bool b;
        if (useAccumulated)
        {
            const float* A = colour + 4 * p; const float* L = albedo + 4 * p; const float* N = normal + 4 * p;
            b = A[3] == 0.0f || L[3] == 0.0f;
            c = A[3] == 0.0f ? mk3(0.0f) : mk3(A[0] / A[3], A[1] / A[3], A[2] / A[3]);
            a = mk3(L[0] / L[3], L[1] / L[3], L[2] / L[3]);
            nrm[p] = mk3(N[0] / L[3], N[1] / L[3], N[2] / L[3]);
            z[p] = N[3] / L[3];
        }
        else
        {
            const RtPixelFeatures& f = feats[p];
            b = f.object == -1;
            c = mk3(colour + 4 * p);
            a = mk3(f.albedo);
            nrm[p] = mk3(f.normal);
            z[p] = f.dst;
        }
        m[p] = mk3(orc::max(a.x, 0.00390625f), orc::max(a.y, 0.00390625f), orc::max(a.z, 0.00390625f));
        e[p] = mk3(c.x / m[p].x, c.y / m[p].y, c.z / m[p].z);
        const float vals[13] = {c.x, c.y, c.z, a.x, a.y, a.z, nrm[p].x, nrm[p].y, nrm[p].z, z[p], e[p].x, e[p].y, e[p].z};
        for (float v : vals) b = b || !finite1(v);
        bg[p] = b;
        if (b) { out[4 * p] = c.x; out[4 * p + 1] = c.y; out[4 * p + 2] = c.z; out[4 * p + 3] = 1.0f; }
    }
    static const float h[5] = {0.0625f, 0.25f, 0.375f, 0.25f, 0.0625f};
    for (int k = 0; k < iterations; k++)
    {
        const int s = 1 << k;
        const float rd[3] = {0.0f, 1.0f / (float)s, 1.0f / (float)(2 * s)};
        std::vector<float3> next(e);
        for (int y = 0; y < H; y++)
            for (int x = 0; x < W; x++)
            {
                const size_t p = (size_t)y * W + x;
                if (bg[p]) continue;
                const float rz = K.invZ / z[p];
                float sw = 0.0f, sr = 0.0f, sg = 0.0f, sb = 0.0f;
                for (int j = -2; j <= 2; j++)
                    for (int i = -2; i <= 2; i++)
                    {
                        const long long qx = x + (long long)s * i, qy = y + (long long)s * j;
                        if (qx < 0 || qy < 0 || qx >= W || qy >= H) continue;
                        const size_t q = (size_t)qy * W + (size_t)qx;
                        if (bg[q]) continue;
                        float w;
                        if (i == 0 && j == 0) w = 0.140625f;
                        else
                        {
                            const float3 de = e[p] - e[q], dn = nrm[p] - nrm[q];
                            const int d = std::max(std::abs(i), std::abs(j));
                            const float t = ((z[p] - z[q]) * rz) * rd[d];
                            const float D = (((de.x * de.x + de.y * de.y) + de.z * de.z) * K.cK[k] + ((dn.x * dn.x + dn.y * dn.y) + dn.z * dn.z) * K.invN) + t * t;
                            w = D <= 103.972076416015625f ? (h[i + 2] * h[j + 2]) * orc::exp(-D) : 0.0f;      // a NaN D weighs 0
                            if (w == 0.0f) continue;
                        }
                        sw = sw + w;
                        sr = sr + w * e[q].x; sg = sg + w * e[q].y; sb = sb + w * e[q].z;
                    }
                next[p] = mk3(sr / sw, sg / sw, sb / sw);
            }
        e.swap(next);
    }
    for (size_t p = 0; p < n; p++)
        if (!bg[p]) { out[4 * p] = e[p].x * m[p].x; out[4 * p + 1] = e[p].y * m[p].y; out[4 * p + 2] = e[p].z * m[p].z; out[4 * p + 3] = 1.0f; }
}

} // namespace

extern "C" {

/* The filter on caller arrays: colour = W*H float4 (AccumulatedRender or FrameRender); useAccumulated = 1: albedo, normalOrFeatures =
 * AccumulatedAlbedo, AccumulatedNormal (float4 each); 0: albedo unused, normalOrFeatures = W*H RtPixelFeatures.  sigma = (colour,
 * normal, depth).  out = W*H float4.  RT_E_INVALID for the arguments rtDenoise refuses. */
int orDenoiseImages(int W, int H, int useAccumulated, const float* colour, const float* albedo, const void* normalOrFeatures, int iterations,
                    const float sigma[3], float* out)
{
    if (W <= 0 || H <= 0 || !colour || !normalOrFeatures || !out || !sigma || (useAccumulated == 1 && !albedo)) return RT_E_INVALID;
    DenoiseConstants K;
    const int rc = denoiseConstants(useAccumulated, iterations, sigma, K);
    if (rc != RT_OK) return rc;
    denoise(W, H, useAccumulated, colour, albedo, (const float*)normalOrFeatures, (const RtPixelFeatures*)normalOrFeatures, iterations, K, out);
    return RT_OK;
}

int rtDenoise(RtContext* c, int useAccumulated, int iterations, float sigmaColour, float sigmaNormal, float sigmaDepth)
{
    if (!c) return RT_E_INVALID;
    const float sigma[3] = {sigmaColour, sigmaNormal, sigmaDepth};
    DenoiseConstants K;
    if (denoiseConstants(useAccumulated, iterations, sigma, K) != RT_OK) return fail(c, RT_E_INVALID, "rtDenoise: bad argument");
    int rc = cameraImage(c, "rtDenoise"); if (rc != RT_OK) return rc;
    const FeatureState& fs = featureState(c);
    if (fs.frame.empty()) return fail(c, RT_E_STATE, "rtDenoise: no rtDispatchFeatures yet");
    if (c->tileWorld > 1) return fail(c, RT_E_STATE, "rtDenoise: the images of a context with rtSetTile world > 1 hold its own bands only");
    std::vector<float> out((size_t)c->width * c->height * 4);
    denoise(c->width, c->height, useAccumulated, useAccumulated ? c->accum.data() : c->frame.data(), fs.albedo.data(), fs.normal.data(),
            fs.frame.data(), iterations, K, out.data());
    std::lock_guard<std::mutex> lock(g_denMutex);
    g_denoised[c].swap(out);
    return RT_OK;
}

int rtDisplayDenoised(RtContext* c, uint8_t* dst, size_t bytes)
{
    if (!c || !dst) return fail(c, RT_E_INVALID, "rtDisplayDenoised: bad argument");
    std::lock_guard<std::mutex> lock(g_denMutex);
    auto it = g_denoised.find(c);
    if (it == g_denoised.end()) return fail(c, RT_E_STATE, "rtDisplayDenoised: no rtDenoise yet");
    if (bytes != it->second.size()) return fail(c, RT_E_INVALID, "rtDisplayDenoised: bytes must equal W*H*4");
    for (size_t i = 0; i < bytes; i++) dst[i] = (uint8_t)DisplayEncode(it->second[i] / 1.0f);
    return RT_OK;
}

/* ---- the three wrapped entry points: defined under a name of their own, exported under the ABI's ------------------------------------ */
int orDenoise_rtDestroy(RtContext* c) __asm__("rtDestroy");
int orDenoise_rtResize(RtContext* c, int w, int h) __asm__("rtResize");
int orDenoise_rtReadback(RtContext* c, const char* tex, float* dst, size_t bytes) __asm__("rtReadback");

int orDenoise_rtDestroy(RtContext* c)
{
    { std::lock_guard<std::mutex> lock(g_denMutex); g_denoised.erase(c); }
    return orFeatures_rtDestroy(c);
}

int orDenoise_rtResize(RtContext* c, int w, int h)
{
    const bool newSize = c && (w != c->width || h != c->height);
    const int rc = orFeatures_rtResize(c, w, h);
    if (rc == RT_OK && newSize)
    {
        std::lock_guard<std::mutex> lock(g_denMutex);
        auto it = g_denoised.find(c);
        if (it != g_denoised.end()) it->second.assign((size_t)w * h * 4, 0.0f);
    }
    return rc;
}

int orDenoise_rtReadback(RtContext* c, const char* tex, float* dst, size_t bytes)
{
    if (!(c && tex && dst && std::string(tex) == "DenoisedRender")) return orFeatures_rtReadback(c, tex, dst, bytes);
    std::lock_guard<std::mutex> lock(g_denMutex);
    auto it = g_denoised.find(c);
    if (it == g_denoised.end()) return fail(c, RT_E_STATE, "rtReadback: no rtDenoise yet");
    if (bytes != it->second.size() * 4) return fail(c, RT_E_INVALID, "rtReadback: bytes must equal W*H*16");
    memcpy(dst, it->second.data(), bytes);
    return RT_OK;
}

} // extern "C"
