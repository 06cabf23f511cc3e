/* rt_oracle_pixel_stats.cpp — the oracle's per-pixel traversal counters ("PixelStats", include/rt_b200.h), built around the oracle
 * (oracle/rt_oracle.cpp) rather than inside it.  Test infrastructure: ray_tracing_b200/build.py compiles THIS file into
 * oracle/liboracle.so, so the library exports the oracle's C-ABI plus rtReadbackPixelStats / rtDisplayPixelStats and the test hook
 * orRenderPixelStats.
 *
 * The oracle's source is included unchanged.  Five of its entry points are renamed on the way in (orBase_*) and wrapped below, so that
 * the counting option, the resets and the resize reach the per-pixel image; everything they did before they still do.  A counting
 * dispatch first runs the oracle's own dispatch (images, RtStats), then traces every pixel that dispatch covered once more with the
 * same uniforms and adds what that trace counted (the Shader's nRays / nBox / nTri / nSphere) into the pixel's record: a pixel's
 * trace depends on nothing but the uniforms and buffers (RayCommon.hlsl:545-582), so the second trace counts exactly what the first
 * one did.  The oracle has no sphere accelerator: sphereBoxTests stays 0 and sphereTests counts every sphere of the linear scan. */
// (g++ warns when a struct in an included file has a member of an anonymous-namespace type; here that file is the whole oracle,
// compiled as this one translation unit, as it is on its own)
#pragma GCC diagnostic ignored "-Wsubobject-linkage"
#define rtDispatch   orBase_rtDispatch
#define rtSetOption  orBase_rtSetOption
#define rtResize     orBase_rtResize
#define rtResetStats orBase_rtResetStats
#define rtDestroy    orBase_rtDestroy
#include "../../oracle/rt_oracle.cpp"
#undef rtDispatch
#undef rtSetOption
#undef rtResize
#undef rtResetStats
#undef rtDestroy

#include <algorithm>
#include <cmath>
#include <map>
#include <mutex>

namespace {

struct PixelState
{
    int countStats = 0;                   // option "countStats"
    std::vector<RtPixelStats> image;      // W*H, [y][x]; empty until the first counting dispatch
};

std::mutex g_pixMutex;
std::map<const RtContext*, PixelState> g_pix;

PixelState& pixelState(const RtContext* c)
{
    std::lock_guard<std::mutex> lock(g_pixMutex);
    return g_pix[c];                      // std::map: references stay valid while other contexts come and go
}

// One RayTrace of each listed pixel (n pairs of global coordinates) with the context's current uniforms; out[i] = what it counted.
// Multi-threaded like the oracle's dispatch; touches neither the images nor RtStats.
void tracePixelCounts(RtContext* c, const int* xy, size_t n, RtPixelStats* out)
{
    std::atomic<size_t> next(0);
    std::vector<std::thread> pool;
    for (int t = 0; t < c->threads; t++)
    {
        pool.emplace_back([&]() {
            Shader s = c->sh;
            bind_buffers(c, s);
            const uint* R = s.Resolution;
            for (;;)
            {
                const size_t i0 = next.fetch_add(64);
                if (i0 >= n) break;
                for (size_t i = i0; i < n && i < i0 + 64; i++)
                {
                    const uint x = (uint)xy[2 * i], y = (uint)xy[2 * i + 1];
                    const float2 uv = mk2((float)x / ((float)R[0] - 1.0f), (float)y / ((float)R[1] - 1.0f));   // RayCompute.compute:15
                    const unsigned long long rays = s.nRays, box = s.nBox, tri = s.nTri, sph = s.nSphere;
                    s.RayTrace(uv, R);
                    RtPixelStats& o = out[i];
                    o.rays = (uint32_t)(s.nRays - rays); o.boxTests = (uint32_t)(s.nBox - box); o.triTests = (uint32_t)(s.nTri - tri);
                    o.sphereTests = (uint32_t)(s.nSphere - sph); o.sphereBoxTests = 0;
                }
            }
        });
    }
    for (auto& th : pool) th.join();
}

} // namespace

extern "C" {

int rtDestroy(RtContext* c)
{
    { std::lock_guard<std::mutex> lock(g_pixMutex); g_pix.erase(c); }
    return orBase_rtDestroy(c);
}

int rtSetOption(RtContext* c, const char* name, int value)
{
    const int rc = orBase_rtSetOption(c, name, value);
    if (rc == RT_OK && std::string(name) == "countStats") pixelState(c).countStats = value != 0;
    return rc;
}

int rtResize(RtContext* c, int w, int h)
{
    const bool newSize = c && (w != c->width || h != c->height);
    const int rc = orBase_rtResize(c, w, h);
    if (rc == RT_OK && newSize)
    {
        PixelState& ps = pixelState(c);
        if (!ps.image.empty()) ps.image.assign((size_t)w * h, RtPixelStats());      // follows the image size, zero-filled
    }
    return rc;
}

int rtResetStats(RtContext* c)
{
    const int rc = orBase_rtResetStats(c);
    if (rc == RT_OK)
    {
        PixelState& ps = pixelState(c);
        std::fill(ps.image.begin(), ps.image.end(), RtPixelStats());
    }
    return rc;
}

int rtDispatch(RtContext* c, int kernelIndex, int gx, int gy, int gz)
{
    const int rc = orBase_rtDispatch(c, kernelIndex, gx, gy, gz);
    if (rc != RT_OK || kernelIndex != RT_KERNEL_RAYTRACE) return rc;
    PixelState& ps = pixelState(c);
    if (!ps.countStats) return rc;
    // the pixels the dispatch traced: x < min(W, 8 gx), y < min(H, 8 gy), in this context's row bands (rtDispatch of rt_oracle.cpp)
    const uint W = c->sh.Resolution[0], H = c->sh.Resolution[1];
    const uint limX = gz == 0 ? 0u : ((uint)gx * 8u < W ? (uint)gx * 8u : W), limY = gz == 0 ? 0u : ((uint)gy * 8u < H ? (uint)gy * 8u : H);
    if (ps.image.empty()) ps.image.assign((size_t)W * H, RtPixelStats());
    std::vector<int> xy;
    for (uint y = 0; y < limY; y++)
    {
        if ((int)((y / (uint)c->bandRows) % (uint)c->tileWorld) != c->tileRank) continue;
        for (uint x = 0; x < limX; x++) { xy.push_back((int)x); xy.push_back((int)y); }
    }
    std::vector<RtPixelStats> counts(xy.size() / 2);
    tracePixelCounts(c, xy.data(), counts.size(), counts.data());
    for (size_t i = 0; i < counts.size(); i++)
    {
        RtPixelStats& d = ps.image[(size_t)xy[2 * i + 1] * W + (size_t)xy[2 * i]];      // uint32 sums: wrap like the product's
        d.rays += counts[i].rays; d.boxTests += counts[i].boxTests; d.triTests += counts[i].triTests;
        d.sphereTests += counts[i].sphereTests; d.sphereBoxTests += counts[i].sphereBoxTests;
    }
    return rc;
}

int rtReadbackPixelStats(RtContext* c, RtPixelStats* dst, size_t bytes)
{
    if (!c || !dst) return fail(c, RT_E_INVALID, "rtReadbackPixelStats: bad argument");
    const PixelState& ps = pixelState(c);
    if (ps.image.empty()) return fail(c, RT_E_STATE, "rtReadbackPixelStats: no counting dispatch yet");
    if (bytes != ps.image.size() * sizeof(RtPixelStats)) return fail(c, RT_E_INVALID, "rtReadbackPixelStats: bytes must equal W*H*20");
    memcpy(dst, ps.image.data(), bytes);
    return RT_OK;
}

// The heat-map encode of include/rt_b200.h, one binary32 operation at a time (-ffp-contract=off)
int rtDisplayPixelStats(RtContext* c, int visMode, float debugVisScale, uint8_t* dst, size_t bytes)
{
    if (!c || !dst) return fail(c, RT_E_INVALID, "rtDisplayPixelStats: bad argument");
    if (visMode < 1 || visMode > 4) return fail(c, RT_E_INVALID, "rtDisplayPixelStats: visMode must be 1..4");
    if (!std::isfinite(debugVisScale) || !(debugVisScale > 0.0f)) return fail(c, RT_E_INVALID, "rtDisplayPixelStats: debugVisScale must be finite and > 0");
    const PixelState& ps = pixelState(c);
    if (ps.image.empty()) return fail(c, RT_E_STATE, "rtDisplayPixelStats: no counting dispatch yet");
    if (bytes != ps.image.size() * 4) return fail(c, RT_E_INVALID, "rtDisplayPixelStats: bytes must equal W*H*4");
    for (size_t i = 0; i < ps.image.size(); i++)
    {
        const RtPixelStats& s = ps.image[i];
        uint8_t* o = dst + 4 * i;
        o[3] = 255;
        if (s.rays == 0) { o[0] = o[1] = o[2] = 0; continue; }
        const uint32_t count = visMode == 1 ? s.boxTests : visMode == 2 ? s.triTests : s.sphereTests + s.sphereBoxTests;
        const float v = visMode == 4 ? (float)s.rays : (float)count / (float)s.rays;
        const float t = v / debugVisScale;
        if (t > 1.0f) { o[0] = 255; o[1] = o[2] = 0; continue; }
        o[0] = o[1] = o[2] = (uint8_t)orc::f2uint_rz(t * 255.0f + 0.5f);
    }
    return RT_OK;
}

/* Test hook beside orRenderPixels: out = n RtPixelStats, the counts of one RayTrace of each listed pixel (xy = n pairs of global
 * coordinates) with the context's current uniforms — what one counting dispatch adds to that pixel's record.  Touches neither the
 * images, nor RtStats, nor PixelStats. */
int orRenderPixelStats(RtContext* c, const int* xy, int n, RtPixelStats* out)
{
    if (!c || !xy || !out || n < 0) return fail(c, RT_E_INVALID, "orRenderPixelStats: bad argument");
    if (c->sh.modelCount > (int)c->models.size()) return fail(c, RT_E_STATE, "orRenderPixelStats: modelCount exceeds ModelInfo length");
    { std::string why; if (bvhTooDeepOrBroken(c, why)) return fail(c, RT_E_STATE, "orRenderPixelStats: " + why); }
    tracePixelCounts(c, xy, (size_t)n, out);
    return RT_OK;
}

} // extern "C"
