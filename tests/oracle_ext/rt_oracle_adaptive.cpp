/* rt_oracle_adaptive.cpp — rtDispatchAdaptive and rtDisplayMean (include/rt_b200.h) for the oracle, built around it rather than inside
 * it.  Test infrastructure: ray_tracing_b200/build.py compiles THIS file into oracle/liboracle.so.  It includes the oracle with the
 * temporal denoiser (rt_oracle_temporal.cpp, which includes the rest) and restates the call from the header's statement: the selection
 * in binary32, one operation at a time in the stated order (-ffp-contract=off), then for each active pixel the reference kernel
 * Shader::Kernel_RayTrace (with the per-pixel counts of the PixelStats layer when "countStats" is on) and the moments update.
 *
 * Four entry points the layers below already wrap have to reach the moments as well: rtDestroy, rtResize (a new size zeroes them),
 * rtDispatch (ResetAccumulated zeroes their region) and rtReadback (one new name).  As those layers do with the layers below them, the
 * wrappers they define are declared here first with an assembler name of their own (orTmp_*, orFeat_rtDispatch), and the wrappers at
 * the end of this file get the plain symbols the ABI exports; the warning about the lower layers' own labels is silenced around the
 * include. */
struct RtContext;
extern "C" {
int orTemporal_rtDestroy(RtContext* c) __asm__("orTmp_rtDestroy");
int orTemporal_rtResize(RtContext* c, int w, int h) __asm__("orTmp_rtResize");
int orTemporal_rtReadback(RtContext* c, const char* tex, float* dst, unsigned long bytes) __asm__("orTmp_rtReadback");
int orFeatures_rtDispatch(RtContext* c, int kernelIndex, int gx, int gy, int gz) __asm__("orFeat_rtDispatch");
}
#pragma GCC diagnostic push
#pragma GCC diagnostic ignored "-Wpragmas"
#include "rt_oracle_temporal.cpp"
#pragma GCC diagnostic pop

namespace {

std::mutex g_adaMutex;
std::map<const RtContext*, std::vector<float>> g_moments;      // "AdaptiveMoments", W*H float4; absent until the first traced call

// include/rt_b200.h, rtDispatchAdaptive: the selection criterion, one binary32 operation each in the order written
bool adaptiveActive(const float* m, float threshold, float minFrames, float maxFrames)
{
    const float n = m[2];
    const float mu = m[0] / n;
    const float v = orc::max(m[1] / n - mu * mu, 0.0f);
    return n < minFrames || (n < maxFrames && v > ((threshold * threshold) * n) * (mu * mu + RT_ADAPTIVE_EPSILON));
}

} // namespace

extern "C" {

int rtDispatchAdaptive(RtContext* c, int gx, int gy, int gz, float threshold, int minFrames, int maxFrames, int64_t* activePixels)
{
    if (!c || gx < 0 || gy < 0 || gz < 0) return fail(c, RT_E_INVALID, "rtDispatchAdaptive: bad argument");
    if (!std::isfinite(threshold) || threshold < 0.0f || !std::isfinite(threshold * threshold))
        return fail(c, RT_E_INVALID, "rtDispatchAdaptive: threshold must be finite and >= 0, with a finite square");
    if (minFrames < 2) return fail(c, RT_E_INVALID, "rtDispatchAdaptive: minFrames must be at least 2");
    if (maxFrames < minFrames || maxFrames > RT_ADAPTIVE_MAX_FRAMES) return fail(c, RT_E_INVALID, "rtDispatchAdaptive: maxFrames out of range");
    if (c->width == 0) return fail(c, RT_E_STATE, "rtDispatchAdaptive: rtResize has not been called");
    const uint W = c->sh.Resolution[0], H = c->sh.Resolution[1];
    if ((int)W != c->width || (int)H != c->height) return fail(c, RT_E_STATE, "rtDispatchAdaptive: Resolution does not match the textures");
    if (!c->sh.accumulate) return fail(c, RT_E_STATE, "rtDispatchAdaptive: needs accumulate = 1");
    const uint limX = gz == 0 ? 0u : ((uint)gx * 8u < W ? (uint)gx * 8u : W), limY = gz == 0 ? 0u : ((uint)gy * 8u < H ? (uint)gy * 8u : H);
    if (activePixels) *activePixels = 0;
    if (limX == 0 || limY == 0) return RT_OK;
    if (c->sh.modelCount > (int)c->models.size()) return fail(c, RT_E_STATE, "rtDispatchAdaptive: modelCount exceeds ModelInfo length");
    { std::string why; if (bvhTooDeepOrBroken(c, why)) return fail(c, RT_E_STATE, "rtDispatchAdaptive: " + why); }

    std::lock_guard<std::mutex> lock(g_adaMutex);
    auto it = g_moments.find(c);
    const std::vector<float> zero(4, 0.0f);
    std::vector<int> xy;
    for (uint y = 0; y < limY; y++)
    {
        if ((int)((y / (uint)c->bandRows) % (uint)c->tileWorld) != c->tileRank) continue;
        for (uint x = 0; x < limX; x++)
        {
            const float* m = it == g_moments.end() ? zero.data() : &it->second[((size_t)y * W + x) * 4];
            if (adaptiveActive(m, threshold, (float)minFrames, (float)maxFrames)) { xy.push_back((int)x); xy.push_back((int)y); }
        }
    }
    const size_t n = xy.size() / 2;
    if (activePixels) *activePixels = (int64_t)n;
    if (n == 0) return RT_OK;
    std::vector<float>& mom = g_moments[c];
    if (mom.empty()) mom.assign((size_t)W * H * 4, 0.0f);

    // the reference kernel per active pixel, with the counters of the oracle's own dispatch
    auto t0 = std::chrono::steady_clock::now();
    std::atomic<size_t> next(0);
    std::vector<Shader> shaders(c->threads, c->sh);
    std::vector<std::thread> pool;
    for (int t = 0; t < c->threads; t++)
    {
        pool.emplace_back([&, t]() {
            Shader& s = shaders[t];
            bind_buffers(c, s);
            for (size_t i; (i = next.fetch_add(1)) < n;)
            {
                const uint x = (uint)xy[2 * i], y = (uint)xy[2 * i + 1];
                s.Kernel_RayTrace(x, y, c->frame.data(), c->accum.data());
                const size_t o = ((size_t)y * W + x) * 4;
                const float r = c->frame[o], g = c->frame[o + 1], b = c->frame[o + 2];
                const float l = (0.2126f * r + 0.7152f * g) + 0.0722f * b;
                mom[o] += l; mom[o + 1] += l * l; mom[o + 2] += 1.0f;
            }
        });
    }
    for (auto& th : pool) th.join();
    for (auto& s : shaders) { c->stats.rays += s.nRays; c->stats.boxTests += s.nBox; c->stats.triTests += s.nTri; c->stats.sphereTests += s.nSphere; }
    c->stats.dispatches++;
    c->stats.kernelMs += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();

    PixelState& ps = pixelState(c);
    if (ps.countStats)
    {
        if (ps.image.empty()) ps.image.assign((size_t)W * H, RtPixelStats());
        std::vector<RtPixelStats> counts(n);
        tracePixelCounts(c, xy.data(), n, counts.data());
        for (size_t i = 0; i < n; i++)
        {
            RtPixelStats& d = ps.image[(size_t)xy[2 * i + 1] * W + (size_t)xy[2 * i]];
            d.rays += counts[i].rays; d.boxTests += counts[i].boxTests; d.triTests += counts[i].triTests;
            d.sphereTests += counts[i].sphereTests; d.sphereBoxTests += counts[i].sphereBoxTests;
        }
    }
    return RT_OK;
}

int rtDisplayMean(RtContext* c, uint8_t* dst, size_t bytes)
{
    if (!c || !dst) return fail(c, RT_E_INVALID, "rtDisplayMean: bad argument");
    if (c->accum.empty()) return fail(c, RT_E_STATE, "rtDisplayMean: rtResize has not been called");
    if (bytes != c->accum.size()) return fail(c, RT_E_INVALID, "rtDisplayMean: bytes must equal W*H*4");
    for (size_t p = 0; p < bytes / 4; p++)
    {
        const float* a = &c->accum[p * 4];
        uint8_t* o = dst + 4 * p;
        if (a[3] == 0.0f) { o[0] = o[1] = o[2] = 0; o[3] = 255; continue; }
        for (int k = 0; k < 4; k++) o[k] = (uint8_t)DisplayEncode(a[k] / a[3]);
    }
    return RT_OK;
}

/* ---- the four wrapped entry points: defined under a name of their own, exported under the ABI's ------------------------------------ */
int orAdaptive_rtDestroy(RtContext* c) __asm__("rtDestroy");
int orAdaptive_rtResize(RtContext* c, int w, int h) __asm__("rtResize");
int orAdaptive_rtDispatch(RtContext* c, int kernelIndex, int gx, int gy, int gz) __asm__("rtDispatch");
int orAdaptive_rtReadback(RtContext* c, const char* tex, float* dst, size_t bytes) __asm__("rtReadback");

int orAdaptive_rtDestroy(RtContext* c)
{
    { std::lock_guard<std::mutex> lock(g_adaMutex); g_moments.erase(c); }
    return orTemporal_rtDestroy(c);
}

int orAdaptive_rtResize(RtContext* c, int w, int h)
{
    const bool newSize = c && (w != c->width || h != c->height);
    const int rc = orTemporal_rtResize(c, w, h);
    if (rc == RT_OK && newSize)
    {
        std::lock_guard<std::mutex> lock(g_adaMutex);
        auto it = g_moments.find(c);
        if (it != g_moments.end()) it->second.assign((size_t)w * h * 4, 0.0f);
    }
    return rc;
}

int orAdaptive_rtDispatch(RtContext* c, int kernelIndex, int gx, int gy, int gz)
{
    const int rc = orFeatures_rtDispatch(c, kernelIndex, gx, gy, gz);
    if (rc != RT_OK || kernelIndex != RT_KERNEL_RESET_ACCUMULATED) return rc;
    std::lock_guard<std::mutex> lock(g_adaMutex);
    auto it = g_moments.find(c);
    if (it == g_moments.end()) return rc;
    const uint W = (uint)c->width, H = (uint)c->height;          // ResetAccumulated's region (rtDispatch of rt_oracle.cpp)
    const uint limX = gz == 0 ? 0u : ((uint)gx * 8u < W ? (uint)gx * 8u : W), limY = gz == 0 ? 0u : ((uint)gy * 8u < H ? (uint)gy * 8u : H);
    for (uint y = 0; y < limY; y++) memset(&it->second[((size_t)y * W) * 4], 0, (size_t)limX * 16);
    return rc;
}

int orAdaptive_rtReadback(RtContext* c, const char* tex, float* dst, size_t bytes)
{
    if (!(c && tex && dst && std::string(tex) == "AdaptiveMoments")) return orTemporal_rtReadback(c, tex, dst, bytes);
    std::lock_guard<std::mutex> lock(g_adaMutex);
    auto it = g_moments.find(c);
    if (it == g_moments.end()) return fail(c, RT_E_STATE, "rtReadback: no rtDispatchAdaptive yet");
    if (bytes != it->second.size() * 4) return fail(c, RT_E_INVALID, "rtReadback: bytes must equal W*H*16");
    memcpy(dst, it->second.data(), bytes);
    return RT_OK;
}

} // extern "C"
