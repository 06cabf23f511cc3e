/* rt_oracle_features.cpp — rtDispatchFeatures / rtCameraRays / rtCameraRaysDevice (include/rt_b200.h) for the oracle, built around it
 * rather than inside it.  Test infrastructure: ray_tracing_b200/build.py compiles THIS file into oracle/liboracle.so.  It includes the
 * oracle with rtTracePaths (rt_oracle_paths.cpp, which includes the rest) and adds the feature images.
 *
 * A pixel's feature ray is orCameraSample for the pixel's own seed (rt_oracle_paths.cpp: RayTrace, HL:545-576, up to the ray it hands
 * to Trace).  Its hit is Shader::CalculateRayCollision (whose counters RtStats gets), the winner's kind and index come from
 * tracedWinner (rt_oracle_trace_rays.cpp), the albedo from Shader::GetMaterialColour.
 *
 * Four entry points the layers below already define have to reach the feature images as well: rtDestroy, rtResize (a new size zeroes
 * them), rtDispatch (ResetAccumulated zeroes the two accumulators) and rtReadback (three new names).  Those layers rename what THEY
 * wrap with macros that they also undefine, so a further macro cannot rename their definitions.  Instead the four names are declared
 * here first with an assembler name of their own (orInner_*): the definitions that follow get that symbol, and the wrappers at the
 * end of this file are given the plain symbols the ABI exports. */
struct RtContext;
extern "C" {
int rtDestroy(RtContext* c) __asm__("orInner_rtDestroy");
int rtResize(RtContext* c, int w, int h) __asm__("orInner_rtResize");
int rtDispatch(RtContext* c, int kernelIndex, int gx, int gy, int gz) __asm__("orInner_rtDispatch");
int rtReadback(RtContext* c, const char* tex, float* dst, unsigned long bytes) __asm__("orInner_rtReadback");
}
#include "rt_oracle_paths.cpp"

static_assert(sizeof(unsigned long) == sizeof(size_t), "the declaration of rtReadback above");

namespace {

struct FeatureState
{
    std::vector<RtPixelFeatures> frame;       // W*H, [y][x]; empty until the first rtDispatchFeatures
    std::vector<float> albedo, normal;        // W*H float4 each
};

std::mutex g_featMutex;
std::map<const RtContext*, FeatureState> g_feat;

FeatureState& featureState(const RtContext* c)
{
    std::lock_guard<std::mutex> lock(g_featMutex);
    return g_feat[c];
}

int cameraImage(RtContext* c, const char* what)
{
    if (c->width == 0) return fail(c, RT_E_STATE, std::string(what) + ": rtResize has not been called");
    if ((int)c->sh.Resolution[0] != c->width || (int)c->sh.Resolution[1] != c->height) return fail(c, RT_E_STATE, std::string(what) + ": Resolution does not match the textures");
    if (c->width > 65535 || c->height > 65535) return fail(c, RT_E_STATE, std::string(what) + ": a resolution above 65535 is not supported");
    return RT_OK;
}

// The record of one pixel (include/rt_b200.h); counts into s, the winner's loop into w
RtPixelFeatures pixelFeatures(RtContext* c, Shader& s, Shader& w, int x, int y)
{
    RtPathRay cam;
    orCameraSample(c, x, y, nullptr, &cam);
    Shader::Ray ray;
    memset(&ray, 0, sizeof(ray));
    ray.pos = mk3(cam.origin); ray.dir = mk3(cam.dir); ray.invDir = 1.0f / ray.dir;
    const Shader::ModelHitInfo hit = s.CalculateRayCollision(ray, false);                 // HL:487
    int kind, index;
    tracedWinner(w, ray.pos, ray.dir, false, kind, index);
    RtPixelFeatures f;
    memset(&f, 0, sizeof(f));
    f.dst = hit.dst; f.object = -1;
    if (kind == RT_HIT_NONE) return f;
    const float3 albedo = hit.material.flag == Shader::MATERIAL_GLASS ? mk3(1.0f) : Shader::GetMaterialColour(hit.material, hit.pos, hit.normal, false);
    f.albedo[0] = albedo.x; f.albedo[1] = albedo.y; f.albedo[2] = albedo.z;
    f.normal[0] = hit.normal.x; f.normal[1] = hit.normal.y; f.normal[2] = hit.normal.z;
    f.object = kind == RT_HIT_SPHERE ? -2 - index : index;
    return f;
}

} // namespace

extern "C" {

int rtDispatchFeatures(RtContext* c, int gx, int gy, int gz)
{
    if (!c) return RT_E_INVALID;
    if (gx < 0 || gy < 0 || gz < 0) return fail(c, RT_E_INVALID, "rtDispatchFeatures: bad argument");
    int rc = cameraImage(c, "rtDispatchFeatures"); if (rc != RT_OK) return rc;
    const uint W = c->sh.Resolution[0], H = c->sh.Resolution[1];
    FeatureState& fs = featureState(c);
    if (fs.frame.empty())
    {
        fs.frame.assign((size_t)W * H, RtPixelFeatures());
        fs.albedo.assign((size_t)W * H * 4, 0.0f);
        fs.normal.assign((size_t)W * H * 4, 0.0f);
    }
    const uint limX = gz == 0 ? 0u : ((unsigned long long)gx * 8ull < W ? (uint)gx * 8u : W), limY = gz == 0 ? 0u : ((unsigned long long)gy * 8ull < H ? (uint)gy * 8u : H);
    if (limX == 0 || limY == 0) return RT_OK;
    if ((rc = traceChecks(c, "rtDispatchFeatures", c, c, 1, 0)) != RT_OK) return rc;     // the scene checks of rtDispatch

    std::atomic<uint> nextRow(0);
    std::vector<Shader> shaders(c->threads, c->sh);
    std::vector<std::thread> pool;
    for (int t = 0; t < c->threads; t++)
    {
        pool.emplace_back([&, t]() {
            Shader& s = shaders[t];
            bind_buffers(c, s);
            Shader w = s;                                // the winner's loop counts into a copy that is thrown away
            for (;;)
            {
                const uint y = nextRow.fetch_add(1);
                if (y >= limY) break;
                if ((int)((y / (uint)c->bandRows) % (uint)c->tileWorld) != c->tileRank) continue;
                for (uint x = 0; x < limX; x++)
                {
                    const size_t o = (size_t)y * W + x;
                    const RtPixelFeatures f = pixelFeatures(c, s, w, (int)x, (int)y);
                    fs.frame[o] = f;
                    if (c->sh.accumulate && f.object != -1)
                    {
                        float* a = &fs.albedo[o * 4]; float* n = &fs.normal[o * 4];
                        a[0] += f.albedo[0]; a[1] += f.albedo[1]; a[2] += f.albedo[2]; a[3] += 1.0f;
                        n[0] += f.normal[0]; n[1] += f.normal[1]; n[2] += f.normal[2]; n[3] += f.dst;
                    }
                }
            }
        });
    }
    for (auto& th : pool) th.join();
    for (auto& s : shaders) { c->stats.rays += s.nRays; c->stats.boxTests += s.nBox; c->stats.triTests += s.nTri; c->stats.sphereTests += s.nSphere; }
    return RT_OK;
}

int rtCameraRays(RtContext* c, RtPathRay* rays, size_t bytes)
{
    if (!c) return RT_E_INVALID;
    if (!rays) return fail(c, RT_E_INVALID, "rtCameraRays: rays is NULL");
    const int rc = cameraImage(c, "rtCameraRays"); if (rc != RT_OK) return rc;
    if (bytes != (size_t)c->width * c->height * sizeof(RtPathRay)) return fail(c, RT_E_INVALID, "rtCameraRays: bytes must equal W*H*28");
    for (int y = 0; y < c->height; y++)
        for (int x = 0; x < c->width; x++) orCameraSample(c, x, y, nullptr, rays + (size_t)y * c->width + x);
    return RT_OK;
}

int rtCameraRaysDevice(RtContext* c, void*, size_t) { return c ? fail(c, RT_E_STATE, "oracle: no device memory") : RT_E_INVALID; }

/* Test hook beside orRenderPixels: out = n RtPixelFeatures, the FeatureFrame record of each listed pixel (xy = n pairs of global pixel
 * coordinates) for the context's current uniforms; the feature images are not touched.  Exact, because a pixel's feature ray depends on
 * its own coordinates and seed only.  Multi-threaded; the counts go to RtStats as rtDispatchFeatures's do. */
int orFeaturePixels(RtContext* c, const int* xy, int n, RtPixelFeatures* out)
{
    if (!c) return RT_E_INVALID;
    if (!xy || !out || n < 0) return fail(c, RT_E_INVALID, "orFeaturePixels: bad argument");
    int rc = cameraImage(c, "orFeaturePixels"); if (rc != RT_OK) return rc;
    if ((rc = traceChecks(c, "orFeaturePixels", c, c, 1, 0)) != RT_OK) return rc;
    std::atomic<int> next(0);
    std::vector<Shader> shaders(c->threads, c->sh);
    std::vector<std::thread> pool;
    for (int t = 0; t < c->threads; t++)
    {
        pool.emplace_back([&, t]() {
            Shader& s = shaders[t];
            bind_buffers(c, s);
            Shader w = s;
            for (;;)
            {
                const int i0 = next.fetch_add(64);
                if (i0 >= n) break;
                for (int i = i0; i < n && i < i0 + 64; i++) out[i] = pixelFeatures(c, s, w, xy[2 * i], xy[2 * i + 1]);
            }
        });
    }
    for (auto& th : pool) th.join();
    for (auto& s : shaders) { c->stats.rays += s.nRays; c->stats.boxTests += s.nBox; c->stats.triTests += s.nTri; c->stats.sphereTests += s.nSphere; }
    return RT_OK;
}

/* ---- the four wrapped entry points: defined under a name of their own, exported under the ABI's ------------------------------------ */
int orFeatures_rtDestroy(RtContext* c) __asm__("rtDestroy");
int orFeatures_rtResize(RtContext* c, int w, int h) __asm__("rtResize");
int orFeatures_rtDispatch(RtContext* c, int kernelIndex, int gx, int gy, int gz) __asm__("rtDispatch");
int orFeatures_rtReadback(RtContext* c, const char* tex, float* dst, size_t bytes) __asm__("rtReadback");

int orFeatures_rtDestroy(RtContext* c)
{
    { std::lock_guard<std::mutex> lock(g_featMutex); g_feat.erase(c); }
    return rtDestroy(c);
}

int orFeatures_rtResize(RtContext* c, int w, int h)
{
    const bool newSize = c && (w != c->width || h != c->height);
    const int rc = rtResize(c, w, h);
    if (rc == RT_OK && newSize)
    {
        FeatureState& fs = featureState(c);
        if (!fs.frame.empty())
        {
            fs.frame.assign((size_t)w * h, RtPixelFeatures());
            fs.albedo.assign((size_t)w * h * 4, 0.0f);
            fs.normal.assign((size_t)w * h * 4, 0.0f);
        }
    }
    return rc;
}

int orFeatures_rtDispatch(RtContext* c, int kernelIndex, int gx, int gy, int gz)
{
    const int rc = rtDispatch(c, kernelIndex, gx, gy, gz);
    if (rc != RT_OK || kernelIndex != RT_KERNEL_RESET_ACCUMULATED) return rc;
    FeatureState& fs = featureState(c);
    if (fs.frame.empty()) return rc;
    const uint W = c->sh.Resolution[0], H = c->sh.Resolution[1];
    const uint limX = gz == 0 ? 0u : ((uint)gx * 8u < W ? (uint)gx * 8u : W), limY = gz == 0 ? 0u : ((uint)gy * 8u < H ? (uint)gy * 8u : H);
    for (uint y = 0; y < limY; y++)
    {
        memset(&fs.albedo[((size_t)y * W) * 4], 0, (size_t)limX * 16);
        memset(&fs.normal[((size_t)y * W) * 4], 0, (size_t)limX * 16);
    }
    return rc;
}

int orFeatures_rtReadback(RtContext* c, const char* tex, float* dst, size_t bytes)
{
    const std::string n(c && tex && dst ? tex : "");
    if (n != "FeatureFrame" && n != "AccumulatedAlbedo" && n != "AccumulatedNormal") return rtReadback(c, tex, dst, bytes);
    const FeatureState& fs = featureState(c);
    if (fs.frame.empty()) return fail(c, RT_E_STATE, "rtReadback: no rtDispatchFeatures yet");
    const void* src = n == "FeatureFrame" ? (const void*)fs.frame.data() : n == "AccumulatedAlbedo" ? (const void*)fs.albedo.data() : (const void*)fs.normal.data();
    const size_t size = n == "FeatureFrame" ? fs.frame.size() * sizeof(RtPixelFeatures) : fs.albedo.size() * 4;
    if (bytes != size) return fail(c, RT_E_INVALID, "rtReadback: wrong bytes for the image");
    memcpy(dst, src, bytes);
    return RT_OK;
}

} // extern "C"
