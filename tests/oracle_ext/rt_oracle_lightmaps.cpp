/* rt_oracle_lightmaps.cpp — rtBakeLightmap / rtBakeLightmapDevice (include/rt_b200.h) for the oracle, built around it rather than inside
 * it.  Test infrastructure: ray_tracing_b200/build.py compiles THIS file into oracle/liboracle.so.  It includes the oracle with
 * rtBakeCubemaps (rt_oracle_cubemaps.cpp, which includes the rest) and restates the lightmap bake from the header's statement: the
 * normal, Duff et al.'s tangent frame, the R2 point and the cosine-weighted direction in binary32, one operation at a time
 * (-ffp-contract=off), the origin lifted by 0.001 along the normal, Shader::Trace (oracle/rt_oracle.cpp, HL:479-542) per sample from
 * CreateRay(o, d, 1, 0) with state H(H(seed + p) + k), the chunk sums in k order, and the full binary tree over the chunk count padded
 * with +0 chunks to a power of two, written out level by level, over S.  Its box / triangle / sphere tests and CalculateRayCollision
 * calls are the counters RtStats gets.
 *
 * Test hooks: orLightmapRays returns every sample's start (o, d, state) as an RtPathRay, so that a test can rebuild a texel through
 * rtTracePaths(samples = 1) and check the directions; orLightmapTexels bakes only texels first .. first + count - 1 of a call, so that a
 * test can check rows of a call too large for the oracle to bake whole. */
#include "rt_oracle_cubemaps.cpp"

namespace {

// Sample k of the texel at (position P, normal M): its origin and direction
void surfaceRay(const RtSurfacePoint& pt, uint k, float3& o, float3& d)
{
    const float u = (float)(uint)(k * 3242174889u + 2147483648u) * 2.3283064365386963e-10f;     // R2, as cubeDirection
    const float v = (float)(uint)(k * 2447445414u + 2147483648u) * 2.3283064365386963e-10f;
    const float3 n = normalize(mk3(pt.normal));
    const float sg = std::copysign(1.0f, n.z);
    const float a = -1.0f / (sg + n.z);
    const float b = (n.x * n.y) * a;
    const float3 T = mk3(1.0f + ((sg * n.x) * n.x) * a, sg * b, -(sg * n.x));
    const float3 B = mk3(b, sg + (n.y * n.y) * a, -n.y);
    const float r = orc::sqrt(u);
    const float phi = v * 6.28318548f;
    const float s = orc::sin(phi), c = orc::cos(phi);
    const float x = r * c, y = r * s, z = orc::sqrt(std::max(1.0f - u, 0.0f));
    d = normalize(mk3((T.x * x + B.x * y) + n.x * z, (T.y * x + B.y * y) + n.y * z, (T.z * x + B.z * y) + n.z * z));
    o = mk3(pt.position[0] + n.x * 0.001f, pt.position[1] + n.y * 0.001f, pt.position[2] + n.z * 0.001f);
}

int lightmapChecks(RtContext* c, const char* what, const void* points, const void* out, int n, int samples)
{
    if (n < 0 || (n > 0 && (!points || !out))) return fail(c, RT_E_INVALID, std::string(what) + ": bad argument");
    if (samples < 1 || samples > RT_MAX_BATCH_SAMPLES) return fail(c, RT_E_INVALID, std::string(what) + ": samples must be 1 .. RT_MAX_BATCH_SAMPLES");
    if (n == 0) return RT_OK;
    if (c->sh.MaxBounceCount < 0 || c->sh.MaxBounceCount > 200) return fail(c, RT_E_STATE, std::string(what) + ": MaxBounceCount must be 0 .. 200 (as rtDispatch)");
    return traceChecks(c, what, points, out, n, 0);
}

// Texels first .. first + count - 1 of the call rtBakeLightmap(points, samples, seed) -> out[0 .. count - 1]
void lightmapTexels(RtContext* c, const RtSurfacePoint* points, int samples, uint32_t seed, uint first, int count, RtCubeTexel* out)
{
    const int chunks = (samples + RT_PROBE_CHUNK - 1) / RT_PROBE_CHUNK;
    std::vector<float> sums((size_t)count * chunks * 3, 0.0f);                  // [texel][chunk][rgb], each from +0
    std::vector<uint32_t> rejected((size_t)count * chunks, 0u);
    std::atomic<long long> next(0);
    const long long jobs = (long long)count * chunks;
    std::vector<Shader> shaders(c->threads, c->sh);
    std::vector<std::thread> pool;
    for (int t = 0; t < c->threads; t++)
    {
        pool.emplace_back([&, t]() {
            Shader& s = shaders[t];
            bind_buffers(c, s);
            for (;;)
            {
                const long long j = next.fetch_add(1);
                if (j >= jobs) break;
                const uint p = first + (uint)(j / chunks);
                const int chunk = (int)(j % chunks);
                float* sum = &sums[(size_t)j * 3];
                const uint key = probeHash(seed + p);
                for (int k = chunk * RT_PROBE_CHUNK; k < samples && k < (chunk + 1) * RT_PROBE_CHUNK; k++)
                {
                    float3 o, d;
                    surfaceRay(points[p], (uint)k, o, d);
                    uint rngState = probeHash(key + (uint)k);
                    const float3 L = s.Trace(Shader::CreateRay(o, d, mk3(1.0f), 0), rngState);
                    if (!std::isfinite(L.x) || !std::isfinite(L.y) || !std::isfinite(L.z)) { rejected[(size_t)j]++; continue; }
                    sum[0] += L.x; sum[1] += L.y; sum[2] += L.z;
                }
            }
        });
    }
    for (auto& th : pool) th.join();
    for (auto& s : shaders) { c->stats.rays += s.nRays; c->stats.boxTests += s.nBox; c->stats.triTests += s.nTri; c->stats.sphereTests += s.nSphere; }
    int padded = 1;
    while (padded < chunks) padded *= 2;
    std::vector<float> level(padded);
    for (int i = 0; i < count; i++)
    {
        for (int v = 0; v < 3; v++)
        {
            for (int k = 0; k < padded; k++) level[k] = k < chunks ? sums[((size_t)i * chunks + k) * 3 + v] : 0.0f;
            for (int w = padded; w > 1; w /= 2)
                for (int k = 0; k < w / 2; k++) level[k] = level[2 * k] + level[2 * k + 1];
            out[i].rgb[v] = level[0] / (float)samples;
        }
        uint32_t r = 0;
        for (int k = 0; k < chunks; k++) r += rejected[(size_t)i * chunks + k];
        out[i].rejected = r;
    }
}

} // namespace

extern "C" {

int rtBakeLightmap(RtContext* c, const RtSurfacePoint* points, int n, int samples, uint32_t seed, RtCubeTexel* out)
{
    if (!c) return RT_E_INVALID;
    const int rc = lightmapChecks(c, "rtBakeLightmap", points, out, n, samples);
    if (rc != RT_OK || n == 0) return rc;
    lightmapTexels(c, points, samples, seed, 0u, n, out);
    return RT_OK;
}

int rtBakeLightmapDevice(RtContext* c, const void*, void*, int, int, uint32_t) { return c ? fail(c, RT_E_STATE, "oracle: no device memory") : RT_E_INVALID; }

/* Test hook: texels first .. first + count - 1 of rtBakeLightmap(points, n, samples, seed) -> out[0 .. count - 1], with the call's
 * checks; RtStats grows by those texels' work only. */
int orLightmapTexels(RtContext* c, const RtSurfacePoint* points, int n, int samples, uint32_t seed, int first, int count, RtCubeTexel* out)
{
    if (!c) return RT_E_INVALID;
    const int rc = lightmapChecks(c, "orLightmapTexels", points, out, n, samples);
    if (rc != RT_OK) return rc;
    if (first < 0 || count < 0 || (long long)first + count > (long long)n) return fail(c, RT_E_INVALID, "orLightmapTexels: bad range");
    if (count > 0) lightmapTexels(c, points, samples, seed, (uint)first, count, out);
    return RT_OK;
}

/* Test hook: the start of every sample of rtBakeLightmap(points, n, samples, seed), out[p * samples + k] = {o, d, H(H(seed + p) + k)}:
 * rtTracePaths(out, samples = 1).rgb is the sample's radiance. */
int orLightmapRays(RtContext* c, const RtSurfacePoint* points, int n, int samples, uint32_t seed, RtPathRay* out)
{
    if (!c || n < 0 || samples < 1 || (n > 0 && (!points || !out))) return fail(c, RT_E_INVALID, "orLightmapRays: bad argument");
    for (int p = 0; p < n; p++)
    {
        const uint key = probeHash(seed + (uint)p);
        for (int k = 0; k < samples; k++)
        {
            RtPathRay& r = out[(size_t)p * samples + k];
            float3 o, d;
            surfaceRay(points[p], (uint)k, o, d);
            r.origin[0] = o.x; r.origin[1] = o.y; r.origin[2] = o.z;
            r.dir[0] = d.x; r.dir[1] = d.y; r.dir[2] = d.z;
            r.rngState = probeHash(key + (uint)k);
        }
    }
    return RT_OK;
}

} // extern "C"
