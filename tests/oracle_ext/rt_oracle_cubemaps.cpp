/* rt_oracle_cubemaps.cpp — rtBakeCubemaps / rtBakeCubemapsDevice (include/rt_b200.h) for the oracle, built around it rather than inside
 * it.  Test infrastructure: ray_tracing_b200/build.py compiles THIS file into oracle/liboracle.so.  It includes the oracle with
 * rtBakeProbes (rt_oracle_probes.cpp, which includes the rest) and restates the cube-map bake from the header's statement: the R2
 * sub-texel offsets and the face table in binary32, one operation at a time (-ffp-contract=off), Shader::Trace (oracle/rt_oracle.cpp,
 * HL:479-542) per sample from CreateRay(position, d, 1, 0) with state H(H(seed + tau) + k), the chunk sums in k order, and the full
 * binary tree over the chunk count padded with +0 chunks to a power of two, written out level by level, over S.  Its box / triangle /
 * sphere tests and CalculateRayCollision calls are the counters RtStats gets.
 *
 * Test hooks: orCubemapRays returns every sample's start (position, d, state) as an RtPathRay, so that a test can rebuild a texel
 * through rtTracePaths(samples = 1); orCubemapTexels bakes only texels first .. first + count - 1 of a call, so that a test can check
 * rows of a call too large for the oracle to bake whole. */
#include "rt_oracle_probes.cpp"

namespace {

float3 cubeDirection(uint f, uint x, uint y, uint k, int N)
{
    const float u = (float)(uint)(k * 3242174889u + 2147483648u) * 2.3283064365386963e-10f;     // R2, RandomValue's conversion
    const float v = (float)(uint)(k * 2447445414u + 2147483648u) * 2.3283064365386963e-10f;
    const float a = (((float)x + u) / (float)N) * 2.0f - 1.0f;
    const float b = (((float)y + v) / (float)N) * 2.0f - 1.0f;
    const float3 w[6] = {mk3(1.0f, -b, -a), mk3(-1.0f, -b, a), mk3(a, 1.0f, b), mk3(a, -1.0f, -b), mk3(a, -b, 1.0f), mk3(-a, -b, -1.0f)};
    return normalize(w[f]);
}

// The texel tau of a call: its probe, face, column and row
struct CubeTexel { uint p, f, x, y; };
CubeTexel cubeTexel(uint tau, int N)
{
    const uint n = (uint)N;
    return {tau / (6u * n * n), (tau / (n * n)) % 6u, tau % n, (tau / n) % n};
}

int cubeChecks(RtContext* c, const char* what, const void* positions, const void* out, int n, int faceSize, int samples)
{
    if (n < 0 || (n > 0 && (!positions || !out))) return fail(c, RT_E_INVALID, std::string(what) + ": bad argument");
    if (samples < 1 || samples > RT_MAX_BATCH_SAMPLES) return fail(c, RT_E_INVALID, std::string(what) + ": samples must be 1 .. RT_MAX_BATCH_SAMPLES");
    if (faceSize < 1 || faceSize > RT_CUBE_MAX_FACE) return fail(c, RT_E_INVALID, std::string(what) + ": faceSize must be 1 .. RT_CUBE_MAX_FACE");
    if ((long long)n * 6 * faceSize * faceSize > 0x7fffffffLL) return fail(c, RT_E_INVALID, std::string(what) + ": too many texels");
    if (n == 0) return RT_OK;
    if (c->sh.MaxBounceCount < 0 || c->sh.MaxBounceCount > 200) return fail(c, RT_E_STATE, std::string(what) + ": MaxBounceCount must be 0 .. 200 (as rtDispatch)");
    return traceChecks(c, what, positions, out, n, 0);
}

// Texels first .. first + count - 1 of the call rtBakeCubemaps(positions, faceSize, samples, seed) -> out[0 .. count - 1]
void cubeTexels(RtContext* c, const float* positions, int faceSize, int samples, uint32_t seed, uint first, int count, RtCubeTexel* out)
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
                const uint tau = first + (uint)(j / chunks);
                const int chunk = (int)(j % chunks);
                const CubeTexel T = cubeTexel(tau, faceSize);
                float* sum = &sums[(size_t)j * 3];
                const uint key = probeHash(seed + tau);
                for (int k = chunk * RT_PROBE_CHUNK; k < samples && k < (chunk + 1) * RT_PROBE_CHUNK; k++)
                {
                    const float3 d = cubeDirection(T.f, T.x, T.y, (uint)k, faceSize);
                    uint rngState = probeHash(key + (uint)k);
                    const float3 L = s.Trace(Shader::CreateRay(mk3(positions + 3 * (size_t)T.p), d, mk3(1.0f), 0), rngState);
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

int rtBakeCubemaps(RtContext* c, const float* positions, int n, int faceSize, int samples, uint32_t seed, RtCubeTexel* out)
{
    if (!c) return RT_E_INVALID;
    const int rc = cubeChecks(c, "rtBakeCubemaps", positions, out, n, faceSize, samples);
    if (rc != RT_OK || n == 0) return rc;
    cubeTexels(c, positions, faceSize, samples, seed, 0u, n * 6 * faceSize * faceSize, out);
    return RT_OK;
}

int rtBakeCubemapsDevice(RtContext* c, const void*, void*, int, int, int, uint32_t) { return c ? fail(c, RT_E_STATE, "oracle: no device memory") : RT_E_INVALID; }

/* Test hook: texels first .. first + count - 1 of rtBakeCubemaps(positions, n, faceSize, samples, seed) -> out[0 .. count - 1], with
 * the call's checks; RtStats grows by those texels' work only. */
int orCubemapTexels(RtContext* c, const float* positions, int n, int faceSize, int samples, uint32_t seed, int first, int count, RtCubeTexel* out)
{
    if (!c) return RT_E_INVALID;
    const int rc = cubeChecks(c, "orCubemapTexels", positions, out, n, faceSize, samples);
    if (rc != RT_OK) return rc;
    if (first < 0 || count < 0 || (long long)first + count > (long long)n * 6 * faceSize * faceSize) return fail(c, RT_E_INVALID, "orCubemapTexels: bad range");
    if (count > 0) cubeTexels(c, positions, faceSize, samples, seed, (uint)first, count, out);
    return RT_OK;
}

/* Test hook: the start of every sample of rtBakeCubemaps(positions, n, faceSize, samples, seed), out[tau * samples + k] = {positions[p],
 * d, H(H(seed + tau) + k)}: rtTracePaths(out, samples = 1).rgb is the sample's radiance. */
int orCubemapRays(RtContext* c, const float* positions, int n, int faceSize, int samples, uint32_t seed, RtPathRay* out)
{
    if (!c || n < 0 || samples < 1 || faceSize < 1 || (n > 0 && (!positions || !out))) return fail(c, RT_E_INVALID, "orCubemapRays: bad argument");
    const uint texels = (uint)n * 6u * (uint)faceSize * (uint)faceSize;
    for (uint tau = 0; tau < texels; tau++)
    {
        const CubeTexel T = cubeTexel(tau, faceSize);
        const uint key = probeHash(seed + tau);
        for (int k = 0; k < samples; k++)
        {
            RtPathRay& r = out[(size_t)tau * samples + k];
            const float3 d = cubeDirection(T.f, T.x, T.y, (uint)k, faceSize);
            for (int a = 0; a < 3; a++) r.origin[a] = positions[3 * (size_t)T.p + a];
            r.dir[0] = d.x; r.dir[1] = d.y; r.dir[2] = d.z;
            r.rngState = probeHash(key + (uint)k);
        }
    }
    return RT_OK;
}

} // extern "C"
