/* rt_oracle_probes.cpp — rtBakeProbes / rtBakeProbesDevice (include/rt_b200.h) for the oracle, built around it rather than inside it.
 * Test infrastructure: ray_tracing_b200/build.py compiles THIS file into oracle/liboracle.so.  It includes the oracle with
 * rtDispatchAdaptive (rt_oracle_adaptive.cpp, which includes the rest) and restates the probe bake from the header's statement: the
 * spherical Fibonacci directions in binary32, one operation at a time (-ffp-contract=off), Shader::Trace (oracle/rt_oracle.cpp,
 * HL:479-542) per sample from CreateRay(position, d_k, 1, 0) with state H(H(seed + p) + k), the basis, the chunk sums in k order, and
 * the full binary tree over the chunk count padded with +0 chunks to a power of two, written out level by level.  Its box / triangle /
 * sphere tests and CalculateRayCollision calls are the counters RtStats gets.
 *
 * The test hook orProbeRays returns every sample's start (position, d_k, state) as an RtPathRay, so that a test can rebuild a probe
 * through rtTracePaths(samples = 1). */
#include "rt_oracle_adaptive.cpp"

namespace {

// H(x): the value NextRandom returns from state x
uint probeHash(uint x) { return Shader::NextRandom(x); }

float3 probeDirection(uint k, int samples)
{
    const float t = (float)(uint)(k * 2654435769u) / 4294967296.0f;           // RandomValue's conversion (HL:137)
    const float phi = t * 6.28318548f;
    const float s = orc::sin(phi), c = orc::cos(phi);
    const float z = 1.0f - (float)(2u * k + 1u) / (float)samples;
    const float r = orc::sqrt(std::max(1.0f - z * z, 0.0f));
    return mk3(r * c, r * s, z);
}

void probeBasis(float3 d, float Y[9])
{
    Y[0] = 0.282094792f;
    Y[1] = 0.488602512f * d.y; Y[2] = 0.488602512f * d.z; Y[3] = 0.488602512f * d.x;
    Y[4] = 1.09254843f * (d.x * d.y); Y[5] = 1.09254843f * (d.y * d.z);
    Y[6] = 0.315391565f * ((3.0f * (d.z * d.z)) - 1.0f);
    Y[7] = 1.09254843f * (d.x * d.z);
    Y[8] = 0.546274215f * ((d.x * d.x) - (d.y * d.y));
}

int probeChecks(RtContext* c, const char* what, const void* positions, const void* out, int n, int samples)
{
    if (n < 0 || (n > 0 && (!positions || !out))) return fail(c, RT_E_INVALID, std::string(what) + ": bad argument");
    if (samples < 1 || samples > RT_MAX_BATCH_SAMPLES) return fail(c, RT_E_INVALID, std::string(what) + ": samples must be 1 .. RT_MAX_BATCH_SAMPLES");
    if (n == 0) return RT_OK;
    if (c->sh.MaxBounceCount < 0 || c->sh.MaxBounceCount > 200) return fail(c, RT_E_STATE, std::string(what) + ": MaxBounceCount must be 0 .. 200 (as rtDispatch)");
    return traceChecks(c, what, positions, out, n, 0);
}

} // namespace

extern "C" {

int rtBakeProbes(RtContext* c, const float* positions, int n, int samples, uint32_t seed, RtProbeSH* out)
{
    if (!c) return RT_E_INVALID;
    const int rc = probeChecks(c, "rtBakeProbes", positions, out, n, samples);
    if (rc != RT_OK || n == 0) return rc;
    const int chunks = (samples + RT_PROBE_CHUNK - 1) / RT_PROBE_CHUNK;
    std::vector<float> sums((size_t)n * chunks * 27, 0.0f);                     // [probe][chunk][ch * 9 + i], each from +0
    std::vector<uint32_t> rejected((size_t)n * chunks, 0u);
    std::atomic<long long> next(0);
    const long long jobs = (long long)n * chunks;
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
                const int p = (int)(j / chunks), chunk = (int)(j % chunks);
                float* sum = &sums[(size_t)j * 27];
                const uint key = probeHash(seed + (uint)p);
                for (int k = chunk * RT_PROBE_CHUNK; k < samples && k < (chunk + 1) * RT_PROBE_CHUNK; k++)
                {
                    const float3 d = probeDirection((uint)k, samples);
                    uint rngState = probeHash(key + (uint)k);
                    const float3 L = s.Trace(Shader::CreateRay(mk3(positions + 3 * (size_t)p), d, mk3(1.0f), 0), rngState);
                    if (!std::isfinite(L.x) || !std::isfinite(L.y) || !std::isfinite(L.z)) { rejected[(size_t)j]++; continue; }
                    float Y[9]; probeBasis(d, Y);
                    for (int i = 0; i < 9; i++) { sum[i] += L.x * Y[i]; sum[9 + i] += L.y * Y[i]; sum[18 + i] += L.z * Y[i]; }
                }
            }
        });
    }
    for (auto& th : pool) th.join();
    for (auto& s : shaders) { c->stats.rays += s.nRays; c->stats.boxTests += s.nBox; c->stats.triTests += s.nTri; c->stats.sphereTests += s.nSphere; }
    int padded = 1;
    while (padded < chunks) padded *= 2;
    const float scale = 12.566371f / (float)samples;
    std::vector<float> level(padded);
    for (int p = 0; p < n; p++)
    {
        for (int v = 0; v < 27; v++)
        {
            for (int k = 0; k < padded; k++) level[k] = k < chunks ? sums[((size_t)p * chunks + k) * 27 + v] : 0.0f;
            for (int w = padded; w > 1; w /= 2)
                for (int k = 0; k < w / 2; k++) level[k] = level[2 * k] + level[2 * k + 1];
            out[p].sh[v / 9][v % 9] = level[0] * scale;
        }
        uint32_t r = 0;
        for (int k = 0; k < chunks; k++) r += rejected[(size_t)p * chunks + k];
        out[p].rejected = r;
    }
    return RT_OK;
}

int rtBakeProbesDevice(RtContext* c, const void*, void*, int, int, uint32_t) { return c ? fail(c, RT_E_STATE, "oracle: no device memory") : RT_E_INVALID; }

/* Test hook: the start of every sample of rtBakeProbes(positions, n, samples, seed), out[p * samples + k] = {positions[p], d_k,
 * H(H(seed + p) + k)}: rtTracePaths(out, samples = 1).rgb is the sample's radiance L_pk. */
int orProbeRays(RtContext* c, const float* positions, int n, int samples, uint32_t seed, RtPathRay* out)
{
    if (!c || n < 0 || samples < 1 || (n > 0 && (!positions || !out))) return fail(c, RT_E_INVALID, "orProbeRays: bad argument");
    for (int p = 0; p < n; p++)
    {
        const uint key = probeHash(seed + (uint)p);
        for (int k = 0; k < samples; k++)
        {
            RtPathRay& r = out[(size_t)p * samples + k];
            const float3 d = probeDirection((uint)k, samples);
            for (int a = 0; a < 3; a++) r.origin[a] = positions[3 * (size_t)p + a];
            r.dir[0] = d.x; r.dir[1] = d.y; r.dir[2] = d.z;
            r.rngState = probeHash(key + (uint)k);
        }
    }
    return RT_OK;
}

} // extern "C"
