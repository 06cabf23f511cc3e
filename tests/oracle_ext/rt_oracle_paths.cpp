/* rt_oracle_paths.cpp — rtTracePaths / rtTracePathsDevice (include/rt_b200.h) for the oracle, built around it rather than inside it.
 * Test infrastructure: ray_tracing_b200/build.py compiles THIS file into oracle/liboracle.so.  It includes the oracle with
 * rtTraceOcclusion (rt_oracle_occlusion.cpp, which includes the rest) and adds the path query.
 *
 * rtTracePaths is the reference's per-pixel sample loop (HL:560-581) with the caller's ray in place of the jittered camera ray:
 * Shader::Trace (oracle/rt_oracle.cpp, HL:479-542) once per sample on one RNG chain, the sum over (float)samples.  Its box / triangle /
 * sphere tests and CalculateRayCollision calls are the counters RtStats gets.  The test hook orCameraSample returns the camera ray of a
 * pixel and the RNG state after its four jitter draws (HL:565-572) — exactly what RayTrace hands to Trace — so that a test can rebuild a
 * pixel of rtDispatch sample by sample through rtTracePaths. */
#include "rt_oracle_occlusion.cpp"

namespace {

int pathChecks(RtContext* c, const char* what, const void* rays, const void* out, int n, int samples)
{
    if (n < 0 || (n > 0 && (!rays || !out))) return fail(c, RT_E_INVALID, std::string(what) + ": bad argument");
    if (samples < 1 || samples > RT_MAX_BATCH_SAMPLES) return fail(c, RT_E_INVALID, std::string(what) + ": samples must be 1 .. RT_MAX_BATCH_SAMPLES");
    if (n == 0) return RT_OK;
    if (c->sh.MaxBounceCount < 0 || c->sh.MaxBounceCount > 200) return fail(c, RT_E_STATE, std::string(what) + ": MaxBounceCount must be 0 .. 200 (as rtDispatch)");
    return traceChecks(c, what, rays, out, n, 0);
}

} // namespace

extern "C" {

int rtTracePaths(RtContext* c, const RtPathRay* rays, int n, int samples, RtPathRadiance* out)
{
    if (!c) return RT_E_INVALID;
    const int rc = pathChecks(c, "rtTracePaths", rays, out, n, samples);
    if (rc != RT_OK || n == 0) return rc;
    std::atomic<int> next(0);
    std::vector<Shader> shaders(c->threads, c->sh);
    std::vector<std::thread> pool;
    for (int t = 0; t < c->threads; t++)
    {
        pool.emplace_back([&, t]() {
            Shader& s = shaders[t];
            bind_buffers(c, s);
            for (;;)
            {
                const int i0 = next.fetch_add(16);
                if (i0 >= n) break;
                for (int i = i0; i < n && i < i0 + 16; i++)
                {
                    uint rngState = rays[i].rngState;
                    float3 total = mk3(0.0f);
                    for (int k = 0; k < samples; k++)
                        total += s.Trace(Shader::CreateRay(mk3(rays[i].origin), mk3(rays[i].dir), mk3(1.0f), 0), rngState);     // HL:578
                    const float3 col = total / (float)samples;                                                                  // HL:581
                    out[i].rgb[0] = col.x; out[i].rgb[1] = col.y; out[i].rgb[2] = col.z;
                    out[i].rngState = rngState;
                }
            }
        });
    }
    for (auto& th : pool) th.join();
    for (auto& s : shaders) { c->stats.rays += s.nRays; c->stats.boxTests += s.nBox; c->stats.triTests += s.nTri; c->stats.sphereTests += s.nSphere; }
    return RT_OK;
}

int rtTracePathsDevice(RtContext* c, const void*, void*, int, int) { return c ? fail(c, RT_E_STATE, "oracle: no device memory") : RT_E_INVALID; }

/* Test hook: the camera ray of pixel (x, y) and the RNG state after its four jitter draws (HL:565-572), as RayTrace computes them for
 * the current camera, "Resolution", "DefocusStrength" and "DivergeStrength".  The draws start from *stateIn, or, with stateIn NULL,
 * from the pixel's own seed for the current "Frame" and "renderSeed" (HL:550-552, the pixel index taken from uv as there). */
int orCameraSample(RtContext* c, int x, int y, const uint32_t* stateIn, RtPathRay* out)
{
    if (!c || !out || x < 0 || y < 0) return fail(c, RT_E_INVALID, "orCameraSample: bad argument");
    const Shader& s = c->sh;
    const uint* numPixels = s.Resolution;
    const float2 uv = mk2((float)(uint)x / ((float)numPixels[0] - 1.0f), (float)(uint)y / ((float)numPixels[1] - 1.0f));   // RayCompute.compute:15
    // RayTrace (HL:545-576) up to the ray it hands to Trace
    float3 camOrigin = mul_xyz(s.CamLocalToWorldMatrix, mk4(mk3(0.0f, 0.0f, 0.0f), 1.0f));
    uint pixelCoordX = orc::f2uint_rz(uv.x * (float)numPixels[0]);
    uint pixelCoordY = orc::f2uint_rz(uv.y * (float)numPixels[1]);
    uint pixelIndex = pixelCoordY * numPixels[0] + pixelCoordX;
    uint rngState = stateIn ? *stateIn : pixelIndex + (uint)s.Frame * 719393u + (uint)s.renderSeed;
    float3 focusPointLocal = mk3(uv.x - 0.5f, uv.y - 0.5f, 1.0f) * s.ViewParams;
    float3 focusPoint = mul_xyz(s.CamLocalToWorldMatrix, mk4(focusPointLocal, 1.0f));
    float3 camRight = mk3(M(s.CamLocalToWorldMatrix,0,0), M(s.CamLocalToWorldMatrix,1,0), M(s.CamLocalToWorldMatrix,2,0));
    float3 camUp = mk3(M(s.CamLocalToWorldMatrix,0,1), M(s.CamLocalToWorldMatrix,1,1), M(s.CamLocalToWorldMatrix,2,1));
    float2 defocusJitter = Shader::RandomPointInCircle(rngState) * s.DefocusStrength / (float)numPixels[0];
    float3 rayOrigin = camOrigin + camRight * defocusJitter.x + camUp * defocusJitter.y;
    float2 jitter = Shader::RandomPointInCircle(rngState) * s.DivergeStrength / (float)numPixels[0];
    float3 jitteredFocusPoint = focusPoint + camRight * jitter.x + camUp * jitter.y;
    float3 rayDir = normalize(jitteredFocusPoint - rayOrigin);
    out->origin[0] = rayOrigin.x; out->origin[1] = rayOrigin.y; out->origin[2] = rayOrigin.z;
    out->dir[0] = rayDir.x; out->dir[1] = rayDir.y; out->dir[2] = rayDir.z;
    out->rngState = rngState;
    return RT_OK;
}

/* Test hook: orCameraSample for n pixels (xy = n pairs), each from statesIn[i] or, with statesIn NULL, from its own seed. */
int orCameraSamples(RtContext* c, const int* xy, int n, const uint32_t* statesIn, RtPathRay* out)
{
    if (!c || n < 0 || (n > 0 && (!xy || !out))) return fail(c, RT_E_INVALID, "orCameraSamples: bad argument");
    for (int i = 0; i < n; i++)
    {
        const int rc = orCameraSample(c, xy[2 * i], xy[2 * i + 1], statesIn ? statesIn + i : nullptr, out + i);
        if (rc != RT_OK) return rc;
    }
    return RT_OK;
}

} // extern "C"
