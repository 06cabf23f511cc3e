/* rt_oracle_trace_rays.cpp — rtTraceRays / rtTraceRaysDevice (include/rt_b200.h) for the oracle, built around it rather than inside
 * it.  Test infrastructure: ray_tracing_b200/build.py compiles THIS file into oracle/liboracle.so.  It includes the oracle with its
 * per-pixel counters and rtDispatchFrames (rt_oracle_frames.cpp, which includes oracle/rt_oracle.cpp unchanged) and adds the query:
 * Shader::CalculateRayCollision per ray, multi-threaded like orRenderPixels, its counters added to RtStats.
 *
 * The oracle's hit carries a copy of the winner's material, not its index.  So the winner is found by a restatement of the
 * collision loop (tracedWinner) over the oracle's own RaySphere / RayTriangleBVH that also records which entry won; the test hook
 * orTraceRaysLoop returns that loop's hits, and a test checks that they equal CalculateRayCollision's for every ray. */
#include "rt_oracle_frames.cpp"

namespace {

// CalculateRayCollision (oracle/rt_oracle.cpp, HL:335-374 with the sphere extension first), recording the winner's kind and index
Shader::ModelHitInfo tracedWinner(Shader& s, float3 pos, float3 dir, bool forceDontCullBack, int& kind, int& index)
{
    Shader::ModelHitInfo result;
    memset(&result, 0, sizeof(result));
    result.dst = rt_inf();
    kind = RT_HIT_NONE; index = -1;
    for (int i = 0; i < s.sphereCount; i++)
    {
        const RtSphere& sphere = s.Spheres[i];
        Shader::ModelHitInfo h = Shader::RaySphere(pos, dir, mk3(sphere.centre), sphere.radius);
        if (h.didHit && h.dst < result.dst) { result = h; kind = RT_HIT_SPHERE; index = i; }
    }
    for (int i = 0; i < s.modelCount; i++)
    {
        const RtModel& model = s.ModelInfo[i];
        float4x4 worldToLocalMatrix, localToWorldMatrix;
        memcpy(worldToLocalMatrix.m, model.worldToLocal, 64);
        memcpy(localToWorldMatrix.m, model.localToWorld, 64);
        Shader::Ray localRay;
        localRay.transmittance = mk3(0.0f);
        localRay.bounceCount = 0;
        localRay.pos = mul_xyz(worldToLocalMatrix, mk4(pos, 1.0f));
        localRay.dir = mul_xyz(worldToLocalMatrix, mk4(dir, 0.0f));
        localRay.invDir = 1.0f / localRay.dir;
        const bool cullBackface = !forceDontCullBack && model.material.flag != Shader::MATERIAL_GLASS;
        Shader::TriangleHitInfo hit = s.RayTriangleBVH(localRay, result.dst, model.nodeOffset, model.triOffset, cullBackface);
        if (hit.dst < result.dst)
        {
            result.didHit = true;
            result.isBackface = hit.isBackface;
            result.dst = hit.dst;
            result.normal = normalize(mul_xyz(localToWorldMatrix, mk4(hit.normal, 0.0f)));
            result.pos = pos + dir * hit.dst;
            kind = RT_HIT_MODEL; index = i;
        }
    }
    return result;
}

void putHit(RtRayHit& o, const Shader::ModelHitInfo& h, int kind, int index)
{
    memset(&o, 0, sizeof(o));
    o.dst = h.dst;
    o.pos[0] = h.pos.x; o.pos[1] = h.pos.y; o.pos[2] = h.pos.z;
    o.normal[0] = h.normal.x; o.normal[1] = h.normal.y; o.normal[2] = h.normal.z;
    o.isBackface = h.isBackface ? 1 : 0;
    o.kind = kind; o.index = index;
}

// The argument and scene checks of the product's rtTraceRays (the scene checks are rtDispatch's)
int traceChecks(RtContext* c, const char* what, const void* rays, const void* hits, int n, int flags)
{
    if (n < 0 || (n > 0 && (!rays || !hits))) return fail(c, RT_E_INVALID, std::string(what) + ": bad argument");
    if (flags != 0 && flags != RT_TRACE_NO_CULL) return fail(c, RT_E_INVALID, std::string(what) + ": flags must be 0 or RT_TRACE_NO_CULL");
    if (n == 0) return RT_OK;
    if (c->sh.modelCount < 0 || c->sh.modelCount > (int)c->models.size()) return fail(c, RT_E_STATE, std::string(what) + ": modelCount exceeds ModelInfo length");
    if (c->sh.modelCount > 0 && (c->nodes.empty() || c->triangles.empty())) return fail(c, RT_E_STATE, std::string(what) + ": models without Nodes / Triangles buffers");
    for (int i = 0; i < c->sh.modelCount; i++)
        if (c->models[i].triOffset < 0 || (size_t)c->models[i].triOffset > c->triangles.size()) return fail(c, RT_E_STATE, std::string(what) + ": model triOffset out of range");
    std::string why;
    if (bvhTooDeepOrBroken(c, why)) return fail(c, RT_E_STATE, std::string(what) + ": " + why);
    return RT_OK;
}

// n rays on the context's threads; loop = false: CalculateRayCollision + the winner (counters into RtStats), true: tracedWinner alone
int traceAll(RtContext* c, const RtRay* rays, int n, RtRayHit* hits, int flags, bool loop)
{
    const bool noCull = (flags & RT_TRACE_NO_CULL) != 0;
    std::atomic<int> next(0);
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
                const int i0 = next.fetch_add(64);
                if (i0 >= n) break;
                for (int i = i0; i < n && i < i0 + 64; i++)
                {
                    Shader::Ray ray;
                    memset(&ray, 0, sizeof(ray));
                    ray.pos = mk3(rays[i].origin); ray.dir = mk3(rays[i].dir); ray.invDir = 1.0f / ray.dir;
                    int kind, index;
                    const Shader::ModelHitInfo winner = tracedWinner(w, ray.pos, ray.dir, noCull, kind, index);
                    putHit(hits[i], loop ? winner : s.CalculateRayCollision(ray, noCull), kind, index);
                }
            }
        });
    }
    for (auto& th : pool) th.join();
    if (!loop)
        for (auto& s : shaders) { c->stats.rays += s.nRays; c->stats.boxTests += s.nBox; c->stats.triTests += s.nTri; c->stats.sphereTests += s.nSphere; }
    return RT_OK;
}

} // namespace

extern "C" {

int rtTraceRays(RtContext* c, const RtRay* rays, int n, RtRayHit* hits, int flags)
{
    if (!c) return RT_E_INVALID;
    const int rc = traceChecks(c, "rtTraceRays", rays, hits, n, flags);
    if (rc != RT_OK || n == 0) return rc;
    return traceAll(c, rays, n, hits, flags, false);
}

int rtTraceRaysDevice(RtContext* c, const void*, void*, int, int) { return c ? fail(c, RT_E_STATE, "oracle: no device memory") : RT_E_INVALID; }

/* Test hook: the hits of the winner-recording loop alone (RtStats untouched), to compare with rtTraceRays' CalculateRayCollision. */
int orTraceRaysLoop(RtContext* c, const RtRay* rays, int n, RtRayHit* hits, int flags)
{
    if (!c) return RT_E_INVALID;
    const int rc = traceChecks(c, "orTraceRaysLoop", rays, hits, n, flags);
    if (rc != RT_OK || n == 0) return rc;
    return traceAll(c, rays, n, hits, flags, true);
}

} // extern "C"
