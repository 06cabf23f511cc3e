/* rt_oracle_occlusion.cpp — rtTraceOcclusion / rtTraceOcclusionDevice (include/rt_b200.h) for the oracle, built around it rather than
 * inside it.  Test infrastructure: ray_tracing_b200/build.py compiles THIS file into oracle/liboracle.so.  It includes the oracle with
 * rtTraceRays (rt_oracle_trace_rays.cpp, which includes the rest) and adds the occlusion query.
 *
 * rtTraceOcclusion is the definition's early-exit form, restated over the oracle's own RaySphere, RayTriangle and RayBoundingBoxDst:
 * spheres in buffer order, then every model in buffer order, each BVH walked as RayTriangleBVH walks it (HL:234-287) but bounded by
 * the segment's tMax and ended by the first primitive that hits closer than tMax.  Its box / triangle / sphere tests are the counters
 * RtStats gets.  The test hook orTraceOcclusionFull is the definition itself: CalculateRayCollision's loop (HL:335-374, sphere
 * extension first) with result.dst starting at tMax and no exit, RayTriangleBVH seeded with the running result as the reference seeds
 * it.  A test checks that the two booleans agree on every segment. */
#include "rt_oracle_trace_rays.cpp"

namespace {

Shader::Ray localRayOf(const RtModel& model, float3 pos, float3 dir)
{
    float4x4 worldToLocalMatrix;
    memcpy(worldToLocalMatrix.m, model.worldToLocal, 64);
    Shader::Ray localRay;
    localRay.transmittance = mk3(0.0f);
    localRay.bounceCount = 0;
    localRay.pos = mul_xyz(worldToLocalMatrix, mk4(pos, 1.0f));
    localRay.dir = mul_xyz(worldToLocalMatrix, mk4(dir, 0.0f));
    localRay.invDir = 1.0f / localRay.dir;
    return localRay;
}

bool cullsBackfaces(const RtModel& model, bool forceDontCullBack)
{
    return !forceDontCullBack && model.material.flag != Shader::MATERIAL_GLASS;
}

// RayTriangleBVH (HL:234-287) with result.dst fixed at rayLength: true at the first triangle that hits closer than rayLength
bool meshHitBefore(Shader& s, const Shader::Ray& ray, float rayLength, int nodeOffset, int triOffset, bool cullBackface)
{
    int stack[64];
    int stackCount = 0;
    stack[stackCount++] = nodeOffset + 0;
    while (stackCount > 0)
    {
        const RtNode& node = s.Nodes[stack[--stackCount]];
        if (node.triangleCount > 0)
        {
            for (int i = 0; i < node.triangleCount; i++)
            {
                const Shader::TriangleHitInfo h = Shader::RayTriangle(ray, s.Triangles[triOffset + node.startIndex + i], cullBackface);
                s.nTri++;
                if (h.didHit && h.dst < rayLength) return true;
            }
        }
        else
        {
            const int childIndexA = nodeOffset + node.startIndex + 0;
            const int childIndexB = nodeOffset + node.startIndex + 1;
            const RtNode& childA = s.Nodes[childIndexA];
            const RtNode& childB = s.Nodes[childIndexB];
            const float dstA = Shader::RayBoundingBoxDst(ray, mk3(childA.boundsMin), mk3(childA.boundsMax));
            const float dstB = Shader::RayBoundingBoxDst(ray, mk3(childB.boundsMin), mk3(childB.boundsMax));
            s.nBox += 2;
            const bool isNearestA = dstA <= dstB;
            const float dstNear = isNearestA ? dstA : dstB;
            const float dstFar = isNearestA ? dstB : dstA;
            if (dstFar < rayLength) stack[stackCount++] = isNearestA ? childIndexB : childIndexA;
            if (dstNear < rayLength) stack[stackCount++] = isNearestA ? childIndexA : childIndexB;
        }
    }
    return false;
}

// The early-exit walk: rtTraceOcclusion's answer and counters
bool occludedEarly(Shader& s, float3 pos, float3 dir, float tMax, bool forceDontCullBack)
{
    s.nRays++;
    for (int i = 0; i < s.sphereCount; i++)
    {
        const RtSphere& sphere = s.Spheres[i];
        const Shader::ModelHitInfo h = Shader::RaySphere(pos, dir, mk3(sphere.centre), sphere.radius);
        s.nSphere++;
        if (h.didHit && h.dst < tMax) return true;
    }
    for (int i = 0; i < s.modelCount; i++)
    {
        const RtModel& model = s.ModelInfo[i];
        if (meshHitBefore(s, localRayOf(model, pos, dir), tMax, model.nodeOffset, model.triOffset, cullsBackfaces(model, forceDontCullBack)))
            return true;
    }
    return false;
}

// The definition: CalculateRayCollision's loop from result.dst = tMax, to the end
bool occludedFull(Shader& s, float3 pos, float3 dir, float tMax, bool forceDontCullBack)
{
    float resultDst = tMax;
    bool didHit = false;
    for (int i = 0; i < s.sphereCount; i++)
    {
        const RtSphere& sphere = s.Spheres[i];
        const Shader::ModelHitInfo h = Shader::RaySphere(pos, dir, mk3(sphere.centre), sphere.radius);
        if (h.didHit && h.dst < resultDst) { resultDst = h.dst; didHit = true; }
    }
    for (int i = 0; i < s.modelCount; i++)
    {
        const RtModel& model = s.ModelInfo[i];
        Shader::Ray localRay = localRayOf(model, pos, dir);
        const Shader::TriangleHitInfo hit = s.RayTriangleBVH(localRay, resultDst, model.nodeOffset, model.triOffset, cullsBackfaces(model, forceDontCullBack));
        if (hit.dst < resultDst) { resultDst = hit.dst; didHit = true; }
    }
    return didHit;
}

// n segments on the context's threads; full = false: the early-exit walk (counters into RtStats), true: the full loop alone
int occlusionAll(RtContext* c, const RtRaySegment* segs, int n, uint8_t* occluded, int flags, bool full)
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
            for (;;)
            {
                const int i0 = next.fetch_add(64);
                if (i0 >= n) break;
                for (int i = i0; i < n && i < i0 + 64; i++)
                {
                    const float3 pos = mk3(segs[i].origin), dir = mk3(segs[i].dir);
                    const bool o = full ? occludedFull(s, pos, dir, segs[i].tMax, noCull) : occludedEarly(s, pos, dir, segs[i].tMax, noCull);
                    occluded[i] = o ? 1 : 0;
                }
            }
        });
    }
    for (auto& th : pool) th.join();
    if (!full)
        for (auto& s : shaders) { c->stats.rays += s.nRays; c->stats.boxTests += s.nBox; c->stats.triTests += s.nTri; c->stats.sphereTests += s.nSphere; }
    return RT_OK;
}

} // namespace

extern "C" {

int rtTraceOcclusion(RtContext* c, const RtRaySegment* segs, int n, uint8_t* occluded, int flags)
{
    if (!c) return RT_E_INVALID;
    const int rc = traceChecks(c, "rtTraceOcclusion", segs, occluded, n, flags);
    if (rc != RT_OK || n == 0) return rc;
    return occlusionAll(c, segs, n, occluded, flags, false);
}

int rtTraceOcclusionDevice(RtContext* c, const void*, void*, int, int) { return c ? fail(c, RT_E_STATE, "oracle: no device memory") : RT_E_INVALID; }

/* Test hook: the full tMax-initialised loop without an exit (RtStats untouched), to compare with rtTraceOcclusion's early exit. */
int orTraceOcclusionFull(RtContext* c, const RtRaySegment* segs, int n, uint8_t* occluded, int flags)
{
    if (!c) return RT_E_INVALID;
    const int rc = traceChecks(c, "orTraceOcclusionFull", segs, occluded, n, flags);
    if (rc != RT_OK || n == 0) return rc;
    return occlusionAll(c, segs, n, occluded, flags, true);
}

} // extern "C"
