// host_capi.cpp — flat C entry points over the C++ host classes (BVH, RayComputeManager) so that
// Python (ctypes) tests, bench.py and other FFI hosts can drive them.  No arithmetic of the path here.
#include "RayComputeManager.h"

#include <cstring>
#include <exception>
#include <string>

using namespace Seb;

namespace {
struct Handle
{
    RayComputeManager* mgr = nullptr;
    std::vector<std::shared_ptr<Mesh>> meshes;
    std::string err;
};
thread_local std::string g_err;
}

#define GUARD(h) if (!(h) || !(h)->mgr) return RT_E_INVALID
#define CATCH_ALL(h) catch (const std::exception& e) { (h)->err = e.what(); (h)->mgr->lastError = e.what(); return RT_E_INVALID; }

extern "C" {

/* ---- BVH builder -------------------------------------------------------------------------------------------------------- */

/* Builds the BVH of one mesh.  outNodes must hold 2*triCount+1 entries, outTris triCount entries.
 * stats (optional) receives 9 ints: TimeMs, TriangleCount, TotalNodeCount, LeafNodeCount, LeafDepthMin, LeafDepthMax,
 * LeafDepthSum, LeafMinTriCount, LeafMaxTriCount.  Returns the node count, or a negative RT_E_* code. */
int rthBuildBVH(const float* verts, int vertCount, const int* indices, int indexCount, const float* normals, int quality,
                RtTriangle* outTris, RtNode* outNodes, int nodeCapacity, int* stats)
{
    try
    {
        if (quality < 0 || quality > 2) { g_err = "quality must be 0 (Low), 1 (High) or 2 (Disabled)"; return RT_E_INVALID; }
        BVH bvh(reinterpret_cast<const Vector3*>(verts), vertCount, indices, indexCount, reinterpret_cast<const Vector3*>(normals),
                (BVH::Quality)quality);
        if ((int)bvh.Nodes.size() > nodeCapacity) { g_err = "node capacity too small"; return RT_E_INVALID; }
        memcpy(outTris, bvh.Triangles.data(), bvh.Triangles.size() * sizeof(RtTriangle));
        memcpy(outNodes, bvh.Nodes.data(), bvh.Nodes.size() * sizeof(RtNode));
        if (stats)
        {
            const BVH::BuildStats& s = bvh.stats;
            const int v[9] = {s.TimeMs, s.TriangleCount, s.TotalNodeCount, s.LeafNodeCount, s.LeafDepthMin, s.LeafDepthMax,
                              s.LeafDepthSum, s.LeafMinTriCount, s.LeafMaxTriCount};
            memcpy(stats, v, sizeof(v));
        }
        return (int)bvh.Nodes.size();
    }
    catch (const std::exception& e) { g_err = e.what(); return RT_E_INVALID; }
}

/* Host threads a BVH build may use: 0 = all hardware threads (default), 1 = single-threaded like the reference.  The built
 * buffers do not depend on it.  Returns the previous value. */
int rthSetBuildThreads(int threads) { const int old = BVH::BuildThreads; BVH::BuildThreads = threads < 0 ? 0 : threads; return old; }

const char* rthLastError(void) { return g_err.c_str(); }

/* ---- RayComputeManager ------------------------------------------------------------------------------------------------------ */

int rcmCreate(const char* backendLibrary, int device, void** out)
{
    if (!backendLibrary || !out) { g_err = "rcmCreate: bad argument"; return RT_E_INVALID; }
    Handle* h = new Handle();
    h->mgr = new RayComputeManager(backendLibrary, device);
    if (!h->mgr->Context())
    {
        g_err = h->mgr->lastError;
        delete h->mgr; delete h;
        *out = nullptr;
        return RT_E_NO_DEVICE;
    }
    *out = h;
    return RT_OK;
}

int rcmCreateMulti(const char* backendLibrary, const int* devices, int deviceCount, void** out)
{
    if (!backendLibrary || !out || deviceCount < 1) { g_err = "rcmCreateMulti: bad argument"; return RT_E_INVALID; }
    Handle* h = new Handle();
    h->mgr = new RayComputeManager(backendLibrary, devices, deviceCount);
    if (!h->mgr->Context())
    {
        g_err = h->mgr->lastError;
        delete h->mgr; delete h;
        *out = nullptr;
        return RT_E_NO_DEVICE;
    }
    *out = h;
    return RT_OK;
}

int rcmDestroy(void* hv) { Handle* h = (Handle*)hv; if (!h) return RT_E_INVALID; delete h->mgr; delete h; return RT_OK; }

const char* rcmLastError(void* hv) { Handle* h = (Handle*)hv; return h && h->mgr ? h->mgr->lastError.c_str() : g_err.c_str(); }

void* rcmContext(void* hv) { Handle* h = (Handle*)hv; return h && h->mgr ? (void*)h->mgr->Context() : nullptr; }

/* public fields by name (the inspector fields of RayComputeManager.cs:9-42) */
int rcmSetInt(void* hv, const char* field, int v)
{
    Handle* h = (Handle*)hv; GUARD(h);
    RayComputeManager& m = *h->mgr;
    const std::string f(field);
    if (f == "maxBounceCount") m.maxBounceCount = v;
    else if (f == "numRaysPerPixel") m.numRaysPerPixel = v;
    else if (f == "renderSeed") m.renderSeed = v;
    else if (f == "numAccumulatedFrames") m.numAccumulatedFrames = v;
    else if (f == "bvhQuality") { if (v < 0 || v > 2) return RT_E_INVALID; m.bvhQuality = (BVH::Quality)v; }
    else if (f == "rayTracingEnabled") m.rayTracingEnabled = v != 0;
    else if (f == "buildBVHOnDevice") m.buildBVHOnDevice = v != 0;
    else if (f == "accumulate") m.accumulate = v != 0;
    else if (f == "useSky") m.useSky = v != 0;
    else if (f == "randomizeSeedOnEnable") m.randomizeSeedOnEnable = v != 0;
    else { m.lastError = "unknown int field " + f; return RT_E_UNKNOWN_NAME; }
    return RT_OK;
}

int rcmGetInt(void* hv, const char* field, int* out)
{
    Handle* h = (Handle*)hv; GUARD(h);
    RayComputeManager& m = *h->mgr;
    const std::string f(field);
    if (f == "maxBounceCount") *out = m.maxBounceCount;
    else if (f == "numRaysPerPixel") *out = m.numRaysPerPixel;
    else if (f == "renderSeed") *out = m.renderSeed;
    else if (f == "numAccumulatedFrames") *out = m.numAccumulatedFrames;
    else if (f == "bvhQuality") *out = (int)m.bvhQuality;
    else if (f == "accumulate") *out = m.accumulate;
    else if (f == "buildBVHOnDevice") *out = m.buildBVHOnDevice;
    else if (f == "useSky") *out = m.useSky;
    else { m.lastError = "unknown int field " + f; return RT_E_UNKNOWN_NAME; }
    return RT_OK;
}

int rcmSetFloat(void* hv, const char* field, float v)
{
    Handle* h = (Handle*)hv; GUARD(h);
    RayComputeManager& m = *h->mgr;
    const std::string f(field);
    if (f == "defocusStrength") m.defocusStrength = v;
    else if (f == "divergeStrength") m.divergeStrength = v;
    else if (f == "focusDistance") m.focusDistance = v;
    else if (f == "sunFocus") m.sunFocus = v;
    else if (f == "sunIntensity") m.sunIntensity = v;
    else { m.lastError = "unknown float field " + f; return RT_E_UNKNOWN_NAME; }
    return RT_OK;
}

int rcmSetSun(void* hv, const float color[4], const float* forward /* NULL = no sunTransform */)
{
    Handle* h = (Handle*)hv; GUARD(h);
    RayComputeManager& m = *h->mgr;
    if (color) m.sunColor = Color{color[0], color[1], color[2], color[3]};
    m.hasSunTransform = forward != nullptr;
    if (forward) m.sunForward = Vector3{forward[0], forward[1], forward[2]};
    return RT_OK;
}

int rcmSetScreen(void* hv, int width, int height)
{
    Handle* h = (Handle*)hv; GUARD(h);
    h->mgr->Screen.width = width; h->mgr->Screen.height = height;
    h->mgr->mainCamera.aspect = (float)width / (float)height;         // Camera.aspect follows the screen
    return RT_OK;
}

int rcmSetCamera(void* hv, float fieldOfView, const float localToWorld[16])
{
    Handle* h = (Handle*)hv; GUARD(h);
    h->mgr->mainCamera.fieldOfView = fieldOfView;
    memcpy(h->mgr->mainCamera.transform.localToWorldMatrix.m, localToWorld, 64);
    return RT_OK;
}

int rcmAddMesh(void* hv, const float* verts, int vertCount, const int* indices, int indexCount, const float* normals)
{
    Handle* h = (Handle*)hv; GUARD(h);
    if (!verts || !indices || !normals || vertCount <= 0 || indexCount <= 0) return RT_E_INVALID;
    auto mesh = std::make_shared<Mesh>();
    mesh->vertices.assign(reinterpret_cast<const Vector3*>(verts), reinterpret_cast<const Vector3*>(verts) + vertCount);
    mesh->normals.assign(reinterpret_cast<const Vector3*>(normals), reinterpret_cast<const Vector3*>(normals) + vertCount);
    mesh->triangles.assign(indices, indices + indexCount);
    h->meshes.push_back(mesh);
    return (int)h->meshes.size() - 1;
}

int rcmAddModel(void* hv, int meshId, const float localToWorld[16], const float worldToLocal[16], const RtMaterial* material)
{
    Handle* h = (Handle*)hv; GUARD(h);
    if (meshId < 0 || meshId >= (int)h->meshes.size() || !localToWorld || !worldToLocal || !material) return RT_E_INVALID;
    Model m;
    m.mesh = h->meshes[meshId];
    memcpy(m.transform.localToWorldMatrix.m, localToWorld, 64);
    memcpy(m.transform.worldToLocalMatrix.m, worldToLocal, 64);
    m.material = *material;
    h->mgr->models.push_back(m);
    h->mgr->InvalidateBVH();
    return (int)h->mgr->models.size() - 1;
}

int rcmSetModelTransform(void* hv, int model, const float localToWorld[16], const float worldToLocal[16])
{
    Handle* h = (Handle*)hv; GUARD(h);
    if (model < 0 || model >= (int)h->mgr->models.size()) return RT_E_INVALID;
    memcpy(h->mgr->models[model].transform.localToWorldMatrix.m, localToWorld, 64);
    memcpy(h->mgr->models[model].transform.worldToLocalMatrix.m, worldToLocal, 64);
    return RT_OK;
}

int rcmSetModelMaterial(void* hv, int model, const RtMaterial* material)
{
    Handle* h = (Handle*)hv; GUARD(h);
    if (model < 0 || model >= (int)h->mgr->models.size() || !material) return RT_E_INVALID;
    h->mgr->models[model].material = *material;
    return RT_OK;
}

int rcmSetSpheres(void* hv, const RtSphere* spheres, int count)
{
    Handle* h = (Handle*)hv; GUARD(h);
    if (count < 0 || (count > 0 && !spheres)) return RT_E_INVALID;
    h->mgr->spheres.assign(spheres, spheres + count);
    return RT_OK;
}

int rcmOnEnable(void* hv) { Handle* h = (Handle*)hv; GUARD(h); try { return h->mgr->OnEnable(); } CATCH_ALL(h) }
int rcmResetAccumulatedRender(void* hv) { Handle* h = (Handle*)hv; GUARD(h); try { return h->mgr->ResetAccumulatedRender(); } CATCH_ALL(h) }
int rcmRenderFrame(void* hv) { Handle* h = (Handle*)hv; GUARD(h); try { return h->mgr->RenderFrame(); } CATCH_ALL(h) }
int rcmRenderFrames(void* hv, int n) { Handle* h = (Handle*)hv; GUARD(h); try { return h->mgr->RenderFrames(n); } CATCH_ALL(h) }
int rcmRenderFrameAdaptive(void* hv, float threshold, int minFrames, int maxFrames, int64_t* activePixels)
{ Handle* h = (Handle*)hv; GUARD(h); try { return h->mgr->RenderFrameAdaptive(threshold, minFrames, maxFrames, activePixels); } CATCH_ALL(h) }
int rcmDisplayMean(void* hv, uint8_t* dst, size_t bytes) { Handle* h = (Handle*)hv; GUARD(h); return h->mgr->DisplayMean(dst, bytes); }
int rcmReadFrame(void* hv, float* dst, size_t bytes) { Handle* h = (Handle*)hv; GUARD(h); return h->mgr->ReadFrame(dst, bytes); }
int rcmReadAccumulated(void* hv, float* dst, size_t bytes) { Handle* h = (Handle*)hv; GUARD(h); return h->mgr->ReadAccumulated(dst, bytes); }
int rcmReadPixelStats(void* hv, RtPixelStats* dst, size_t bytes) { Handle* h = (Handle*)hv; GUARD(h); return h->mgr->ReadPixelStats(dst, bytes); }
int rcmDisplayDebugView(void* hv, int visMode, float debugVisScale, uint8_t* dst, size_t bytes)
{ Handle* h = (Handle*)hv; GUARD(h); return h->mgr->DisplayDebugView(visMode, debugVisScale, dst, bytes); }
int rcmTraceRays(void* hv, const RtRay* rays, int n, RtRayHit* hits, int flags)
{ Handle* h = (Handle*)hv; GUARD(h); try { return h->mgr->TraceRays(rays, n, hits, flags); } CATCH_ALL(h) }

int rcmTraceOcclusion(void* hv, const RtRaySegment* segs, int n, uint8_t* occluded, int flags)
{ Handle* h = (Handle*)hv; GUARD(h); try { return h->mgr->TraceOcclusion(segs, n, occluded, flags); } CATCH_ALL(h) }

int rcmTracePaths(void* hv, const RtPathRay* rays, int n, int samples, RtPathRadiance* out)
{ Handle* h = (Handle*)hv; GUARD(h); try { return h->mgr->TracePaths(rays, n, samples, out); } CATCH_ALL(h) }

int rcmBakeProbes(void* hv, const float* positions, int n, int samples, uint32_t seed, RtProbeSH* out)
{ Handle* h = (Handle*)hv; GUARD(h); try { return h->mgr->BakeProbes(positions, n, samples, seed, out); } CATCH_ALL(h) }

int rcmBakeCubemaps(void* hv, const float* positions, int n, int faceSize, int samples, uint32_t seed, RtCubeTexel* out)
{ Handle* h = (Handle*)hv; GUARD(h); try { return h->mgr->BakeCubemaps(positions, n, faceSize, samples, seed, out); } CATCH_ALL(h) }

int rcmBakeLightmap(void* hv, const RtSurfacePoint* points, int n, int samples, uint32_t seed, RtCubeTexel* out)
{ Handle* h = (Handle*)hv; GUARD(h); try { return h->mgr->BakeLightmap(points, n, samples, seed, out); } CATCH_ALL(h) }

int rcmRenderFeatures(void* hv) { Handle* h = (Handle*)hv; GUARD(h); try { return h->mgr->RenderFeatures(); } CATCH_ALL(h) }
int rcmReadFeatureImage(void* hv, const char* name, void* dst, size_t bytes) { Handle* h = (Handle*)hv; GUARD(h); return h->mgr->ReadFeatureImage(name, dst, bytes); }
int rcmCameraRays(void* hv, RtPathRay* rays, size_t bytes) { Handle* h = (Handle*)hv; GUARD(h); try { return h->mgr->CameraRays(rays, bytes); } CATCH_ALL(h) }
int rcmDenoise(void* hv, int iterations, float sigmaColour, float sigmaNormal, float sigmaDepth)
{ Handle* h = (Handle*)hv; GUARD(h); try { return h->mgr->Denoise(iterations, sigmaColour, sigmaNormal, sigmaDepth); } CATCH_ALL(h) }
int rcmDenoiseTemporal(void* hv, int iterations, float sigmaLuminance, float sigmaNormal, float sigmaDepth, float alpha, int resetHistory)
{ Handle* h = (Handle*)hv; GUARD(h); try { return h->mgr->DenoiseTemporal(iterations, sigmaLuminance, sigmaNormal, sigmaDepth, alpha, resetHistory); } CATCH_ALL(h) }
int rcmReadDenoised(void* hv, float* dst, size_t bytes) { Handle* h = (Handle*)hv; GUARD(h); return h->mgr->ReadDenoised(dst, bytes); }
/* the pick ray through pixel (x, y) into *ray (may be NULL) and its closest hit into *hit (may be NULL: the ray alone) */
int rcmPick(void* hv, float x, float y, RtRay* ray, RtRayHit* hit)
{
    Handle* h = (Handle*)hv; GUARD(h);
    if (ray) h->mgr->PickRay(x, y, ray);
    if (!hit) return RT_OK;
    try { return h->mgr->Pick(x, y, hit); } CATCH_ALL(h)
}

/* BVH statistics of the last build: writes up to cap entries of 9 ints each (see rthBuildBVH); returns the mesh count */
int rcmGetBVHStats(void* hv, int* out, int cap)
{
    Handle* h = (Handle*)hv; GUARD(h);
    const auto& v = h->mgr->bvhStats;
    for (int i = 0; i < (int)v.size() && i < cap; i++)
    {
        const BVH::BuildStats& s = v[i];
        const int vals[9] = {s.TimeMs, s.TriangleCount, s.TotalNodeCount, s.LeafNodeCount, s.LeafDepthMin, s.LeafDepthMax,
                             s.LeafDepthSum, s.LeafMinTriCount, s.LeafMaxTriCount};
        memcpy(out + 9 * i, vals, sizeof(vals));
    }
    return (int)v.size();
}

} // extern "C"
