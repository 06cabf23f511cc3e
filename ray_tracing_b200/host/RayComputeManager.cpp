// RayComputeManager.cpp — see RayComputeManager.h.  Call sequence per frame follows
// Assets/Scripts/Tracer/RayComputeManager.cs:61-236 of the reference; every ComputeShader / ComputeHelper
// call there becomes the C-ABI call that replaces it (include/rt_b200.h).
#include "RayComputeManager.h"

#include <cmath>
#include <cstring>
#include <dlfcn.h>
#include <random>
#include <stdexcept>

namespace Seb {

std::string RtApi::Load(const char* path)
{
    dl = dlopen(path, RTLD_NOW | RTLD_LOCAL);
    if (!dl) return std::string("dlopen failed: ") + dlerror();
#define RESOLVE(field, sym) field = reinterpret_cast<decltype(field)>(dlsym(dl, sym)); if (!field) return std::string("missing symbol ") + sym;
    RESOLVE(Create, "rtCreate") RESOLVE(Destroy, "rtDestroy") RESOLVE(LastError, "rtLastError")
    RESOLVE(SetBuffer, "rtSetBuffer") RESOLVE(SetInt, "rtSetInt") RESOLVE(SetInts, "rtSetInts")
    RESOLVE(SetFloat, "rtSetFloat") RESOLVE(SetVector, "rtSetVector") RESOLVE(SetMatrix, "rtSetMatrix")
    RESOLVE(SetBool, "rtSetBool") RESOLVE(Resize, "rtResize") RESOLVE(Dispatch, "rtDispatch")
    RESOLVE(Readback, "rtReadback") RESOLVE(Synchronize, "rtSynchronize")
#undef RESOLVE
    BuildBVH = reinterpret_cast<decltype(BuildBVH)>(dlsym(dl, "rtBuildBVH"));
    CreateMulti = reinterpret_cast<decltype(CreateMulti)>(dlsym(dl, "rtCreateMulti"));
    ReadbackAsync = reinterpret_cast<decltype(ReadbackAsync)>(dlsym(dl, "rtReadbackAsync"));
    ReadbackWait = reinterpret_cast<decltype(ReadbackWait)>(dlsym(dl, "rtReadbackWait"));
    ReadbackPixelStats = reinterpret_cast<decltype(ReadbackPixelStats)>(dlsym(dl, "rtReadbackPixelStats"));
    DisplayPixelStats = reinterpret_cast<decltype(DisplayPixelStats)>(dlsym(dl, "rtDisplayPixelStats"));
    DispatchFrames = reinterpret_cast<decltype(DispatchFrames)>(dlsym(dl, "rtDispatchFrames"));
    TraceRays = reinterpret_cast<decltype(TraceRays)>(dlsym(dl, "rtTraceRays"));
    TraceOcclusion = reinterpret_cast<decltype(TraceOcclusion)>(dlsym(dl, "rtTraceOcclusion"));
    TracePaths = reinterpret_cast<decltype(TracePaths)>(dlsym(dl, "rtTracePaths"));
    BakeProbesFn = reinterpret_cast<decltype(BakeProbesFn)>(dlsym(dl, "rtBakeProbes"));
    BakeCubemapsFn = reinterpret_cast<decltype(BakeCubemapsFn)>(dlsym(dl, "rtBakeCubemaps"));
    BakeLightmapFn = reinterpret_cast<decltype(BakeLightmapFn)>(dlsym(dl, "rtBakeLightmap"));
    DispatchFeatures = reinterpret_cast<decltype(DispatchFeatures)>(dlsym(dl, "rtDispatchFeatures"));
    CameraRaysFn = reinterpret_cast<decltype(CameraRaysFn)>(dlsym(dl, "rtCameraRays"));
    DenoiseFn = reinterpret_cast<decltype(DenoiseFn)>(dlsym(dl, "rtDenoise"));
    DenoiseTemporalFn = reinterpret_cast<decltype(DenoiseTemporalFn)>(dlsym(dl, "rtDenoiseTemporal"));
    DispatchAdaptiveFn = reinterpret_cast<decltype(DispatchAdaptiveFn)>(dlsym(dl, "rtDispatchAdaptive"));
    DisplayMeanFn = reinterpret_cast<decltype(DisplayMeanFn)>(dlsym(dl, "rtDisplayMean"));
    return "";
}

void RtApi::Unload() { if (dl) dlclose(dl); dl = nullptr; }

static const int kernelRayTrace = RT_KERNEL_RAYTRACE;                  // RayComputeManager.cs:57-58
static const int kernelResetAccumulated = RT_KERNEL_RESET_ACCUMULATED;

RayComputeManager::RayComputeManager(const char* backendLibrary, int device)
{
    lastError = api.Load(backendLibrary);
    if (!lastError.empty()) return;
    const int rc = api.Create(&ctx, device);
    if (rc != RT_OK) { lastError = std::string("rtCreate: ") + api.LastError(nullptr); ctx = nullptr; }
}

RayComputeManager::RayComputeManager(const char* backendLibrary, const int* devices, int deviceCount)
{
    lastError = api.Load(backendLibrary);
    if (!lastError.empty()) return;
    if (!api.CreateMulti) { lastError = "the library does not export rtCreateMulti"; return; }
    const int rc = api.CreateMulti(&ctx, devices, deviceCount);
    if (rc != RT_OK) { lastError = std::string("rtCreateMulti: ") + api.LastError(nullptr); ctx = nullptr; }
}

RayComputeManager::~RayComputeManager() { OnDestroy(); api.Unload(); }

int RayComputeManager::Check(int rc, const char* what)
{
    if (rc != RT_OK) lastError = std::string(what) + ": " + (ctx ? api.LastError(ctx) : "no context");
    return rc;
}

#define TRY(expr) do { int rc_ = Check((expr), #expr); if (rc_ != RT_OK) return rc_; } while (0)

int RayComputeManager::OnEnable()
{
    if (!ctx) return RT_E_STATE;
    hasBVH = false;
    if (randomizeSeedOnEnable) { std::random_device rd; renderSeed = (int)(rd() & 0x7fffffffu); }   // new System.Random().Next()
    return ResetAccumulatedRender();
}

int RayComputeManager::ResetAccumulatedRender()
{
    if (!ctx) return RT_E_STATE;
    numAccumulatedFrames = 1;
    int rc = InitFrame();
    if (rc != RT_OK) return rc;
    // ComputeHelper.Dispatch(cs, width, height, kernelIndex) -> ceil(n / 8) groups (ComputeHelper.cs:25-32)
    TRY(api.Dispatch(ctx, kernelResetAccumulated, (texWidth + 7) / 8, (texHeight + 7) / 8, 1));
    return RT_OK;
}

int RayComputeManager::RenderFrame()
{
    if (!ctx) return RT_E_STATE;
    if (!IsRendering()) return RT_OK;
    int rc = InitFrame();
    if (rc != RT_OK) return rc;
    TRY(api.Dispatch(ctx, kernelRayTrace, (texWidth + 7) / 8, (texHeight + 7) / 8, 1));
    if (accumulate) numAccumulatedFrames++;
    return RT_OK;
}

int RayComputeManager::RenderFrames(int n)
{
    if (!ctx) return RT_E_STATE;
    if (n < 1) { lastError = "RenderFrames: n must be >= 1"; return RT_E_INVALID; }
    if (!accumulate)                             // only the last frame would be observable: the frames one by one
    {
        for (int k = 0; k < n; k++) { const int rc = RenderFrame(); if (rc != RT_OK) return rc; }
        return RT_OK;
    }
    if (!IsRendering()) return RT_OK;
    if (!api.DispatchFrames) { lastError = "the library does not export rtDispatchFrames"; return RT_E_STATE; }
    int rc = InitFrame();                        // Frame = numAccumulatedFrames, the batch's first frame
    if (rc != RT_OK) return rc;
    TRY(api.DispatchFrames(ctx, (texWidth + 7) / 8, (texHeight + 7) / 8, 1, n));
    numAccumulatedFrames += n;
    return RT_OK;
}

int RayComputeManager::RenderFrameAdaptive(float threshold, int minFrames, int maxFrames, int64_t* activePixels)
{
    if (activePixels) *activePixels = 0;
    if (!ctx) return RT_E_STATE;
    if (!IsRendering()) return RT_OK;
    if (!api.DispatchAdaptiveFn) { lastError = "the library does not export rtDispatchAdaptive"; return RT_E_STATE; }
    int rc = InitFrame();
    if (rc != RT_OK) return rc;
    TRY(api.DispatchAdaptiveFn(ctx, (texWidth + 7) / 8, (texHeight + 7) / 8, 1, threshold, minFrames, maxFrames, activePixels));
    numAccumulatedFrames++;                      // accumulate is on (the call refuses otherwise)
    return RT_OK;
}

int RayComputeManager::DisplayMean(uint8_t* dst, size_t bytes)
{
    if (!ctx) return RT_E_STATE;
    if (!api.DisplayMeanFn) { lastError = "the library does not export rtDisplayMean"; return RT_E_STATE; }
    TRY(api.DisplayMeanFn(ctx, dst, bytes));
    return RT_OK;
}

int RayComputeManager::InitFrame()
{
    int rc;
    if ((rc = InitTexturesAndBuffers()) != RT_OK) return rc;
    if ((rc = InitBVH()) != RT_OK) return rc;
    if ((rc = UpdateModels()) != RT_OK) return rc;
    if ((rc = UpdateCameraParams(mainCamera)) != RT_OK) return rc;
    return SetShaderParams();
}

int RayComputeManager::InitTexturesAndBuffers()
{
    const int width = Screen.width, height = Screen.height;
    TRY(api.Resize(ctx, width, height));                              // CreateRenderTexture x2 + SetTexture x3
    texWidth = width; texHeight = height;
    const int res[2] = {width, height};
    TRY(api.SetInts(ctx, "Resolution", res, 2));
    const float dbg[4] = {debugParams.x, debugParams.y, debugParams.z, debugParams.w};
    TRY(api.SetVector(ctx, "debugParams", dbg));
    return RT_OK;
}

int RayComputeManager::InitBVH()
{
    if (hasBVH) return RT_OK;
    hasBVH = true;
    MeshDataLists data = CreateAllMeshData();
    meshInfo = data.meshInfo;
    TRY(api.SetBuffer(ctx, "ModelInfo", meshInfo.data(), (int)meshInfo.size(), (int)sizeof(RtModel)));
    TRY(api.SetBuffer(ctx, "Triangles", data.triangles.data(), (int)data.triangles.size(), (int)sizeof(RtTriangle)));
    TRY(api.SetInt(ctx, "triangleCount", (int)data.triangles.size()));
    TRY(api.SetBuffer(ctx, "Nodes", data.nodes.data(), (int)data.nodes.size(), (int)sizeof(RtNode)));
    return RT_OK;
}

int RayComputeManager::SetShaderParams()
{
    TRY(api.SetInt(ctx, "Frame", numAccumulatedFrames));
    TRY(api.SetInt(ctx, "UseSky", useSky ? 1 : 0));
    TRY(api.SetInt(ctx, "MaxBounceCount", maxBounceCount));
    TRY(api.SetInt(ctx, "NumRaysPerPixel", numRaysPerPixel));
    TRY(api.SetFloat(ctx, "DefocusStrength", defocusStrength));
    TRY(api.SetFloat(ctx, "DivergeStrength", divergeStrength));
    TRY(api.SetFloat(ctx, "SunFocus", sunFocus));
    TRY(api.SetFloat(ctx, "SunIntensity", sunIntensity));
    const float sc[4] = {sunColor.r, sunColor.g, sunColor.b, sunColor.a};
    TRY(api.SetVector(ctx, "SunColour", sc));
    float ds[4] = {0.0f, -1.0f, 0.0f, 0.0f};                             // Vector3.down
    if (hasSunTransform) { ds[0] = -sunForward.x; ds[1] = -sunForward.y; ds[2] = -sunForward.z; }
    TRY(api.SetVector(ctx, "dirToSun", ds));
    TRY(api.SetInt(ctx, "renderSeed", renderSeed));
    TRY(api.SetBool(ctx, "accumulate", accumulate ? 1 : 0));
    return RT_OK;
}

int RayComputeManager::UpdateCameraParams(const Camera& cam)
{
    const float Deg2Rad = 0.0174532924f;                                  // Mathf.Deg2Rad
    const float planeHeight = focusDistance * (float)std::tan((double)(cam.fieldOfView * 0.5f * Deg2Rad)) * 2;
    const float planeWidth = planeHeight * cam.aspect;
    const float vp[4] = {planeWidth, planeHeight, focusDistance, 0.0f};
    TRY(api.SetVector(ctx, "ViewParams", vp));
    TRY(api.SetMatrix(ctx, "CamLocalToWorldMatrix", cam.transform.localToWorldMatrix.m));
    return RT_OK;
}

int RayComputeManager::UpdateModels()
{
    if (meshInfo.size() != models.size())
    {
        lastError = "UpdateModels: the model list changed after the BVH was built (call InvalidateBVH)";
        return RT_E_STATE;
    }
    for (size_t i = 0; i < models.size(); i++)
    {
        memcpy(meshInfo[i].worldToLocal, models[i].transform.worldToLocalMatrix.m, 64);
        memcpy(meshInfo[i].localToWorld, models[i].transform.localToWorldMatrix.m, 64);
        meshInfo[i].material = models[i].material;
    }
    TRY(api.SetBuffer(ctx, "ModelInfo", meshInfo.data(), (int)meshInfo.size(), (int)sizeof(RtModel)));
    TRY(api.SetInt(ctx, "modelCount", (int)models.size()));
    // extension: analytic spheres travel with the per-frame model update
    TRY(api.SetBuffer(ctx, "Spheres", spheres.data(), (int)spheres.size(), (int)sizeof(RtSphere)));
    return RT_OK;
}

RayComputeManager::MeshDataLists RayComputeManager::CreateAllMeshData()
{
    MeshDataLists allData;
    std::map<const Mesh*, std::pair<int, int>> meshLookup;                // mesh -> (nodeOffset, triOffset)
    bvhStats.clear();
    for (const Model& model : models)
    {
        const Mesh* mesh = model.mesh.get();
        // Construct BVH if this is the first time seeing the current mesh (otherwise reuse)
        if (!meshLookup.count(mesh))
        {
            meshLookup[mesh] = std::make_pair((int)allData.nodes.size(), (int)allData.triangles.size());
            if (buildBVHOnDevice && api.BuildBVH && ctx)
            {
                // the same Nodes / Triangles, built by the backend (rtBuildBVH); statistics are the host builder's business
                const int triCount = (int)mesh->triangles.size() / 3;
                std::vector<RtTriangle> t((size_t)(triCount > 0 ? triCount : 1));
                std::vector<RtNode> n((size_t)2 * (triCount > 0 ? triCount : 1) + 1);
                int nodeCount = 0;
                const int rc = api.BuildBVH(ctx, &mesh->vertices[0].x, (int)mesh->vertices.size(), mesh->triangles.data(), (int)mesh->triangles.size(),
                                            &mesh->normals[0].x, (int)bvhQuality, t.data(), n.data(), (int)n.size(), &nodeCount);
                if (rc != RT_OK) throw std::runtime_error(std::string("rtBuildBVH: ") + api.LastError(ctx));
                BVH::BuildStats st; st.quality = bvhQuality; st.TriangleCount = triCount; st.TotalNodeCount = nodeCount;
                bvhStats.push_back(st);
                allData.triangles.insert(allData.triangles.end(), t.begin(), t.begin() + triCount);
                allData.nodes.insert(allData.nodes.end(), n.begin(), n.begin() + nodeCount);
            }
            else
            {
            BVH bvh(mesh->vertices.data(), (int)mesh->vertices.size(), mesh->triangles.data(), (int)mesh->triangles.size(),
                    mesh->normals.data(), bvhQuality);
            bvhStats.push_back(bvh.stats);
            allData.triangles.insert(allData.triangles.end(), bvh.Triangles.begin(), bvh.Triangles.end());
            allData.nodes.insert(allData.nodes.end(), bvh.Nodes.begin(), bvh.Nodes.end());
            }
        }
        RtModel info;
        memset(&info, 0, sizeof(info));
        info.nodeOffset = meshLookup[mesh].first;
        info.triOffset = meshLookup[mesh].second;
        memcpy(info.worldToLocal, model.transform.worldToLocalMatrix.m, 64);
        info.material = model.material;
        allData.meshInfo.push_back(info);
    }
    return allData;
}

int RayComputeManager::OnDestroy()
{
    if (ctx) { api.Destroy(ctx); ctx = nullptr; }
    return RT_OK;
}

int RayComputeManager::ReadFrame(float* dst, size_t bytes)
{
    if (!ctx) return RT_E_STATE;
    TRY(api.Readback(ctx, "FrameRender", dst, bytes));
    return RT_OK;
}

int RayComputeManager::ReadAccumulated(float* dst, size_t bytes)
{
    if (!ctx) return RT_E_STATE;
    TRY(api.Readback(ctx, "AccumulatedRender", dst, bytes));
    return RT_OK;
}

// Pipelined form for hosts that read every frame (rtReadbackAsync): the copy of this frame's image travels while the next frame renders;
// dst (pinned memory for a real overlap) is valid after WaitReadback().
int RayComputeManager::ReadAccumulatedAsync(float* dst, size_t bytes)
{
    if (!ctx) return RT_E_STATE;
    if (!api.ReadbackAsync) return ReadAccumulated(dst, bytes);
    TRY(api.ReadbackAsync(ctx, "AccumulatedRender", dst, bytes));
    return RT_OK;
}

int RayComputeManager::ReadPixelStats(RtPixelStats* dst, size_t bytes)
{
    if (!ctx) return RT_E_STATE;
    if (!api.ReadbackPixelStats) { lastError = "the library does not export rtReadbackPixelStats"; return RT_E_STATE; }
    TRY(api.ReadbackPixelStats(ctx, dst, bytes));
    return RT_OK;
}

int RayComputeManager::DisplayDebugView(int visMode, float debugVisScale, uint8_t* dst, size_t bytes)
{
    if (!ctx) return RT_E_STATE;
    if (!api.DisplayPixelStats) { lastError = "the library does not export rtDisplayPixelStats"; return RT_E_STATE; }
    TRY(api.DisplayPixelStats(ctx, visMode, debugVisScale, dst, bytes));
    return RT_OK;
}

int RayComputeManager::TraceRays(const RtRay* rays, int n, RtRayHit* hits, int flags)
{
    if (!ctx) return RT_E_STATE;
    if (!api.TraceRays) { lastError = "the library does not export rtTraceRays"; return RT_E_STATE; }
    int rc;
    if ((rc = InitBVH()) != RT_OK || (rc = UpdateModels()) != RT_OK) return rc;
    TRY(api.TraceRays(ctx, rays, n, hits, flags));
    return RT_OK;
}

int RayComputeManager::TraceOcclusion(const RtRaySegment* segs, int n, uint8_t* occluded, int flags)
{
    if (!ctx) return RT_E_STATE;
    if (!api.TraceOcclusion) { lastError = "the library does not export rtTraceOcclusion"; return RT_E_STATE; }
    int rc;
    if ((rc = InitBVH()) != RT_OK || (rc = UpdateModels()) != RT_OK) return rc;
    TRY(api.TraceOcclusion(ctx, segs, n, occluded, flags));
    return RT_OK;
}

int RayComputeManager::TracePaths(const RtPathRay* rays, int n, int samples, RtPathRadiance* out)
{
    if (!ctx) return RT_E_STATE;
    if (!api.TracePaths) { lastError = "the library does not export rtTracePaths"; return RT_E_STATE; }
    int rc;
    if ((rc = InitBVH()) != RT_OK || (rc = UpdateModels()) != RT_OK) return rc;
    TRY(api.TracePaths(ctx, rays, n, samples, out));
    return RT_OK;
}

int RayComputeManager::BakeProbes(const float* positions, int n, int samples, uint32_t seed, RtProbeSH* out)
{
    if (!ctx) return RT_E_STATE;
    if (!api.BakeProbesFn) { lastError = "the library does not export rtBakeProbes"; return RT_E_STATE; }
    int rc;
    if ((rc = InitBVH()) != RT_OK || (rc = UpdateModels()) != RT_OK) return rc;
    TRY(api.BakeProbesFn(ctx, positions, n, samples, seed, out));
    return RT_OK;
}

int RayComputeManager::BakeCubemaps(const float* positions, int n, int faceSize, int samples, uint32_t seed, RtCubeTexel* out)
{
    if (!ctx) return RT_E_STATE;
    if (!api.BakeCubemapsFn) { lastError = "the library does not export rtBakeCubemaps"; return RT_E_STATE; }
    int rc;
    if ((rc = InitBVH()) != RT_OK || (rc = UpdateModels()) != RT_OK) return rc;
    TRY(api.BakeCubemapsFn(ctx, positions, n, faceSize, samples, seed, out));
    return RT_OK;
}

int RayComputeManager::BakeLightmap(const RtSurfacePoint* points, int n, int samples, uint32_t seed, RtCubeTexel* out)
{
    if (!ctx) return RT_E_STATE;
    if (!api.BakeLightmapFn) { lastError = "the library does not export rtBakeLightmap"; return RT_E_STATE; }
    int rc;
    if ((rc = InitBVH()) != RT_OK || (rc = UpdateModels()) != RT_OK) return rc;
    TRY(api.BakeLightmapFn(ctx, points, n, samples, seed, out));
    return RT_OK;
}

int RayComputeManager::RenderFeatures()
{
    if (!ctx) return RT_E_STATE;
    if (!api.DispatchFeatures) { lastError = "the library does not export rtDispatchFeatures"; return RT_E_STATE; }
    if (!IsRendering()) return RT_OK;
    int rc = InitFrame();                        // Frame = numAccumulatedFrames: the frame the next RenderFrame renders
    if (rc != RT_OK) return rc;
    TRY(api.DispatchFeatures(ctx, (texWidth + 7) / 8, (texHeight + 7) / 8, 1));
    return RT_OK;
}

int RayComputeManager::ReadFeatureImage(const char* name, void* dst, size_t bytes)
{
    if (!ctx) return RT_E_STATE;
    TRY(api.Readback(ctx, name, static_cast<float*>(dst), bytes));
    return RT_OK;
}

int RayComputeManager::CameraRays(RtPathRay* rays, size_t bytes)
{
    if (!ctx) return RT_E_STATE;
    if (!api.CameraRaysFn) { lastError = "the library does not export rtCameraRays"; return RT_E_STATE; }
    int rc = InitFrame();
    if (rc != RT_OK) return rc;
    TRY(api.CameraRaysFn(ctx, rays, bytes));
    return RT_OK;
}

int RayComputeManager::Denoise(int iterations, float sigmaColour, float sigmaNormal, float sigmaDepth)
{
    if (!ctx) return RT_E_STATE;
    if (!api.DenoiseFn) { lastError = "the library does not export rtDenoise"; return RT_E_STATE; }
    TRY(api.DenoiseFn(ctx, accumulate ? 1 : 0, iterations, sigmaColour, sigmaNormal, sigmaDepth));
    return RT_OK;
}

int RayComputeManager::DenoiseTemporal(int iterations, float sigmaLuminance, float sigmaNormal, float sigmaDepth, float alpha, int resetHistory)
{
    if (!ctx) return RT_E_STATE;
    if (!api.DenoiseTemporalFn) { lastError = "the library does not export rtDenoiseTemporal"; return RT_E_STATE; }
    TRY(api.DenoiseTemporalFn(ctx, iterations, sigmaLuminance, sigmaNormal, sigmaDepth, alpha, resetHistory));
    return RT_OK;
}

int RayComputeManager::ReadDenoised(float* dst, size_t bytes)
{
    if (!ctx) return RT_E_STATE;
    TRY(api.Readback(ctx, "DenoisedRender", dst, bytes));
    return RT_OK;
}

void RayComputeManager::PickRay(float x, float y, RtRay* ray) const
{
    // ViewParams as UpdateCameraParams computes them; uv, origin and focus point as SetupPixel does (HL:547-558), left to right, unfused
    const float Deg2Rad = 0.0174532924f;
    const float planeHeight = focusDistance * (float)std::tan((double)(mainCamera.fieldOfView * 0.5f * Deg2Rad)) * 2;
    const float planeWidth = planeHeight * mainCamera.aspect;
    const float* M = mainCamera.transform.localToWorldMatrix.m;            // column-major
    const float u = x / ((float)Screen.width - 1.0f), v = y / ((float)Screen.height - 1.0f);
    const float local[3] = {(u - 0.5f) * planeWidth, (v - 0.5f) * planeHeight, 1.0f * focusDistance};
    float o[3], d[3];
    for (int a = 0; a < 3; a++)
    {
        o[a] = ((M[a] * 0.0f + M[4 + a] * 0.0f) + M[8 + a] * 0.0f) + M[12 + a] * 1.0f;
        const float f = ((M[a] * local[0] + M[4 + a] * local[1]) + M[8 + a] * local[2]) + M[12 + a] * 1.0f;
        d[a] = f - o[a];
    }
    const float inv = 1.0f / std::sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]);
    for (int a = 0; a < 3; a++) { ray->origin[a] = o[a]; ray->dir[a] = d[a] * inv; }
}

int RayComputeManager::Pick(float x, float y, RtRayHit* hit)
{
    RtRay ray;
    PickRay(x, y, &ray);
    return TraceRays(&ray, 1, hit, 0);
}

int RayComputeManager::WaitReadback()
{
    if (!ctx) return RT_E_STATE;
    if (!api.ReadbackWait) return RT_OK;
    TRY(api.ReadbackWait(ctx));
    return RT_OK;
}

} // namespace Seb
