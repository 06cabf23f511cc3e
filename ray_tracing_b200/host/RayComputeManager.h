// RayComputeManager.h — C++ host side above the C-ABI, mirroring the reference's C# MonoBehaviour
// Assets/Scripts/Tracer/RayComputeManager.cs (same public field names, ResetAccumulatedRender(),
// RenderFrame(), the same per-frame call sequence InitFrame -> InitTexturesAndBuffers / InitBVH /
// UpdateModels / UpdateCameraParams / SetShaderParams -> Dispatch).  The reference's toolchain (C# / Unity)
// does not exist in this image, so the host is C++; the C# P/Invoke version of the same class is shipped as
// source in INTEGRATION.md.  Unity engine objects the manager pulls from the scene (Screen, Camera.main,
// FindObjectsByType<Model>) are explicit members here.
//
// The manager talks to an implementation of include/rt_b200.h loaded at run time (RtApi): the product
// passes librt_b200.so; tests may pass the CPU oracle, which exports the same ABI.
#pragma once
#include "BVH.h"
#include "rt_b200.h"

#include <map>
#include <memory>
#include <string>
#include <vector>

namespace Seb {

struct Matrix4x4 { float m[16]; };            // column-major, like UnityEngine.Matrix4x4
struct Color { float r, g, b, a; };
struct Vector4 { float x, y, z, w; };

struct Mesh                                     // UnityEngine.Mesh: vertices / triangles / normals
{
    std::vector<Vector3> vertices;
    std::vector<int> triangles;
    std::vector<Vector3> normals;
};

struct Transform { Matrix4x4 localToWorldMatrix, worldToLocalMatrix; };

struct Model                                    // Assets/Scripts/Types/Model.cs: material + mesh + transform
{
    RtMaterial material;
    std::shared_ptr<Mesh> mesh;
    Transform transform;
    bool logBVHStats = false;
};

struct Camera { float fieldOfView = 60.0f; float aspect = 1.0f; Transform transform; };
struct ScreenInfo { int width = 0, height = 0; };

// Function table of the C-ABI, resolved with dlsym from the library given to the manager.
struct RtApi
{
    void* dl = nullptr;
    decltype(&rtCreate) Create = nullptr; decltype(&rtDestroy) Destroy = nullptr; decltype(&rtLastError) LastError = nullptr;
    decltype(&rtSetBuffer) SetBuffer = nullptr; decltype(&rtSetInt) SetInt = nullptr; decltype(&rtSetInts) SetInts = nullptr;
    decltype(&rtSetFloat) SetFloat = nullptr; decltype(&rtSetVector) SetVector = nullptr; decltype(&rtSetMatrix) SetMatrix = nullptr;
    decltype(&rtSetBool) SetBool = nullptr; decltype(&rtResize) Resize = nullptr; decltype(&rtDispatch) Dispatch = nullptr;
    decltype(&rtReadback) Readback = nullptr; decltype(&rtSynchronize) Synchronize = nullptr;
    decltype(&rtBuildBVH) BuildBVH = nullptr;   // optional: absent from older builds of the library
    decltype(&rtReadbackAsync) ReadbackAsync = nullptr; decltype(&rtReadbackWait) ReadbackWait = nullptr;   // optional: pipelined readback
    decltype(&rtCreateMulti) CreateMulti = nullptr;   // optional: several GPUs behind one context (the all-gather of tiles inside rtDispatch)
    decltype(&rtReadbackPixelStats) ReadbackPixelStats = nullptr; decltype(&rtDisplayPixelStats) DisplayPixelStats = nullptr;   // optional: debug view
    decltype(&rtDispatchFrames) DispatchFrames = nullptr;   // optional: several accumulated frames in one launch (RenderFrames)
    decltype(&rtTraceRays) TraceRays = nullptr;             // optional: closest-hit queries (TraceRays / Pick)
    decltype(&rtTraceOcclusion) TraceOcclusion = nullptr;   // optional: occlusion queries (TraceOcclusion)
    decltype(&rtTracePaths) TracePaths = nullptr;           // optional: radiance along caller rays (TracePaths)
    decltype(&rtBakeProbes) BakeProbesFn = nullptr;         // optional: light probes (BakeProbes)
    decltype(&rtBakeCubemaps) BakeCubemapsFn = nullptr;     // optional: reflection probes (BakeCubemaps)
    decltype(&rtBakeLightmap) BakeLightmapFn = nullptr;     // optional: lightmaps (BakeLightmap)
    decltype(&rtDispatchFeatures) DispatchFeatures = nullptr;   // optional: first-hit feature images (RenderFeatures)
    decltype(&rtCameraRays) CameraRaysFn = nullptr;         // optional: the camera's own rays (CameraRays)
    decltype(&rtDenoise) DenoiseFn = nullptr;               // optional: the a-trous denoiser (Denoise)
    decltype(&rtDenoiseTemporal) DenoiseTemporalFn = nullptr;  // optional: the temporal denoiser (DenoiseTemporal)
    decltype(&rtDispatchAdaptive) DispatchAdaptiveFn = nullptr;  // optional: adaptive sampling (RenderFrameAdaptive)
    decltype(&rtDisplayMean) DisplayMeanFn = nullptr;       // optional: the per-pixel mean on screen (DisplayMean)
    std::string Load(const char* path);        // returns "" on success, else the error text
    void Unload();
};

class RayComputeManager
{
public:
    // [Header("Main Settings")]                                             RayComputeManager.cs:9-19
    bool rayTracingEnabled = true;
    bool accumulate = true;
    BVH::Quality bvhQuality = BVH::Quality::High;
    bool buildBVHOnDevice = false;              // not in the reference: build each mesh's BVH with rtBuildBVH (same buffers) instead of on the host
    int maxBounceCount = 4;
    int numRaysPerPixel = 1;
    float defocusStrength = 0;
    float divergeStrength = 0.3f;
    float focusDistance = 1;

    // [Header("Sky Settings")]                                              :21-27
    bool useSky = false;
    float sunFocus = 500;
    float sunIntensity = 10;
    Color sunColor = {1, 1, 1, 1};
    bool hasSunTransform = false;               // sunTransform == null -> dirToSun = Vector3.down (:176)
    Vector3 sunForward = {0, 0, 1};

    // [Header("Debug Settings")] / [Header("Info")]                         :29-42
    Vector4 debugParams = {0, 0, 0, 0};
    int numAccumulatedFrames = 0;
    int renderSeed = 0;
    bool randomizeSeedOnEnable = false;         // the reference always draws a fresh seed in OnEnable (:64); tests pin it

    // scene objects the reference finds through Unity
    ScreenInfo Screen;
    Camera mainCamera;
    std::vector<Model> models;                  // in the order FindObjectsByType(..., InstanceID) would return them (:118)
    std::vector<RtSphere> spheres;              // extension: analytic spheres (north-star Sphere buffer)

    // results of the last BVH build (for logging / tests)
    std::vector<BVH::BuildStats> bvhStats;
    std::string lastError;

    RayComputeManager(const char* backendLibrary, int device);
    // the same manager on several GPUs of this process: the image is row-tiled over `devices`, rtDispatch ends with one NCCL
    // all-gather of the frame's tiles (rtCreateMulti); nothing else in the call sequence changes
    RayComputeManager(const char* backendLibrary, const int* devices, int deviceCount);
    ~RayComputeManager();
    bool IsRendering() const { return rayTracingEnabled; }                  // :55 (Application.isPlaying is implied)

    int OnEnable();                              // :61-67
    int ResetAccumulatedRender();                // :69-76
    int Update() { return RenderFrame(); }       // :78-82 (HandleInput is UI, out of scope)
    int RenderFrame();                           // :84-95
    // not in the reference: n RenderFrame() calls of a still image in one batch (rtDispatchFrames) — InitFrame, one launch of frames
    // numAccumulatedFrames .. + n - 1, numAccumulatedFrames += n.  With accumulate off, n RenderFrame() calls.
    int RenderFrames(int n);
    // not in the reference: the next frame only where the estimated error is still above `threshold` (rtDispatchAdaptive over the
    // whole image): the upload sequence and InitFrame of RenderFrame, then the adaptive dispatch, numAccumulatedFrames++.
    // *activePixels (may be NULL) receives the number of pixels traced; 0 = converged.  Needs accumulate.  The defaults are capi.py's,
    // chosen by the quality sweep of DESIGN.md section 7d.  DisplayMean: rtDisplayMean, the per-pixel mean as RGBA8.
    int RenderFrameAdaptive(float threshold = 0.2f, int minFrames = 8, int maxFrames = 64, int64_t* activePixels = nullptr);
    int DisplayMean(uint8_t* dst, size_t bytes);
    int OnDestroy();                             // :238-247
    void InvalidateBVH() { hasBVH = false; }     // meshes changed: rebuild on the next frame

    // readback of the two render textures (raytraceFrameTex / accumulatedResult, :53-54)
    int ReadFrame(float* dst, size_t bytes);
    int ReadAccumulated(float* dst, size_t bytes);
    int ReadAccumulatedAsync(float* dst, size_t bytes);      // returns at once; dst is valid after WaitReadback()
    int WaitReadback();
    // the reference's debug view (HL:24-26): per-pixel traversal counters of the counting launches (rtSetOption "countStats" = 1) and
    // their heat map (visMode 1 box tests / ray, 2 triangle tests / ray, 3 sphere tests / ray, 4 rays; debugVisScale = full white)
    int ReadPixelStats(RtPixelStats* dst, size_t bytes);
    int DisplayDebugView(int visMode, float debugVisScale, uint8_t* dst, size_t bytes);
    // not in the reference: the closest hit of caller-supplied rays against the current scene (rtTraceRays; flags RT_TRACE_NO_CULL).
    // The scene is uploaded first as a frame would upload it; the render textures are not touched.
    int TraceRays(const RtRay* rays, int n, RtRayHit* hits, int flags = 0);
    // not in the reference: whether anything lies on caller-supplied segments (rtTraceOcclusion; occluded[i] = 1 or 0) — shadow rays,
    // ambient occlusion, line of sight.  The scene is uploaded first as for TraceRays.
    int TraceOcclusion(const RtRaySegment* segs, int n, uint8_t* occluded, int flags = 0);
    // not in the reference: the path tracer's radiance along caller-supplied rays, the mean of `samples` paths on each ray's RNG chain
    // (rtTracePaths) — custom cameras, probe baking.  The scene is uploaded first as for TraceRays.
    int TracePaths(const RtPathRay* rays, int n, int samples, RtPathRadiance* out);
    // not in the reference: light probes — the L2 spherical harmonics of the radiance arriving at each of n positions (n x 3 floats)
    // from `samples` spherical Fibonacci directions (rtBakeProbes).  The scene is uploaded first as for TraceRays.
    int BakeProbes(const float* positions, int n, int samples, uint32_t seed, RtProbeSH* out);
    // not in the reference: reflection probes — an HDR cube map of the radiance at each of n positions, 6 faces of faceSize^2 texels,
    // each texel the mean of `samples` paths over its area (rtBakeCubemaps).  The scene is uploaded first as for TraceRays.
    int BakeCubemaps(const float* positions, int n, int faceSize, int samples, uint32_t seed, RtCubeTexel* out);
    // not in the reference: lightmaps — the cosine-weighted lighting arriving at each of n surface texels (position, normal), each the
    // mean of `samples` paths over the normal's hemisphere (rtBakeLightmap).  The scene is uploaded first as for TraceRays.
    int BakeLightmap(const RtSurfacePoint* points, int n, int samples, uint32_t seed, RtCubeTexel* out);
    // not in the reference: the denoiser guides of the frame the NEXT RenderFrame() renders (rtDispatchFeatures over the whole image):
    // the upload sequence of RenderFrame, Frame = numAccumulatedFrames, and no step of the frame counter.  Call it right before that
    // RenderFrame; ResetAccumulatedRender resets the accumulated guides with the colour.
    // ReadFeatureImage: "FeatureFrame" (W*H RtPixelFeatures), "AccumulatedAlbedo" or "AccumulatedNormal" (W*H float4).
    int RenderFeatures();
    int ReadFeatureImage(const char* name, void* dst, size_t bytes);
    // not in the reference: the jittered camera ray of every pixel for that same frame and the RNG state after its four draws
    // (rtCameraRays; W*H records, [y][x]): what TracePaths and TraceRays take.
    int CameraRays(RtPathRay* rays, size_t bytes);
    // not in the reference: the a-trous denoiser (rtDenoise) over the whole image, guided by the feature images of RenderFeatures():
    // the accumulated mean when accumulate is on, else the last frame.  The defaults are capi.py's, chosen by the quality sweep of
    // DESIGN.md section 7d.  ReadDenoised: "DenoisedRender", W*H float4, the denoised mean colour.
    int Denoise(int iterations = 5, float sigmaColour = 64.0f, float sigmaNormal = 1.0f, float sigmaDepth = 0.1f);
    // not in the reference: the temporal denoiser (rtDenoiseTemporal, SVGF) of the last frame, for a moving camera: call it once per
    // frame after RenderFeatures() and RenderFrame(); resetHistory = 1 on a jump cut.  The defaults are capi.py's, chosen by the
    // quality sweep of DESIGN.md section 7d.  The result is read with ReadDenoised.
    int DenoiseTemporal(int iterations = 5, float sigmaLuminance = 8.0f, float sigmaNormal = 1.0f, float sigmaDepth = 0.1f, float alpha = 0.1f,
                        int resetHistory = 0);
    int ReadDenoised(float* dst, size_t bytes);
    // picking / autofocus: the un-jittered camera ray through pixel (x, y) of the screen — SetupPixel's operations (HL:547-558) on the
    // manager's own camera fields — and its closest hit
    void PickRay(float x, float y, RtRay* ray) const;
    int Pick(float x, float y, RtRayHit* hit);
    RtContext* Context() const { return ctx; }
    const RtApi& Api() const { return api; }

private:
    struct MeshDataLists { std::vector<RtTriangle> triangles; std::vector<RtNode> nodes; std::vector<RtModel> meshInfo; };   // :249-254

    RtApi api;
    RtContext* ctx = nullptr;
    std::vector<RtModel> meshInfo;               // :49
    bool hasBVH = false;                         // :51
    int texWidth = 0, texHeight = 0;

    int InitFrame();                             // :115-124
    int InitTexturesAndBuffers();                // :126-141
    int InitBVH();                               // :143-161
    int SetShaderParams();                       // :163-181
    int UpdateCameraParams(const Camera& cam);   // :183-190
    int UpdateModels();                          // :192-204
    MeshDataLists CreateAllMeshData();           // :206-236
    int Check(int rc, const char* what);
};

} // namespace Seb
