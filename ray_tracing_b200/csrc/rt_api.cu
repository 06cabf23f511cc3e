// rt_api.cu — the C-ABI of librt_b200.so (include/rt_b200.h): context, named uniforms, structured
// buffers, render targets, dispatch, readback, multi-GPU tile staging.  Host-side state only; all
// arithmetic of the path lives in rt_device.cuh / rt_kernel_*.cuh.
//
// The interface mirrors the ComputeShader calls RayComputeManager makes (SURVEY.md §8b; each entry point
// cites its reference counterpart in the header).  There is deliberately no CPU path: every entry point
// that needs the GPU fails with RT_E_NO_DEVICE / RT_E_CUDA when CUDA is unavailable.
#include "../../include/rt_b200.h"
#include "rt_kernel_mega.cuh"
#include "rt_kernel_wave.cuh"
#include "rt_kernel_pool.cuh"
#include "rt_kernel_query.cuh"
#include "rt_kernel_features.cuh"
#include "rt_kernel_denoise.cuh"
#include "rt_kernel_temporal.cuh"
#include "rt_kernel_adaptive.cuh"
#include "rt_kernel_probes.cuh"
#include "rt_kernel_cubemaps.cuh"
#include "rt_repack.cuh"
#include "rt_bvh_build.cuh"
#include "rt_comm.cuh"

#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <thread>
#include <type_traits>
#include <utility>
#include <vector>

using namespace rtd;

namespace {

template <class T> struct DevBuf
{
    T* p = nullptr; size_t count = 0, cap = 0;
    cudaError_t ensure(size_t n)
    {
        if (n == count && p) return cudaSuccess;             // unchanged size re-uses the allocation (CH:86-92)
        if (n > cap || n == 0) { if (p) cudaFree(p); p = nullptr; cap = 0; if (n) { cudaError_t e = cudaMalloc(&p, n * sizeof(T)); if (e != cudaSuccess) { count = 0; return e; } cap = n; } }
        count = n; return cudaSuccess;
    }
    void release() { if (p) cudaFree(p); p = nullptr; count = cap = 0; }
};

struct EventPair { cudaEvent_t a, b; };

} // namespace

struct RtContext
{
    int device = 0;
    cudaStream_t ownStream = nullptr, stream = nullptr;
    int numSMs = 0;
    unsigned long long dispatchPixels = 0;     // pixels of the RayTrace dispatch being prepared (this rank's tile): enters the automatic kernel choice
    int dispatchFrames = 1;                    // frames of that dispatch (rtDispatchFrames): a pixel's chain is dispatchFrames * NumRaysPerPixel samples
    std::string err;

    // uniforms (host copy)
    DevParams P;

    // reference-layout buffers
    DevBuf<RtNode> nodes; DevBuf<RtTriangle> tris; DevBuf<RtModel> models; DevBuf<RtSphere> spheres;
    std::vector<RtNode> hNodes; std::vector<RtModel> hModels; std::vector<RtSphere> hSpheres;   // host mirrors for the repack
    // repacked buffers
    RepackState repack;
    bool sceneDirty = true, modelsDirty = true, spheresDirty = true;

    // render targets
    DevBuf<float4> frame, accum, tileSend, tileRecv;
    DevBuf<uchar4> display;
    int width = 0, height = 0;
    int tileRank = 0, tileWorld = 1, bandRows = 1;

    // peers (fused tile exchange): IPC-mapped images of the other ranks
    std::vector<void*> peerBase;               // opened IPC mappings (to close)
    float4* peerFrame[RT_MAX_PEERS]; float4* peerAccum[RT_MAX_PEERS]; int nPeers = 0;

    // options
    int optKernel = -1, optCountStats = 0, optSmemPairs = -1, optPoolSlots = 0, optTailLanes = 16, optSortRays = 0, optForceExt = 0, optModelSkip = 1, optPairOrder = 0, optGridFit = 0, optL2Persist = 0, optTreeletPrefetch = 0, optZeroDefocus = 1, optTlas = -1;
    int l2PersistApplied = 0; const void* l2PersistBase = nullptr; size_t l2PersistBytes = 0;   // kernel -1 = automatic   // smemPairs -1 = automatic

    // exchange of finished tiles inside the ABI (rt_comm.cuh): a communicator over the ranks of a tiled render — one process per
    // GPU (rtCommInit) or several GPUs in this process (rtCreateMulti: this context leads, `followers` render the other tiles)
    NcclApi::Comm comm = nullptr; int commRank = 0, commWorld = 1;
    int optExchange = 1;
    std::vector<RtContext*> followers; RtContext* leader = nullptr;

    // pipelined readback (rtReadbackAsync / rtDisplayAsync): a snapshot on the dispatch stream, the device -> host copy on a stream of
    // its own, so that the next frame's kernel runs while the previous frame's result travels over PCIe
    cudaStream_t copyStream = nullptr; cudaEvent_t snapReady = nullptr, copyDone = nullptr; bool copyPending = false;
    DevBuf<float4> snap;

    // kernel 1 on small tiles: hand-off of a pixel's chain between sample chunks (rt_kernel_wave.cuh)
    DevBuf<unsigned long long> handoff; unsigned int chunkSerial = 0; int optSampleChunks = -1;
    DevBuf<float> poolCold;                    // kernel 2 (RT_POOL_COLD_GLOBAL builds): slot fields of the shade phase, one block per resident warp

    // rtBuildBVH: device arena kept between builds, pinned staging chunks for the copies of caller-owned arrays
    DevBuf<unsigned char> buildArena;
    static constexpr size_t STAGE_BYTES = 16u << 20;
    unsigned char* stageBuf[2] = {nullptr, nullptr}; cudaEvent_t stageEv[2] = {nullptr, nullptr};

    // counters / timing
    unsigned long long* dCounters = nullptr;   // 5
    unsigned int* dWork = nullptr;
    DevBuf<RtPixelStats> pixelStats;           // "PixelStats": W*H per-pixel counters of the counting launches (allocated by the first one)
    DevBuf<RtRay> queryRays; DevBuf<RtRayHit> queryHits;     // rtTraceRays: device copies of one batch (<= RT_TRACE_CHUNK_RAYS) of the caller's host arrays
                                                             // (rtTraceOcclusion: its segments in queryHits, its bytes in queryRays;
                                                             //  rtTracePaths: its RtPathRay in queryHits, its RtPathRadiance in queryRays)
    // rtDispatchFeatures: "FeatureFrame", "AccumulatedAlbedo", "AccumulatedNormal" (W*H each, allocated by the first call);
    // rtCameraRays: the device copy of the image's rays (host form only)
    DevBuf<RtPixelFeatures> featureFrame; DevBuf<float4> accumAlbedo, accumNormal; DevBuf<RtPathRay> cameraRays;
    // rtDenoise: "DenoisedRender" (W*H) and its scratch images (3*W*H: two demodulated colours, the guide), allocated by the first call
    DevBuf<float4> denoised, denoiseScratch;
    // rtDenoiseTemporal: "TemporalFrame" (W*H) and the history (6*W*H: two sets of guide, moments and colour history that alternate
    // between calls, set temporalSet written last), allocated by the first call; the camera of the last call that left a history
    DevBuf<float4> temporalFrame, temporalHist;
    int temporalSet = 0; bool temporalHistory = false;
    float temporalCam[16] = {}, temporalVP[3] = {};
    // rtDispatchAdaptive: "AdaptiveMoments" (W*H, allocated zero-filled by the first traced call), the pixel list (W*H), the selection's
    // scratch (a ballot word per 32 jobs, then the block counts and the list length) and the pinned word the length is read into
    DevBuf<float4> moments; DevBuf<unsigned int> adaptiveList, adaptiveScratch; unsigned int* adaptiveCount = nullptr;
    // rtBakeProbes: the chunk records of one launch (both forms), and the host form's device copies of one launch's positions and results
    DevBuf<float> probeScratch, probePositions; DevBuf<RtProbeSH> probeOut;
    // rtBakeCubemaps: the host form's results of one launch (the positions of the whole call go to probePositions, the records to
    // probeScratch)
    DevBuf<RtCubeTexel> cubeOut;
    std::vector<EventPair> pending, pendingX, freeEvents;
    RtStats stats;
};

static std::string g_createErr = "";

#define CK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return failCuda(c, e_, #call); } while (0)

static int fail(RtContext* c, int code, const std::string& msg) { if (c) c->err = msg; else g_createErr = msg; return code; }
static int failCuda(RtContext* c, cudaError_t e, const char* what)
{
    return fail(c, RT_E_CUDA, std::string(what) + ": " + cudaGetErrorString(e));
}

// The calls that work on one GPU's images only refuse every context of a group (rtCreateMulti); the calls a group makes on all its
// GPUs refuse the contexts it made for its followers
static int refuseGroup(RtContext* c, const char* what)
{
    if (c->leader || !c->followers.empty()) return fail(c, RT_E_STATE, std::string(what) + ": not available on a group context (rtCreateMulti)");
    return RT_OK;
}
static int refuseMember(RtContext* c, const char* what)
{
    if (c->leader) return fail(c, RT_E_STATE, std::string(what) + ": this context belongs to a group; call it on the context rtCreateMulti returned");
    return RT_OK;
}

// `one` on the context, then on each follower of its group; a follower's failure is reported on the context
template <class F> static int forGroup(RtContext* c, F one)
{
    int rc = one(c);
    if (rc != RT_OK || !c) return rc;
    for (RtContext* m : c->followers) if ((rc = one(m)) != RT_OK) return fail(c, rc, "GPU " + std::to_string(m->device) + ": " + m->err);
    return RT_OK;
}

// ---- the named per-pixel images: one W x H DevBuf each, served by name to rtReadback and rtGetDevicePointer -----------------------
template <class T> static int allocateZeroed(RtContext* c, DevBuf<T>& b, size_t n)
{
    CK(b.ensure(n));
    CK(cudaMemsetAsync(b.p, 0, n * sizeof(T), c->stream));
    return RT_OK;
}

// An image's DevBuf field of RtContext, whatever its element type
struct ImageBuf
{
    size_t element;                                  // bytes per pixel
    void* (*p)(const RtContext*);
    size_t (*count)(const RtContext*);
    int (*allocateZeroed)(RtContext*, size_t n);
    void (*release)(RtContext*);
};
template <auto F> static constexpr ImageBuf imageBuf()
{
    using T = std::remove_reference_t<decltype(*(std::declval<RtContext&>().*F).p)>;
    return {sizeof(T), [](const RtContext* c) -> void* { return (c->*F).p; }, [](const RtContext* c) { return (c->*F).count; },
            [](RtContext* c, size_t n) { return allocateZeroed(c, c->*F, n); }, [](RtContext* c) { (c->*F).release(); }};
}

struct NamedImage
{
    const char* name;
    ImageBuf buf;
    const char* producer;                            // the call that allocates it, for the "no ... yet" refusal
    bool resizeAlways;                               // rtResize allocates it; the others follow a new size only once allocated
    bool resetAccumulated;                           // RT_KERNEL_RESET_ACCUMULATED zeroes its region: it accumulates over the same frames
    bool readback;                                   // rtReadback serves it (PixelStats has rtReadbackPixelStats)
    bool refuseGroup;                                // rtReadback / rtGetDevicePointer refuse a group context
};

// A new size zeroes every allocated image; the producers that do not write every pixel allocate theirs zero-filled (allocateZeroed)
static const NamedImage kImages[] = {
    // name                buffer                                  producer                                            resize reset  read   group
    {"FrameRender",       imageBuf<&RtContext::frame>(),         "rtResize",                                         true,  false, true,  false},
    {"AccumulatedRender", imageBuf<&RtContext::accum>(),         "rtResize",                                         true,  true,  true,  false},
    {"PixelStats",        imageBuf<&RtContext::pixelStats>(),    "counting dispatch (rtSetOption(\"countStats\", 1))", false, false, false, false},
    {"FeatureFrame",      imageBuf<&RtContext::featureFrame>(),  "rtDispatchFeatures",                               false, false, true,  true},
    {"AccumulatedAlbedo", imageBuf<&RtContext::accumAlbedo>(),   "rtDispatchFeatures",                               false, true,  true,  true},
    {"AccumulatedNormal", imageBuf<&RtContext::accumNormal>(),   "rtDispatchFeatures",                               false, true,  true,  true},
    {"DenoisedRender",    imageBuf<&RtContext::denoised>(),      "rtDenoise",                                        false, false, true,  true},
    {"TemporalFrame",     imageBuf<&RtContext::temporalFrame>(), "rtDenoiseTemporal",                                false, false, true,  true},
    {"AdaptiveMoments",   imageBuf<&RtContext::moments>(),       "rtDispatchAdaptive",                               false, true,  true,  true},
};

static const NamedImage* findImage(const char* name)
{
    for (const NamedImage& img : kImages) if (strcmp(img.name, name) == 0) return &img;
    return nullptr;
}

static int imageReady(RtContext* c, const NamedImage& img, const char* what)
{
    if (img.refuseGroup) { int rc = refuseGroup(c, what); if (rc != RT_OK) return rc; }
    if (!img.buf.p(c)) return fail(c, RT_E_STATE, std::string(what) + ": no " + img.producer + " yet");
    return RT_OK;
}

// The synchronous display calls: wait for a pipelined copy (it may still read `display`), `encode` n pixels into `display`, copy it to dst
template <class Encode> static int displayTo(RtContext* c, Encode encode, uint8_t* dst, size_t bytes)
{
    const size_t n = bytes / 4;
    CK(cudaSetDevice(c->device));
    if (c->copyPending) { CK(cudaEventSynchronize(c->copyDone)); c->copyPending = false; }
    CK(c->display.ensure(n));
    int rc = encode(n); if (rc != RT_OK) return rc;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(dst, c->display.p, bytes, cudaMemcpyDeviceToHost, c->stream));
    CK(cudaStreamSynchronize(c->stream));
    return RT_OK;
}

static int drainEvents(RtContext* c)
{
    for (auto& ev : c->pending)
    {
        CK(cudaEventSynchronize(ev.b));
        float ms = 0; CK(cudaEventElapsedTime(&ms, ev.a, ev.b));
        c->stats.kernelMs += ms;
        c->freeEvents.push_back(ev);
    }
    c->pending.clear();
    for (auto& ev : c->pendingX)
    {
        CK(cudaEventSynchronize(ev.b));
        float ms = 0; CK(cudaEventElapsedTime(&ms, ev.a, ev.b));
        c->stats.exchangeMs += ms;
        c->freeEvents.push_back(ev);
    }
    c->pendingX.clear();
    return RT_OK;
}

static void closePeers(RtContext* c)
{
    for (void* p : c->peerBase) cudaIpcCloseMemHandle(p);
    c->peerBase.clear(); c->nPeers = 0;
}

extern "C" {

static void destroyComm(RtContext* c);

int rtGetVersion(void) { return RT_B200_VERSION; }

int rtCreate(RtContext** out, int device)
{
    if (!out) return fail(nullptr, RT_E_INVALID, "rtCreate: out is NULL");
    *out = nullptr;
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0)
        return fail(nullptr, RT_E_NO_DEVICE, std::string("rtCreate: no CUDA device (") + (e != cudaSuccess ? cudaGetErrorString(e) : "device count 0") + "); librt_b200 has no CPU path");
    if (device < 0 || device >= n) return fail(nullptr, RT_E_INVALID, "rtCreate: device ordinal out of range");
    RtContext* c = new RtContext();
    memset(&c->P, 0, sizeof(c->P));
    memset(&c->stats, 0, sizeof(c->stats));
    c->device = device;
    c->P.tileWorld = 1; c->P.bandRows = 1;
    const float ident[16] = {1,0,0,0, 0,1,0,0, 0,0,1,0, 0,0,0,1};
    memcpy(c->P.cam, ident, sizeof(ident));
    auto bail = [&](cudaError_t err, const char* what)
    {
        const std::string m = std::string(what) + ": " + cudaGetErrorString(err);
        if (c->dCounters) cudaFree(c->dCounters);
        if (c->dWork) cudaFree(c->dWork);
        if (c->ownStream) cudaStreamDestroy(c->ownStream);
        delete c;
        return fail(nullptr, RT_E_CUDA, m);
    };
    if ((e = cudaSetDevice(device)) != cudaSuccess) return bail(e, "cudaSetDevice");
    cudaDeviceProp prop;
    if ((e = cudaGetDeviceProperties(&prop, device)) != cudaSuccess) return bail(e, "cudaGetDeviceProperties");
    if (prop.major != 9 || prop.minor != 0) { delete c; return fail(nullptr, RT_E_NO_DEVICE, "rtCreate: device is not sm_90 (H100-class); this library carries sm_90a code only"); }
    c->numSMs = prop.multiProcessorCount;
    if ((e = cudaStreamCreateWithFlags(&c->ownStream, cudaStreamNonBlocking)) != cudaSuccess) return bail(e, "cudaStreamCreate");
    c->stream = c->ownStream;
    if ((e = cudaMalloc(&c->dCounters, 8 * sizeof(unsigned long long))) != cudaSuccess) return bail(e, "cudaMalloc");
    if ((e = cudaMalloc(&c->dWork, 64)) != cudaSuccess) return bail(e, "cudaMalloc");
    cudaMemset(c->dCounters, 0, 8 * sizeof(unsigned long long));
    cudaMemset(c->dWork, 0, 64);
    if ((e = wave_configure()) != cudaSuccess) return bail(e, "cudaFuncSetAttribute");
    if ((e = pool_configure()) != cudaSuccess) return bail(e, "cudaFuncSetAttribute");
    *out = c;
    return RT_OK;
}

int rtDestroy(RtContext* c)
{
    if (!c) return RT_E_INVALID;
    if (c->leader) return fail(c, RT_E_STATE, "rtDestroy: this context belongs to a group; destroy the context rtCreateMulti returned");
    {
        std::vector<RtContext*> members; members.swap(c->followers);
        destroyComm(c);
        for (RtContext* m : members) { destroyComm(m); m->leader = nullptr; rtDestroy(m); }
    }
    cudaSetDevice(c->device);
    cudaStreamSynchronize(c->stream);
    c->nodes.release(); c->tris.release(); c->models.release(); c->spheres.release();
    if (c->copyStream) { cudaStreamSynchronize(c->copyStream); cudaStreamDestroy(c->copyStream); }
    if (c->snapReady) cudaEventDestroy(c->snapReady);
    if (c->copyDone) cudaEventDestroy(c->copyDone);
    c->snap.release();
    c->buildArena.release(); c->handoff.release(); c->poolCold.release();
    for (int k = 0; k < 2; k++) { if (c->stageBuf[k]) cudaFreeHost(c->stageBuf[k]); if (c->stageEv[k]) cudaEventDestroy(c->stageEv[k]); }
    for (const NamedImage& img : kImages) img.buf.release(c);
    c->tileSend.release(); c->tileRecv.release(); c->display.release();
    c->queryRays.release(); c->queryHits.release(); c->cameraRays.release();
    c->denoiseScratch.release(); c->temporalHist.release();
    c->adaptiveList.release(); c->adaptiveScratch.release();
    c->probeScratch.release(); c->probePositions.release(); c->probeOut.release(); c->cubeOut.release();
    if (c->adaptiveCount) cudaFreeHost(c->adaptiveCount);
    c->repack.release();
    closePeers(c);
    for (auto& ev : c->pending) { cudaEventDestroy(ev.a); cudaEventDestroy(ev.b); }
    for (auto& ev : c->pendingX) { cudaEventDestroy(ev.a); cudaEventDestroy(ev.b); }
    for (auto& ev : c->freeEvents) { cudaEventDestroy(ev.a); cudaEventDestroy(ev.b); }
    if (c->dCounters) cudaFree(c->dCounters);
    if (c->dWork) cudaFree(c->dWork);
    if (c->ownStream) cudaStreamDestroy(c->ownStream);
    delete c;
    return RT_OK;
}

const char* rtLastError(const RtContext* c) { return c ? c->err.c_str() : g_createErr.c_str(); }

int rtSetStream(RtContext* c, void* s)
{
    if (!c) return RT_E_INVALID;
    CK(cudaSetDevice(c->device));
    CK(cudaStreamSynchronize(c->stream));           // work already queued finishes before the switch
    c->stream = s ? (cudaStream_t)s : c->ownStream;
    return RT_OK;
}

static int one_rtSetBuffer(RtContext* c, const char* name, const void* data, int count, int stride)
{
    if (!c || !name || count < 0 || (count > 0 && !data)) return fail(c, RT_E_INVALID, "rtSetBuffer: bad argument");
    CK(cudaSetDevice(c->device));
    const std::string n(name);
    if (n == "Triangles")
    {
        if (stride != (int)sizeof(RtTriangle)) return fail(c, RT_E_INVALID, "rtSetBuffer: Triangles stride must be 72");
        CK(c->tris.ensure(count));
        if (count) CK(cudaMemcpyAsync(c->tris.p, data, (size_t)count * sizeof(RtTriangle), cudaMemcpyHostToDevice, c->stream));
        c->sceneDirty = true;
        return RT_OK;
    }
    if (n == "Nodes")
    {
        if (stride != (int)sizeof(RtNode)) return fail(c, RT_E_INVALID, "rtSetBuffer: Nodes stride must be 32");
        CK(c->nodes.ensure(count));
        c->hNodes.assign((const RtNode*)data, (const RtNode*)data + count);
        if (count) CK(cudaMemcpyAsync(c->nodes.p, c->hNodes.data(), (size_t)count * sizeof(RtNode), cudaMemcpyHostToDevice, c->stream));
        c->sceneDirty = true;
        return RT_OK;
    }
    if (n == "ModelInfo")
    {
        if (stride != (int)sizeof(RtModel)) return fail(c, RT_E_INVALID, "rtSetBuffer: ModelInfo stride must be 224");
        // the BVH repack depends only on the (nodeOffset, triOffset) pairs; matrices / materials change every frame (RCM:192-204)
        bool sameTopology = (size_t)count == c->hModels.size();
        const RtModel* m = (const RtModel*)data;
        // the reference re-sends ModelInfo every frame (RCM:192-204), mostly with the bytes of the frame before: nothing to do then
        if (sameTopology && count > 0 && c->models.count == (size_t)count && memcmp(m, c->hModels.data(), (size_t)count * sizeof(RtModel)) == 0) return RT_OK;
        for (int i = 0; sameTopology && i < count; i++)
            sameTopology = m[i].nodeOffset == c->hModels[i].nodeOffset && m[i].triOffset == c->hModels[i].triOffset;
        if (!sameTopology) c->sceneDirty = true;
        CK(c->models.ensure(count));
        c->hModels.assign(m, m + count);
        if (count) CK(cudaMemcpyAsync(c->models.p, c->hModels.data(), (size_t)count * sizeof(RtModel), cudaMemcpyHostToDevice, c->stream));
        c->modelsDirty = true;
        return RT_OK;
    }
    if (n == "Spheres")
    {
        if (stride != (int)sizeof(RtSphere)) return fail(c, RT_E_INVALID, "rtSetBuffer: Spheres stride must be 104");
        if (count > 0 && c->spheres.count == (size_t)count && c->hSpheres.size() == (size_t)count && memcmp(data, c->hSpheres.data(), (size_t)count * sizeof(RtSphere)) == 0) return RT_OK;
        CK(c->spheres.ensure(count));
        c->hSpheres.assign((const RtSphere*)data, (const RtSphere*)data + count);
        if (count) CK(cudaMemcpyAsync(c->spheres.p, c->hSpheres.data(), (size_t)count * sizeof(RtSphere), cudaMemcpyHostToDevice, c->stream));
        c->spheresDirty = true;
        return RT_OK;
    }
    return fail(c, RT_E_UNKNOWN_NAME, std::string("rtSetBuffer: unknown buffer ") + name);
}

static int one_rtSetInt(RtContext* c, const char* name, int v)
{
    if (!c || !name) return fail(c, RT_E_INVALID, "rtSetInt: bad argument");
    const std::string n(name);
    if (n == "Frame") c->P.Frame = v;
    else if (n == "UseSky") c->P.UseSky = v;
    else if (n == "MaxBounceCount") c->P.MaxBounceCount = v;
    else if (n == "NumRaysPerPixel") c->P.NumRaysPerPixel = v;
    else if (n == "renderSeed") c->P.renderSeed = v;
    else if (n == "modelCount")
    {
        // the pair plan, the mesh roots, the DevModel records and the TLAS are all sized for the count they were built with
        if (v != c->P.modelCount) c->sceneDirty = c->modelsDirty = true;
        c->P.modelCount = v;
    }
    else if (n == "triangleCount" || n == "visMode") { /* declared but never read by the shader (HL:24,120) */ }
    else return fail(c, RT_E_UNKNOWN_NAME, std::string("rtSetInt: unknown uniform ") + name);
    return RT_OK;
}

static int one_rtSetInts(RtContext* c, const char* name, const int* v, int n)
{
    if (!c || !name || !v) return fail(c, RT_E_INVALID, "rtSetInts: bad argument");
    if (std::string(name) == "Resolution")
    {
        if (n != 2 || v[0] <= 0 || v[1] <= 0) return fail(c, RT_E_INVALID, "rtSetInts: Resolution takes 2 positive values");
        c->P.W = (unsigned)v[0]; c->P.H = (unsigned)v[1];
        return RT_OK;
    }
    return fail(c, RT_E_UNKNOWN_NAME, std::string("rtSetInts: unknown uniform ") + name);
}

static int one_rtSetFloat(RtContext* c, const char* name, float v)
{
    if (!c || !name) return fail(c, RT_E_INVALID, "rtSetFloat: bad argument");
    const std::string n(name);
    if (n == "DefocusStrength") c->P.DefocusStrength = v;
    else if (n == "DivergeStrength") c->P.DivergeStrength = v;
    else if (n == "SunFocus") c->P.SunFocus = v;
    else if (n == "SunIntensity") c->P.SunIntensity = v;
    else if (n == "debugVisScale") { }
    else return fail(c, RT_E_UNKNOWN_NAME, std::string("rtSetFloat: unknown uniform ") + name);
    return RT_OK;
}

static int one_rtSetVector(RtContext* c, const char* name, const float v[4])
{
    if (!c || !name || !v) return fail(c, RT_E_INVALID, "rtSetVector: bad argument");
    const std::string n(name);
    if (n == "ViewParams") memcpy(c->P.ViewParams, v, 12);
    else if (n == "SunColour") memcpy(c->P.SunColour, v, 12);
    else if (n == "dirToSun") memcpy(c->P.dirToSun, v, 12);
    else if (n == "debugParams") { }
    else return fail(c, RT_E_UNKNOWN_NAME, std::string("rtSetVector: unknown uniform ") + name);
    return RT_OK;
}

static int one_rtSetMatrix(RtContext* c, const char* name, const float v[16])
{
    if (!c || !name || !v) return fail(c, RT_E_INVALID, "rtSetMatrix: bad argument");
    if (std::string(name) == "CamLocalToWorldMatrix") { memcpy(c->P.cam, v, 64); return RT_OK; }
    return fail(c, RT_E_UNKNOWN_NAME, std::string("rtSetMatrix: unknown uniform ") + name);
}

static int one_rtSetBool(RtContext* c, const char* name, int v)
{
    if (!c || !name) return fail(c, RT_E_INVALID, "rtSetBool: bad argument");
    if (std::string(name) == "accumulate") { c->P.accumulate = v != 0; return RT_OK; }
    return fail(c, RT_E_UNKNOWN_NAME, std::string("rtSetBool: unknown uniform ") + name);
}

static int one_rtResize(RtContext* c, int w, int h)
{
    if (!c || w <= 0 || h <= 0) return fail(c, RT_E_INVALID, "rtResize: bad size");
    CK(cudaSetDevice(c->device));
    if (w != c->width || h != c->height)
    {
        if (c->copyPending) { CK(cudaEventSynchronize(c->copyDone)); c->copyPending = false; }
        const size_t n = (size_t)w * h;
        for (const NamedImage& img : kImages)
            if (img.resizeAlways || img.buf.p(c)) { int rc = img.buf.allocateZeroed(c, n); if (rc != RT_OK) return rc; }
        // the scratch images are freed: the denoiser's, the temporal history (discarded), the adaptive pixel list, the camera's rays
        c->denoiseScratch.release();
        c->temporalHist.release(); c->temporalHistory = false;
        c->adaptiveList.release(); c->adaptiveScratch.release();
        c->cameraRays.release();
        c->width = w; c->height = h;
        c->tileSend.release(); c->tileRecv.release();
        closePeers(c);                                      // peer mappings refer to images of the old size
    }
    c->P.W = (unsigned)w; c->P.H = (unsigned)h;
    return RT_OK;
}

int rtSetTile(RtContext* c, int rank, int world, int bandRows)
{
    if (!c || world < 1 || rank < 0 || rank >= world || bandRows < 1) return fail(c, RT_E_INVALID, "rtSetTile: bad argument");
    if (c->leader) return fail(c, RT_E_STATE, "rtSetTile: this context belongs to a group");
    if (!c->followers.empty())
    {
        // a group's ranks are its GPUs; only the band height is the caller's
        if (rank != 0 || world != (int)c->followers.size() + 1) return fail(c, RT_E_INVALID, "rtSetTile: a group renders as rank 0 of its own GPU count; only bandRows can change");
        for (RtContext* m : c->followers) { if (bandRows != m->bandRows) { m->tileSend.release(); m->tileRecv.release(); } m->bandRows = bandRows; }
    }
    if (c->comm && (rank != c->commRank || world != c->commWorld)) return fail(c, RT_E_INVALID, "rtSetTile: rank / world differ from the communicator's (rtCommInit)");
    if (rank != c->tileRank || world != c->tileWorld || bandRows != c->bandRows) { c->tileSend.release(); c->tileRecv.release(); }
    c->tileRank = rank; c->tileWorld = world; c->bandRows = bandRows;
    return RT_OK;
}

static int one_rtSetOption(RtContext* c, const char* name, int value)
{
    if (!c || !name) return fail(c, RT_E_INVALID, "rtSetOption: bad argument");
    const std::string n(name);
    if (n == "kernel") { if (value < -1 || value > 2) return fail(c, RT_E_INVALID, "rtSetOption: kernel must be -1 (auto), 0, 1 or 2"); c->optKernel = value; }
    else if (n == "countStats") c->optCountStats = value != 0;
    else if (n == "exchange") c->optExchange = value != 0;
    else if (n == "sampleChunks") { if (value < -1 || value > 64) return fail(c, RT_E_INVALID, "rtSetOption: sampleChunks must be -1 (automatic), 0 / 1 (whole pixels) or 2..64"); c->optSampleChunks = value; }
    else if (n == "smemNodes") c->optSmemPairs = value;
    else if (n == "modelSkip") c->optModelSkip = value != 0;
    else if (n == "tlas")
    {
        if (value < -1 || value > 1) return fail(c, RT_E_INVALID, "rtSetOption: tlas must be -1 (automatic), 0 or 1");
        if (value != c->optTlas) { c->optTlas = value; c->modelsDirty = true; }
    }
    else if (n == "extInstantiation") c->optForceExt = value != 0;
    else if (n == "sortRays") c->optSortRays = value != 0;
    else if (n == "gridFit") c->optGridFit = value != 0;
    else if (n == "l2Persist") c->optL2Persist = value != 0;
    else if (n == "zeroDefocusShortcut") c->optZeroDefocus = value != 0;      // only RT_SKIP_ZERO_DEFOCUS builds read the flag it controls
    else if (n == "treeletPrefetch")
    {
#ifdef RT_TREELET_PREFETCH
        c->optTreeletPrefetch = value != 0;
#else
        if (value) return fail(c, RT_E_INVALID, "rtSetOption: treeletPrefetch needs a library built with RT_TREELET_PREFETCH (the default kernels do not strip the flag bit)");
#endif
    }
    else if (n == "pairOrder") { if (value < 0 || value > 32) return fail(c, RT_E_INVALID, "rtSetOption: pairOrder must be 0 (breadth-first) or a treelet depth 1..32"); c->optPairOrder = value; }
    else if (n == "tailLanes") { if (value < 0 || value > 31) return fail(c, RT_E_INVALID, "rtSetOption: tailLanes must be in [0, 31]"); c->optTailLanes = value; }
    else if (n == "poolSlots") { if (value != 0 && value != 32 && value != 64 && value != 96) return fail(c, RT_E_INVALID, "rtSetOption: poolSlots must be 0 (automatic), 32, 64 or 96"); c->optPoolSlots = value; }
    else return fail(c, RT_E_UNKNOWN_NAME, std::string("rtSetOption: unknown option ") + name);
    return RT_OK;
}

// ---- the setters of a context that leads a group (rtCreateMulti) reach every GPU of the group ----
int rtSetBuffer(RtContext* c, const char* name, const void* data, int count, int stride)
{
    return forGroup(c, [&](RtContext* m) { return one_rtSetBuffer(m, name, data, count, stride); });
}
int rtSetInt(RtContext* c, const char* name, int v) { return forGroup(c, [&](RtContext* m) { return one_rtSetInt(m, name, v); }); }
int rtSetInts(RtContext* c, const char* name, const int* v, int n) { return forGroup(c, [&](RtContext* m) { return one_rtSetInts(m, name, v, n); }); }
int rtSetFloat(RtContext* c, const char* name, float v) { return forGroup(c, [&](RtContext* m) { return one_rtSetFloat(m, name, v); }); }
int rtSetVector(RtContext* c, const char* name, const float v[4]) { return forGroup(c, [&](RtContext* m) { return one_rtSetVector(m, name, v); }); }
int rtSetMatrix(RtContext* c, const char* name, const float v[16]) { return forGroup(c, [&](RtContext* m) { return one_rtSetMatrix(m, name, v); }); }
int rtSetBool(RtContext* c, const char* name, int v) { return forGroup(c, [&](RtContext* m) { return one_rtSetBool(m, name, v); }); }
int rtResize(RtContext* c, int w, int h) { return forGroup(c, [&](RtContext* m) { return one_rtResize(m, w, h); }); }
int rtSetOption(RtContext* c, const char* name, int value) { return forGroup(c, [&](RtContext* m) { return one_rtSetOption(m, name, value); }); }

// Automatic choice: with meshes the pooled wavefront kernel wins (BVH traversal needs the ray queue);
// for sphere-only scenes every ray costs the same and one path per lane avoids the pool's shared-memory round trips.
// Small tiles (multi-GPU, small images).  A pixel's samples are one sequential chain, so with about one pixel per pool slot the pools
// have nothing to balance: the slots that get a second pixel run it on a mostly empty machine for another whole pixel-time.  One path
// per lane then finishes earlier although its throughput is lower: below 1.5 pixels per slot (2.5 in the 1-spp mode) the automatic
// choice is kernel 1.  (Thresholds in pixels per slot, so they follow the SM count; not re-tuned on the H100.)
#ifndef RT_SMALL_TILE_PIXELS_PER_SLOT
#define RT_SMALL_TILE_PIXELS_PER_SLOT 1.5
#endif
#ifndef RT_SMALL_TILE_PIXELS_PER_SLOT_1SPP
#define RT_SMALL_TILE_PIXELS_PER_SLOT_1SPP 2.5
#endif
static int effectiveKernel(const RtContext* c)
{
    if (c->optKernel >= 0) return c->optKernel;
    if (c->P.modelCount <= 0) return 1;
    const double slots = (double)c->numSMs * POOL_WARPS * 64.0;
    const long long chain = (long long)c->P.NumRaysPerPixel * c->dispatchFrames;      // samples one slot runs for a pixel
    if (chain > RT_MAX_BATCH_SAMPLES) return 1;          // the pooled kernel's slot counts a pixel's samples in 20 bits (info_pack); kernel 1 in an int
    const double threshold = chain <= 1 ? RT_SMALL_TILE_PIXELS_PER_SLOT_1SPP : RT_SMALL_TILE_PIXELS_PER_SLOT;
    if (c->dispatchPixels > 0 && (double)c->dispatchPixels < threshold * slots) return 1;
    return 2;
}

// "l2Persist": ask the L2 to keep the node-pair records (persisting access-policy window on the dispatch stream; every ray walks
// them, the triangle stream is marked streaming by omission).  The scenes mostly hit in L2 already, so this is a
// candidate for the misses' latency, not for bandwidth; off by default.
static void applyL2Persistence(RtContext* c)
{
#ifndef RT_SIMT_EMU
    const void* base = c->repack.pairs.p;
    const size_t bytes = c->repack.totalPairs * sizeof(NodePair);
    const int want = c->optL2Persist && base && bytes > 0;
    if (want == c->l2PersistApplied && (!want || (base == c->l2PersistBase && bytes == c->l2PersistBytes))) return;
    cudaStreamAttrValue attr; memset(&attr, 0, sizeof(attr));
    if (want)
    {
        cudaDeviceProp prop;
        if (cudaGetDeviceProperties(&prop, c->device) != cudaSuccess || prop.persistingL2CacheMaxSize <= 0) return;
        size_t setAside = bytes < (size_t)prop.persistingL2CacheMaxSize ? bytes : (size_t)prop.persistingL2CacheMaxSize;
        if (cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, setAside) != cudaSuccess) { cudaGetLastError(); return; }
        size_t window = bytes < (size_t)prop.accessPolicyMaxWindowSize ? bytes : (size_t)prop.accessPolicyMaxWindowSize;
        attr.accessPolicyWindow.base_ptr = const_cast<void*>(base);
        attr.accessPolicyWindow.num_bytes = window;
        attr.accessPolicyWindow.hitRatio = window > 0 ? (float)((double)setAside / (double)window > 1.0 ? 1.0 : (double)setAside / (double)window) : 0.0f;
        attr.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
        attr.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
    }
    if (cudaStreamSetAttribute(c->stream, cudaStreamAttributeAccessPolicyWindow, &attr) != cudaSuccess) { cudaGetLastError(); return; }
    if (!want) cudaCtxResetPersistingL2Cache();
    c->l2PersistApplied = want; c->l2PersistBase = base; c->l2PersistBytes = bytes;
#else
    (void)c;
#endif
}

// Scene preparation, shared by rtDispatch (prepareScene) and rtTraceRays (prepareQueryScene); `what` names the call in messages.
// checkScene: the buffers and offsets a trace reads are there.
static int checkScene(RtContext* c, const std::string& what)
{
    if (c->P.modelCount < 0 || (size_t)c->P.modelCount > c->models.count) return fail(c, RT_E_STATE, what + ": modelCount exceeds the ModelInfo buffer");
    if (c->P.modelCount > 0 && (c->nodes.count == 0 || c->tris.count == 0)) return fail(c, RT_E_STATE, what + ": models without Nodes / Triangles buffers");
    for (int i = 0; i < c->P.modelCount; i++)
    {
        const RtModel& m = c->hModels[i];
        if (m.nodeOffset < 0 || (size_t)m.nodeOffset >= c->nodes.count || m.triOffset < 0 || (size_t)m.triOffset > c->tris.count)
            return fail(c, RT_E_STATE, what + ": model nodeOffset / triOffset out of range");
    }
    return RT_OK;
}

// The layout of the pair records a RayTrace dispatch asks for now: the tree-top budget, the record order and the treelet flag
static void sceneLayout(const RtContext* c, int& budget, int& pairOrder, bool& treelets)
{
    // shared-memory budget for the tree tops: what the selected kernel can afford next to its own shared state
    // automatic = 0: staging tree tops never beat leaving that shared memory to L1
    budget = c->optSmemPairs < 0 ? 0 : c->optSmemPairs;
    const int kernelSel = effectiveKernel(c);
    treelets = c->optTreeletPrefetch && kernelSel != 0;                 // two-level treelets with flagged roots; no shared-memory staging with it
    pairOrder = treelets ? 2 : c->optPairOrder;
    if (treelets) budget = 0;
    if (budget > 3072) budget = 3072;                                   // planScene's own clamp (192 KB), so that budgetUsed compares equal
    if (kernelSel == 2) { const int mx = pool_max_smem_pairs(c->optPoolSlots ? c->optPoolSlots : 96, (int)c->spheres.count); if (budget > mx) budget = mx; }
    else if (kernelSel == 0) budget = 0;
}

// The pair records, mesh roots and triangle streams, when the scene's topology changed
static int planSceneIfDirty(RtContext* c, const std::string& what, int budget, int pairOrder, bool treelets)
{
    if (!c->sceneDirty) return RT_OK;
    std::string msg;
    cudaError_t e = c->repack.buildScene(c->hNodes, c->hModels, c->P.modelCount, c->tris.p, c->tris.count, budget, c->stream, msg, pairOrder, treelets);
    if (e != cudaSuccess) return failCuda(c, e, "repack scene");
    if (!msg.empty()) return fail(c, RT_E_STATE, what + ": " + msg);
    c->sceneDirty = false; c->modelsDirty = true;
    return RT_OK;
}

static int fitOriginPadding(RtContext* c);

static int prepareScene(RtContext* c)
{
    int rc = checkScene(c, "rtDispatch"); if (rc != RT_OK) return rc;
    int budget, pairOrder; bool treelets;
    sceneLayout(c, budget, pairOrder, treelets);
    if (budget != c->repack.budgetUsed || pairOrder != c->repack.orderUsed || treelets != c->repack.flagsUsed) c->sceneDirty = true;
    if ((rc = planSceneIfDirty(c, "rtDispatch", budget, pairOrder, treelets)) != RT_OK) return rc;
    return fitOriginPadding(c);
}

// rtTraceRays / rtTraceOcclusion: what does not depend on the image or the kernel choice.  A layout that is already built is kept
// whatever its budget (a query reads every record from global memory); a scene that must be planned anyway gets the layout the next
// dispatch would ask for, so that with default options the query never makes that dispatch plan again.
static int prepareQueryScene(RtContext* c, const char* what)
{
    int rc = checkScene(c, what); if (rc != RT_OK) return rc;
    int budget, pairOrder; bool treelets;
    sceneLayout(c, budget, pairOrder, treelets);
    if ((rc = planSceneIfDirty(c, what, budget, pairOrder, treelets)) != RT_OK) return rc;
    return fitOriginPadding(c);
}

// The model records (with the TLAS) and the sphere accelerator, rebuilt when they changed or when the box of possible camera-ray
// origins outgrew the one their padding was computed for
static int fitOriginPadding(RtContext* c)
{
    {
        // box containing every possible ray origin: the camera (with its defocus disc) and all geometry; it sizes the padding of
        // the models' world boxes and of the sphere accelerator, which are rebuilt when the box outgrows the one they were built for
        float lo[3], hi[3];
        const float jitter = fabsf(c->P.DefocusStrength) / (float)(c->P.W ? c->P.W : 1u) *
                             (fabsf(c->P.cam[0]) + fabsf(c->P.cam[1]) + fabsf(c->P.cam[2]) + fabsf(c->P.cam[4]) + fabsf(c->P.cam[5]) + fabsf(c->P.cam[6]));
        for (int a = 0; a < 3; a++) { lo[a] = c->P.cam[12 + a] - jitter; hi[a] = c->P.cam[12 + a] + jitter; }
        for (const RtSphere& s : c->hSpheres) for (int a = 0; a < 3; a++) { lo[a] = fminf(lo[a], s.centre[a] - fabsf(s.radius)); hi[a] = fmaxf(hi[a], s.centre[a] + fabsf(s.radius)); }
        for (int i = 0; i < c->P.modelCount; i++)
        {
            const RtModel& m = c->hModels[i];
            double mlo[3], mhi[3];
            if (!RepackState::worldBoxOfModel(m, c->repack.roots[std::make_pair(m.nodeOffset, m.triOffset)], mlo, mhi)) { for (int a = 0; a < 3; a++) { lo[a] = -INFINITY; hi[a] = INFINITY; } break; }
            for (int a = 0; a < 3; a++) { lo[a] = fminf(lo[a], std::nextafterf((float)mlo[a], -INFINITY)); hi[a] = fmaxf(hi[a], std::nextafterf((float)mhi[a], INFINITY)); }
        }
        if (!c->modelsDirty && !c->repack.modelBoundCovers(lo, hi)) c->modelsDirty = true;
        if (!c->spheresDirty && c->repack.sphBvh && !c->repack.sphereBoundCovers(lo, hi)) c->spheresDirty = true;
        if (c->modelsDirty || c->spheresDirty)      // some room, so that a moving camera does not rebuild every frame
            for (int a = 0; a < 3; a++) { const float ext = 0.25f * (hi[a] - lo[a]) + 0.01f; lo[a] -= ext; hi[a] += ext; }
        if (c->modelsDirty)
        {
            cudaError_t e = c->repack.buildModels(c->hModels, c->hNodes, c->P.modelCount, c->stream, c->optTlas, lo, hi);
            if (e != cudaSuccess) return failCuda(c, e, "repack models");
            c->modelsDirty = false;
        }
        if (c->spheresDirty)
        {
            cudaError_t e = c->repack.buildSpheres(c->hSpheres, lo, hi, c->stream);
            if (e != cudaSuccess) return failCuda(c, e, "repack spheres");
            c->spheresDirty = false;
        }
    }
    return RT_OK;
}

// The scene's buffers, the counters and the scene options in a parameter block (what both the camera kernels and the queries read)
static void bindScene(const RtContext* c, DevParams& P)
{
    P.sphereCount = (int)c->spheres.count;
    P.Nodes = c->nodes.p; P.Triangles = c->tris.p; P.ModelInfo = c->models.p; P.Spheres = c->spheres.p;
    P.pairs = c->repack.pairs.p; P.triGeom = c->repack.triGeom.p; P.triNormals = c->repack.triNormals.p;
    P.models = c->repack.models.p; P.spheres = c->repack.spheres.p;
    P.sphPairs = c->repack.sphPairs.p; P.sphLeaves = c->repack.sphLeaves.p; P.sphBvh = c->repack.sphBvh;
    P.sphRootStart = c->repack.sphRootStart; P.sphRootCount = c->repack.sphRootCount;
    P.counters = c->dCounters; P.workCounter = c->dWork;
    P.forceExt = c->optForceExt; P.modelSkip = c->optModelSkip;
    P.tlasPairs = c->repack.tlasPairs.p; P.tlasLeaves = c->repack.tlasLeaves.p; P.tlas = c->repack.tlas;
    P.tlasRootStart = c->repack.tlasRootStart; P.tlasRootCount = c->repack.tlasRootCount;
}

// The parameter block of a launch that is not a camera render (queries, paths, features): the scene and the counters, no images, no peers
static DevParams queryParams(const RtContext* c)
{
    DevParams P = c->P;
    bindScene(c, P);
    P.countStats = c->optCountStats;
    P.smemPairs = 0;                                 // no tree-top staging: every record from global memory
    P.FrameRender = P.AccumulatedRender = nullptr; P.pixelStats = nullptr; P.nPeers = 0;
    return P;
}

// The boxes the models' and the spheres' padding was computed for (QueryParams, PathParams, ProbeParams)
static OriginBox sceneBounds(const RtContext* c)
{
    OriginBox b;
    for (int a = 0; a < 3; a++)
    {
        b.modelLo[a] = c->repack.modelBoundLo[a]; b.modelHi[a] = c->repack.modelBoundHi[a];
        b.sphLo[a] = c->repack.sphBoundLo[a]; b.sphHi[a] = c->repack.sphBoundHi[a];
    }
    return b;
}

// The pixels groups of 8 x 8 cover: limX x limY, none when gz = 0
static void groupLimits(int gx, int gy, int gz, unsigned W, unsigned H, unsigned& limX, unsigned& limY)
{
    limX = (unsigned long long)gx * 8ull < W ? (unsigned)gx * 8u : W;
    limY = (unsigned long long)gy * 8ull < H ? (unsigned)gy * 8u : H;
    if (gz == 0) limX = limY = 0;
}

// A pair of timing events: one the context timed before and has read, or a new one
static int takeEventPair(RtContext* c, EventPair& ev)
{
    if (!c->freeEvents.empty()) { ev = c->freeEvents.back(); c->freeEvents.pop_back(); }
    else { CK(cudaEventCreate(&ev.a)); CK(cudaEventCreate(&ev.b)); }
    return RT_OK;
}

// rtDispatchAdaptive's arguments (dispatchLocal); `active` receives the number of pixels traced
struct AdaptiveCall { float threshold; int minFrames, maxFrames; long long active; };

static int adaptiveSelect(RtContext* c, unsigned limX, unsigned limY, AdaptiveCall& ad);

// One GPU's share of a dispatch: the RayTrace kernel over this context's tile (the whole image without rtSetTile).
// frames > 1 (rtDispatchFrames, RayTrace only): frames Frame .. Frame + frames - 1 in one launch of a FRAMES kernel.
// ad (rtDispatchAdaptive, RayTrace only): the selected pixels only, in one launch of a list-driven kernel.
static int dispatchLocal(RtContext* c, int kernelIndex, int gx, int gy, int gz, int frames = 1, AdaptiveCall* ad = nullptr)
{
    if (!c || gx < 0 || gy < 0 || gz < 0) return fail(c, RT_E_INVALID, "rtDispatch: bad argument");
    if (c->width == 0) return fail(c, RT_E_STATE, "rtDispatch: rtResize has not been called");
    if ((int)c->P.W != c->width || (int)c->P.H != c->height) return fail(c, RT_E_STATE, "rtDispatch: Resolution does not match the render textures");
    CK(cudaSetDevice(c->device));
    const unsigned W = c->P.W, H = c->P.H;
    unsigned limX, limY;
    groupLimits(gx, gy, gz, W, H, limX, limY);

    if (kernelIndex == RT_KERNEL_RESET_ACCUMULATED)            // RC:26-32
    {
        if (limX == 0 || limY == 0) return RT_OK;
        for (const NamedImage& img : kImages)
        {
            void* p = img.resetAccumulated ? img.buf.p(c) : nullptr;
            if (p) CK(cudaMemset2DAsync(p, (size_t)W * img.buf.element, 0, (size_t)limX * img.buf.element, limY, c->stream));
        }
        return RT_OK;
    }
    if (kernelIndex != RT_KERNEL_RAYTRACE) return fail(c, RT_E_INVALID, "rtDispatch: kernelIndex must be 0 (RayTrace) or 1 (ResetAccumulated)");
    if (limX == 0 || limY == 0) return RT_OK;
    if (c->P.NumRaysPerPixel < 0) return fail(c, RT_E_STATE, "rtDispatch: NumRaysPerPixel is negative");
    if (c->P.MaxBounceCount > 200 || W > 65535u || H > 65535u) return fail(c, RT_E_STATE, "rtDispatch: MaxBounceCount > 200 or a resolution above 65535 is not supported");
    if (c->P.MaxBounceCount < 0) return fail(c, RT_E_STATE, "rtDispatch: MaxBounceCount is negative (the reference clamps it to [0, 32], RCM:15)");
    if (c->optKernel == 2 && c->P.NumRaysPerPixel > RT_MAX_BATCH_SAMPLES)
        return fail(c, RT_E_STATE, "rtDispatch: \"kernel\" = 2 counts a pixel's samples in 20 bits: NumRaysPerPixel above RT_MAX_BATCH_SAMPLES needs kernel 0 or 1");

    c->dispatchPixels = (unsigned long long)owned_rows(limY, c->bandRows, c->tileWorld, c->tileRank) * limX;
    c->dispatchFrames = frames;
    int rc = RT_OK;
    if (ad)
    {
        // the selection (one synchronisation: the host sizes the launch and chooses the kernel from the count, as for an image of that
        // many pixels); before the scene is prepared, so that the kernel choice sees the count
        if ((rc = checkScene(c, "rtDispatchAdaptive")) != RT_OK) return rc;
        if ((rc = adaptiveSelect(c, limX, limY, *ad)) != RT_OK) return rc;
        if (ad->active == 0) return RT_OK;
        c->dispatchPixels = (unsigned long long)ad->active;
    }
    rc = prepareScene(c);
    if (rc != RT_OK) return rc;
    if (ad && !c->moments.p && (rc = allocateZeroed(c, c->moments, (size_t)W * H)) != RT_OK) return rc;       // the first traced call allocates the moments
    applyL2Persistence(c);
    if (c->optCountStats && !c->pixelStats.p && (rc = allocateZeroed(c, c->pixelStats, (size_t)W * H)) != RT_OK) return rc;     // so does the first counting dispatch the per-pixel counters

    DevParams P = c->P;
    P.limX = limX; P.limY = limY;
    P.tileRank = c->tileRank; P.tileWorld = c->tileWorld; P.bandRows = c->bandRows; P.countStats = c->optCountStats;
    bindScene(c, P);
    P.smemPairs = c->repack.smemPairs; P.tailLanes = c->optTailLanes; P.sortRays = c->optSortRays; P.gridFit = c->optGridFit;
    P.FrameRender = c->frame.p; P.AccumulatedRender = c->accum.p;
    P.pixelStats = c->optCountStats ? c->pixelStats.p : nullptr;
    P.nPeers = c->nPeers;
    P.frames = frames;
    {
        // camOrigin = M * (0,0,0,1) as SetupPixel computes it (left to right, unfused): exact zero components and non-finite axes rule the shortcut out
        bool ok = c->P.DefocusStrength == 0.0f && c->optZeroDefocus != 0;
        for (int a = 0; a < 3 && ok; a++)
        {
            const float o = ((P.cam[a] * 0.0f + P.cam[4 + a] * 0.0f) + P.cam[8 + a] * 0.0f) + P.cam[12 + a] * 1.0f;
            ok = o != 0.0f && std::isfinite(o) && std::isfinite(P.cam[a]) && std::isfinite(P.cam[4 + a]);
        }
        P.zeroDefocus = ok ? 1 : 0;
    }
    for (int k = 0; k < c->nPeers; k++) { P.peerFrame[k] = c->peerFrame[k]; P.peerAccum[k] = c->peerAccum[k]; }

    EventPair ev;
    if ((rc = takeEventPair(c, ev)) != RT_OK) return rc;
    if (c->pending.size() >= 512) { rc = drainEvents(c); if (rc != RT_OK) return rc; }

    int kernel = effectiveKernel(c);
    if (c->P.NumRaysPerPixel == 0) kernel = 0;       // 0 samples: the per-pixel kernel reproduces the reference's 0/0 directly
    // sample chunks (small tiles): a pixel's chain may change lanes / slots between samples; the hand-off buffers belong to the context
    // (kernel 1 only: in the pooled kernel the same hand-off was slower than whole pixels on small tiles and was taken out again)
    P.chunks = kernel == 1 ? wave_chunks(c->optSampleChunks, c->numSMs, c->dispatchPixels, P.NumRaysPerPixel, P.modelCount) : 1;
    if (c->dispatchPixels == 0 || frames > 1 || ad) P.chunks = 1;      // a rank whose tile is empty (an image lower than the band pattern); a batch of frames or a pixel list runs whole pixels
    const size_t jobs = tile_jobs(limX, (unsigned)(c->dispatchPixels / limX));
    if (P.chunks > 1)
    {
        // kernel 1 counts its chunk jobs (jobs x chunks) in a 32-bit work counter that every resident lane draws from once more after
        // the last job: at most 2^31 chunk jobs leave 2^31 of headroom for those draws.  Fewer chunks on large images (chunks are
        // schedule only), whole pixels when fewer than two fit
        const unsigned long long fit = (1ull << 31) / jobs;
        if ((unsigned long long)P.chunks > fit) P.chunks = fit < 2ull ? 1 : (int)fit;
    }
    if (P.chunks > 1)
    {
        // four self-validating 64-bit words per pixel job; the tag carries a serial number of the dispatch, so nothing has to be cleared
        // between frames (only a fresh allocation and the wrap of the 24-bit serial zero the buffer: tag 0 is never expected)
        const size_t before = c->handoff.count;
        CK(c->handoff.ensure(4 * jobs));
        c->chunkSerial = (c->chunkSerial + 1u) & 0xffffffu;
        if (c->handoff.count != before || c->chunkSerial == 0u)
        {
            CK(cudaMemsetAsync(c->handoff.p, 0, c->handoff.count * sizeof(unsigned long long), c->stream));
            if (c->chunkSerial == 0u) c->chunkSerial = 1u;
        }
        P.handoff = c->handoff.p; P.chunkSerial = (int)c->chunkSerial;
    }
    if (kernel == 2 && POOL_COLD_WORDS > 0)
    {
        CK(c->poolCold.ensure((size_t)c->numSMs * POOL_WARPS * POOL_COLD_WORDS * 96));      // sized for the largest pools
        P.poolCold = c->poolCold.p;
    }
    // ad: the same kernels over the selected pixels only (adaptiveList, count long), with their moments
    const CameraForm form = ad ? FORM_LIST : frames > 1 ? FORM_FRAMES : FORM_PLAIN;
    const unsigned count = ad ? (unsigned)ad->active : 0u;
    cudaError_t e;
    if (kernel == 0) e = mega_launch(form, P, count, c->adaptiveList.p, c->moments.p, c->stream, ev.a, ev.b);
    else if (kernel == 1) e = wave_launch(form, P, c->numSMs, count, c->adaptiveList.p, c->moments.p, c->stream, ev.a, ev.b);
    else e = pool_launch(form, P, c->optPoolSlots, c->numSMs, count, c->adaptiveList.p, c->moments.p, c->stream, ev.a, ev.b);
    if (e != cudaSuccess) return failCuda(c, e, ad ? "adaptive launch" : kernel == 0 ? "megakernel launch" : kernel == 1 ? "wavefront launch" : "pool wavefront launch");
    CK(cudaGetLastError());
    c->pending.push_back(ev);
    c->stats.dispatches += (unsigned long long)frames;
    return RT_OK;
}

int rtReadback(RtContext* c, const char* tex, float* dst, size_t bytes)
{
    if (!c || !tex || !dst) return fail(c, RT_E_INVALID, "rtReadback: bad argument");
    const NamedImage* img = findImage(tex);
    if (!img || !img->readback) return fail(c, RT_E_UNKNOWN_NAME, std::string("rtReadback: unknown texture ") + tex);
    int rc = imageReady(c, *img, "rtReadback"); if (rc != RT_OK) return rc;
    if (bytes != (size_t)c->width * c->height * img->buf.element)
        return fail(c, RT_E_INVALID, "rtReadback: bytes must equal W*H*" + std::to_string(img->buf.element));
    CK(cudaSetDevice(c->device));
    CK(cudaMemcpyAsync(dst, img->buf.p(c), bytes, cudaMemcpyDeviceToHost, c->stream));
    CK(cudaStreamSynchronize(c->stream));
    return RT_OK;
}

// rtDisplay's encode of n pixels of src into `display` (tex / Frame as the sRGB 8-bit back buffer)
static void encodeDisplay(RtContext* c, const float4* src, size_t n, float frame)
{
    RT_LAUNCH((unsigned)((n + 255) / 256), 256, 0, c->stream, k_display, src, c->display.p, n, frame);
}

int rtDisplay(RtContext* c, int useAccumulated, int Frame, uint8_t* dst, size_t bytes)
{
    if (!c || !dst) return fail(c, RT_E_INVALID, "rtDisplay: bad argument");
    if (!c->frame.p) return fail(c, RT_E_STATE, "rtDisplay: rtResize has not been called");
    if (bytes != (size_t)c->width * c->height * 4) return fail(c, RT_E_INVALID, "rtDisplay: bytes must equal W*H*4");
    return displayTo(c, [&](size_t n) { encodeDisplay(c, useAccumulated ? c->accum.p : c->frame.p, n, (float)Frame); return RT_OK; }, dst, bytes);
}

// ---- pipelined readback -------------------------------------------------------------------------------------------------------
static int copyPipeline(RtContext* c)
{
    if (!c->copyStream) CK(cudaStreamCreateWithFlags(&c->copyStream, cudaStreamNonBlocking));
    if (!c->snapReady) CK(cudaEventCreateWithFlags(&c->snapReady, cudaEventDisableTiming));
    if (!c->copyDone) CK(cudaEventCreateWithFlags(&c->copyDone, cudaEventDisableTiming));
    if (c->copyPending) CK(cudaStreamWaitEvent(c->stream, c->copyDone, 0));      // the snapshot buffer is free once the copy before has read it
    return RT_OK;
}
static int copyOut(RtContext* c, void* dst, const void* src, size_t bytes)
{
    CK(cudaEventRecord(c->snapReady, c->stream));
    CK(cudaStreamWaitEvent(c->copyStream, c->snapReady, 0));
    CK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, c->copyStream));
    CK(cudaEventRecord(c->copyDone, c->copyStream));
    c->copyPending = true;
    return RT_OK;
}

int rtReadbackAsync(RtContext* c, const char* tex, float* dst, size_t bytes)
{
    if (!c || !tex || !dst) return fail(c, RT_E_INVALID, "rtReadbackAsync: bad argument");
    const std::string n(tex);
    if (n != "FrameRender" && n != "AccumulatedRender") return fail(c, RT_E_UNKNOWN_NAME, std::string("rtReadbackAsync: unknown texture ") + tex);
    const float4* src = n == "FrameRender" ? c->frame.p : c->accum.p;
    if (!src) return fail(c, RT_E_STATE, "rtReadbackAsync: rtResize has not been called");
    if (bytes != (size_t)c->width * c->height * 16) return fail(c, RT_E_INVALID, "rtReadbackAsync: bytes must equal W*H*16");
    CK(cudaSetDevice(c->device));
    int rc = copyPipeline(c); if (rc != RT_OK) return rc;
    CK(c->snap.ensure((size_t)c->width * c->height));
    CK(cudaMemcpyAsync(c->snap.p, src, bytes, cudaMemcpyDeviceToDevice, c->stream));       // the texture as it is after the work queued so far
    return copyOut(c, dst, c->snap.p, bytes);
}

int rtDisplayAsync(RtContext* c, int useAccumulated, int Frame, uint8_t* dst, size_t bytes)
{
    if (!c || !dst) return fail(c, RT_E_INVALID, "rtDisplayAsync: bad argument");
    if (!c->frame.p) return fail(c, RT_E_STATE, "rtDisplayAsync: rtResize has not been called");
    const size_t n = (size_t)c->width * c->height;
    if (bytes != n * 4) return fail(c, RT_E_INVALID, "rtDisplayAsync: bytes must equal W*H*4");
    CK(cudaSetDevice(c->device));
    int rc = copyPipeline(c); if (rc != RT_OK) return rc;
    CK(c->display.ensure(n));
    encodeDisplay(c, useAccumulated ? c->accum.p : c->frame.p, n, (float)Frame);
    CK(cudaGetLastError());
    return copyOut(c, dst, c->display.p, bytes);
}

int rtReadbackWait(RtContext* c)
{
    if (!c) return RT_E_INVALID;
    if (!c->copyPending) return RT_OK;
    CK(cudaSetDevice(c->device));
    CK(cudaEventSynchronize(c->copyDone));
    c->copyPending = false;
    return RT_OK;
}

int rtSynchronize(RtContext* c)
{
    if (!c) return RT_E_INVALID;
    if (c->copyPending) { CK(cudaSetDevice(c->device)); CK(cudaEventSynchronize(c->copyDone)); c->copyPending = false; }
    for (RtContext* m : c->followers) { CK(cudaSetDevice(m->device)); CK(cudaStreamSynchronize(m->stream)); }
    CK(cudaSetDevice(c->device));
    CK(cudaStreamSynchronize(c->stream));
    return RT_OK;
}

// ---- multi-GPU tile staging -----------------------------------------------------------------------------------------------

static size_t tileRows(const RtContext* c, int rank) { return owned_rows((unsigned)c->height, c->bandRows, c->tileWorld, rank); }

static int ensureTileBuffers(RtContext* c)
{
    if (c->width == 0) return fail(c, RT_E_STATE, "tile staging: rtResize has not been called");
    // every rank must contribute the same count to the all-gather: size by the largest share (rank 0's)
    const size_t per = tileRows(c, 0) * (size_t)c->width * 2;    // frame + accumulated
    CK(c->tileSend.ensure(per));
    CK(c->tileRecv.ensure(per * c->tileWorld));
    return RT_OK;
}

int rtPackTile(RtContext* c)
{
    if (!c) return RT_E_INVALID;
    CK(cudaSetDevice(c->device));
    int rc = ensureTileBuffers(c); if (rc != RT_OK) return rc;
    launch_pack_tile(c->frame.p, c->accum.p, c->tileSend.p, c->width, c->height, c->tileRank, c->tileWorld, c->bandRows,
                     (int)tileRows(c, 0), c->stream);
    CK(cudaGetLastError());
    return RT_OK;
}

int rtUnpackTiles(RtContext* c)
{
    if (!c) return RT_E_INVALID;
    CK(cudaSetDevice(c->device));
    int rc = ensureTileBuffers(c); if (rc != RT_OK) return rc;
    launch_unpack_tiles(c->tileRecv.p, c->frame.p, c->accum.p, c->width, c->height, c->tileWorld, c->bandRows,
                        (int)tileRows(c, 0), c->stream);
    CK(cudaGetLastError());
    return RT_OK;
}


// ---- exchange of finished tiles inside the ABI (rtCommInit / rtCreateMulti) -----------------------------------------------------

// true when a RayTrace dispatch on this context is followed by the all-gather of the frame's tiles
static bool exchanges(const RtContext* c) { return c->optExchange && c->tileWorld > 1 && (c->comm || !c->followers.empty() || c->leader); }

static int ncclFail(RtContext* c, NcclApi* api, int r, const char* what)
{
    return fail(c, RT_E_CUDA, std::string(what) + ": " + (api && api->GetErrorString ? api->GetErrorString(r) : "NCCL error") + " (" + std::to_string(r) + ")");
}

// pack -> ncclAllGather -> unpack on the streams of `n` contexts (one per GPU; n > 1 only for a single-process group, whose
// collectives are issued as one NCCL group).  Under the SIMT interpreter the group's all-gather is the copy it stands for.
static int exchangeTiles(RtContext* const* cs, int n)
{
    RtContext* lead = cs[0];
    std::vector<EventPair> evs((size_t)n);
    for (int i = 0; i < n; i++)
    {
        RtContext* c = cs[i];
        CK(cudaSetDevice(c->device));
        int rc = takeEventPair(c, evs[i]); if (rc != RT_OK) return rc;
        CK(cudaEventRecord(evs[i].a, c->stream));
        rc = rtPackTile(c); if (rc != RT_OK) return i ? fail(lead, rc, c->err) : rc;
    }
#ifdef RT_SIMT_EMU
    for (int i = 0; i < n; i++) for (int j = 0; j < n; j++)
        memcpy(cs[i]->tileRecv.p + (size_t)j * cs[j]->tileSend.count, cs[j]->tileSend.p, cs[j]->tileSend.count * sizeof(float4));
#else
    std::string why;
    NcclApi* api = NcclApi::get(why);
    if (!api) return fail(lead, RT_E_STATE, "tile exchange: " + why);
    int r;
    if (n > 1 && (r = api->GroupStart()) != NcclApi::Success) return ncclFail(lead, api, r, "ncclGroupStart");
    for (int i = 0; i < n; i++)
    {
        RtContext* c = cs[i];
        if (!c->comm) return fail(lead, RT_E_STATE, "tile exchange: no communicator (rtCommInit)");
        CK(cudaSetDevice(c->device));
        if ((r = api->AllGather(c->tileSend.p, c->tileRecv.p, c->tileSend.count * sizeof(float4), NcclApi::Char, c->comm, c->stream)) != NcclApi::Success)
            return ncclFail(lead, api, r, "ncclAllGather");
    }
    if (n > 1 && (r = api->GroupEnd()) != NcclApi::Success) return ncclFail(lead, api, r, "ncclGroupEnd");
#endif
    for (int i = 0; i < n; i++)
    {
        RtContext* c = cs[i];
        CK(cudaSetDevice(c->device));
        int rc = rtUnpackTiles(c); if (rc != RT_OK) return i ? fail(lead, rc, c->err) : rc;
        CK(cudaEventRecord(evs[i].b, c->stream));
        c->pendingX.push_back(evs[i]);
    }
    { RtContext* c = lead; CK(cudaSetDevice(c->device)); }
    return RT_OK;
}

// The exchange over this context and the followers of its group
static int exchangeGroup(RtContext* c)
{
    std::vector<RtContext*> all(1, c);
    all.insert(all.end(), c->followers.begin(), c->followers.end());
    return exchangeTiles(all.data(), (int)all.size());
}

int rtDispatch(RtContext* c, int kernelIndex, int gx, int gy, int gz)
{
    if (!c) return RT_E_INVALID;
    int rc = refuseMember(c, "rtDispatch"); if (rc != RT_OK) return rc;
    if ((rc = forGroup(c, [&](RtContext* m) { return dispatchLocal(m, kernelIndex, gx, gy, gz); })) != RT_OK) return rc;
    if (!c->followers.empty()) CK(cudaSetDevice(c->device));
    const bool traced = kernelIndex == RT_KERNEL_RAYTRACE && gz != 0 && gx > 0 && gy > 0;
    if (!traced || !exchanges(c)) return RT_OK;
    return exchangeGroup(c);
}

int rtDispatchFrames(RtContext* c, int gx, int gy, int gz, int frameCount)
{
    if (!c) return RT_E_INVALID;
    int rc = refuseMember(c, "rtDispatchFrames"); if (rc != RT_OK) return rc;
    const long long chain = (long long)frameCount * (c->P.NumRaysPerPixel > 1 ? c->P.NumRaysPerPixel : 1);
    if (frameCount < 1 || chain > RT_MAX_BATCH_SAMPLES)
        return fail(c, RT_E_INVALID, "rtDispatchFrames: frameCount must be >= 1 and frameCount * max(1, NumRaysPerPixel) at most RT_MAX_BATCH_SAMPLES");
    if (!c->P.accumulate) return fail(c, RT_E_STATE, "rtDispatchFrames: needs accumulate = 1 (without accumulation only the last frame is observable)");
    if (frameCount == 1) return rtDispatch(c, RT_KERNEL_RAYTRACE, gx, gy, gz);
    if (c->optSampleChunks >= 2) return fail(c, RT_E_STATE, "rtDispatchFrames: a batch of frames runs whole pixels; sampleChunks is forced to 2 or more");
    if ((rc = forGroup(c, [&](RtContext* m) { return dispatchLocal(m, RT_KERNEL_RAYTRACE, gx, gy, gz, frameCount); })) != RT_OK) return rc;
    if (!c->followers.empty()) CK(cudaSetDevice(c->device));
    const bool traced = gz != 0 && gx > 0 && gy > 0;
    if (!traced || !exchanges(c)) return RT_OK;
    return exchangeGroup(c);                                // one exchange for the whole batch: it carries the last frame and the sum
}

// rtDispatchAdaptive's selection over this context's covered pixels, in the camera kernels' job order: the list and its length, read
// back into ad.active (the call's one synchronisation).  Before the first traced call the moments are all zero (none allocated yet).
static int adaptiveSelect(RtContext* c, unsigned limX, unsigned limY, AdaptiveCall& ad)
{
    const unsigned int rows = owned_rows(limY, c->bandRows, c->tileWorld, c->tileRank);
    const unsigned int tilesX = (limX + 7u) / 8u;
    const unsigned long long jobs = tile_jobs(limX, rows);       // < 2^32: W, H <= 65535
    const unsigned int nBlocks = (unsigned int)((jobs + ADAPTIVE_BLOCK - 1) / ADAPTIVE_BLOCK);
    const size_t n = (size_t)c->width * c->height;
    CK(c->adaptiveList.ensure(n));
    CK(c->adaptiveScratch.ensure((size_t)(jobs / 32) + nBlocks + 1));
    if (!c->adaptiveCount) CK(cudaMallocHost((void**)&c->adaptiveCount, sizeof(unsigned int)));
    AdaptiveParams A;
    A.moments = c->moments.p;
    A.masks = c->adaptiveScratch.p; A.partials = A.masks + jobs / 32; A.count = A.partials + nBlocks; A.list = c->adaptiveList.p;
    A.W = c->P.W; A.limX = limX; A.ownedRows = rows; A.tilesX = tilesX; A.totalJobs = (unsigned int)jobs; A.nBlocks = nBlocks;
    A.tileRank = c->tileRank; A.tileWorld = c->tileWorld; A.bandRows = c->bandRows;
    A.threshold = ad.threshold; A.minFrames = (float)ad.minFrames; A.maxFrames = (float)ad.maxFrames;
    cudaError_t e = adaptive_select(A, c->stream);
    if (e != cudaSuccess) return failCuda(c, e, "adaptive selection");
    CK(cudaMemcpyAsync(c->adaptiveCount, A.count, sizeof(unsigned int), cudaMemcpyDeviceToHost, c->stream));
    CK(cudaStreamSynchronize(c->stream));
    ad.active = (long long)*c->adaptiveCount;
    return RT_OK;
}

int rtDispatchAdaptive(RtContext* c, int gx, int gy, int gz, float threshold, int minFrames, int maxFrames, int64_t* activePixels)
{
    if (!c || gx < 0 || gy < 0 || gz < 0) return fail(c, RT_E_INVALID, "rtDispatchAdaptive: bad argument");
    if (!std::isfinite(threshold) || threshold < 0.0f || !std::isfinite(threshold * threshold))
        return fail(c, RT_E_INVALID, "rtDispatchAdaptive: threshold must be finite and >= 0, with a finite square");
    if (minFrames < 2) return fail(c, RT_E_INVALID, "rtDispatchAdaptive: minFrames must be at least 2");
    if (maxFrames < minFrames || maxFrames > RT_ADAPTIVE_MAX_FRAMES)
        return fail(c, RT_E_INVALID, "rtDispatchAdaptive: maxFrames must lie in minFrames .. RT_ADAPTIVE_MAX_FRAMES");
    int rc = refuseGroup(c, "rtDispatchAdaptive"); if (rc != RT_OK) return rc;
    if (c->comm) return fail(c, RT_E_STATE, "rtDispatchAdaptive: not available on a context with a communicator (rtCommInit)");
    if (c->nPeers > 0) return fail(c, RT_E_STATE, "rtDispatchAdaptive: not available on a context with peers (rtSetPeers)");
    if (!c->P.accumulate) return fail(c, RT_E_STATE, "rtDispatchAdaptive: needs accumulate = 1 (the moments count accumulated frames)");
    if (c->optSampleChunks >= 2) return fail(c, RT_E_STATE, "rtDispatchAdaptive: a pixel list runs whole pixels; sampleChunks is forced to 2 or more");
    AdaptiveCall ad; ad.threshold = threshold; ad.minFrames = minFrames; ad.maxFrames = maxFrames; ad.active = 0;
    rc = dispatchLocal(c, RT_KERNEL_RAYTRACE, gx, gy, gz, 1, &ad);
    if (rc != RT_OK) return rc;
    if (activePixels) *activePixels = (int64_t)ad.active;
    return RT_OK;
}

int rtDisplayMean(RtContext* c, uint8_t* dst, size_t bytes)
{
    if (!c || !dst) return fail(c, RT_E_INVALID, "rtDisplayMean: bad argument");
    if (!c->accum.p) return fail(c, RT_E_STATE, "rtDisplayMean: rtResize has not been called");
    if (bytes != (size_t)c->width * c->height * 4) return fail(c, RT_E_INVALID, "rtDisplayMean: bytes must equal W*H*4");
    return displayTo(c, [&](size_t n) -> int
    {
        CK(c->snap.ensure(n));                              // the pipelined readback's snapshot image is free here (the copy was waited for)
        RT_LAUNCH((unsigned)((n + 255) / 256), 256, 0, c->stream, k_mean_image, c->accum.p, c->snap.p, n);
        encodeDisplay(c, c->snap.p, n, 1.0f);
        return RT_OK;
    }, dst, bytes);
}

// ---- closest-hit and occlusion queries (rtTraceRays, rtTraceOcclusion, rt_kernel_query.cuh) -----------------------------------------
static int stagedH2D(RtContext* c, void* dst, const void* src, size_t bytes);
static int stagedD2H(RtContext* c, void* dst, const void* src, size_t bytes);

// The host form of a batch call: n records in batches of `chunk` through the device buffers dIn and dOut — each batch copied in
// (inBytes per record; none with inBytes = 0, for a call whose input went to the device whole), run by local(i0, m) on records
// i0 .. i0 + m - 1 and copied out (outBytes per record) — then one synchronise
extern "C++" {
template <class Local>
static int hostBatches(RtContext* c, int n, int chunk, void* dIn, const void* in, size_t inBytes, const void* dOut, void* out, size_t outBytes,
                       Local local)
{
    int rc;
    for (int i0 = 0; i0 < n; i0 += chunk)
    {
        const int m = n - i0 < chunk ? n - i0 : chunk;
        if ((rc = stagedH2D(c, dIn, static_cast<const char*>(in) + (size_t)i0 * inBytes, (size_t)m * inBytes)) != RT_OK) return rc;
        if ((rc = local(i0, m)) != RT_OK) return rc;
        if ((rc = stagedD2H(c, static_cast<char*>(out) + (size_t)i0 * outBytes, dOut, (size_t)m * outBytes)) != RT_OK) return rc;
    }
    CK(cudaStreamSynchronize(c->stream));
    return RT_OK;
}
} // extern "C++"

static int traceArgs(RtContext* c, const char* what, const void* rays, const void* hits, int n, int flags)
{
    int rc = refuseMember(c, what); if (rc != RT_OK) return rc;
    if (n < 0 || (n > 0 && (!rays || !hits))) return fail(c, RT_E_INVALID, std::string(what) + ": bad argument (n < 0, or rays / hits NULL)");
    if (flags != 0 && flags != RT_TRACE_NO_CULL) return fail(c, RT_E_INVALID, std::string(what) + ": flags must be 0 or RT_TRACE_NO_CULL");
    return RT_OK;
}

// n rays (Q.rays -> Q.hits) or, with `occlusion`, n segments (Q.segs -> Q.occluded) in device memory of this context's GPU;
// asynchronous on the context's stream.  RtStats.rays grows by n through the kernel's counters; no timing events, so dispatches /
// kernelMs stay the camera kernels'.
static int queryLocal(RtContext* c, const char* what, QueryParams& Q, int n, int flags, bool occlusion)
{
    int rc = prepareQueryScene(c, what); if (rc != RT_OK) return rc;
    const DevParams P = queryParams(c);
    Q.n = (unsigned int)n; Q.noCull = flags & RT_TRACE_NO_CULL;
    Q.box = sceneBounds(c);
    cudaError_t e = occlusion ? query_launch<true>(P, Q, c->numSMs, c->stream) : query_launch<false>(P, Q, c->numSMs, c->stream);
    if (e != cudaSuccess) return failCuda(c, e, occlusion ? "rtTraceOcclusion launch" : "rtTraceRays launch");
    return RT_OK;
}

static int traceLocal(RtContext* c, const RtRay* dRays, RtRayHit* dHits, int n, int flags)
{
    QueryParams Q = {};
    Q.rays = dRays; Q.hits = dHits;
    return queryLocal(c, "rtTraceRays", Q, n, flags, false);
}

static int occlusionLocal(RtContext* c, const RtRaySegment* dSegs, unsigned char* dOccluded, int n, int flags)
{
    QueryParams Q = {};
    Q.segs = dSegs; Q.occluded = dOccluded;
    return queryLocal(c, "rtTraceOcclusion", Q, n, flags, true);
}

// The device buffers of the host forms: one batch of at most RT_TRACE_CHUNK_RAYS records, 72 bytes each (72 MiB at most)
static int queryBuffers(RtContext* c, int chunk)
{
    if (c->queryRays.cap < (size_t)chunk) { CK(c->queryRays.ensure((size_t)chunk)); CK(c->queryHits.ensure((size_t)chunk)); }
    return RT_OK;
}

int rtTraceRays(RtContext* c, const RtRay* rays, int n, RtRayHit* hits, int flags)
{
    if (!c) return RT_E_INVALID;
    int rc = traceArgs(c, "rtTraceRays", rays, hits, n, flags); if (rc != RT_OK) return rc;
    if (n == 0) return RT_OK;
    CK(cudaSetDevice(c->device));
    // batches of at most RT_TRACE_CHUNK_RAYS through device buffers of that size, kept by the context (72 MB at most)
    const int chunk = n < RT_TRACE_CHUNK_RAYS ? n : RT_TRACE_CHUNK_RAYS;
    if ((rc = queryBuffers(c, chunk)) != RT_OK) return rc;
    return hostBatches(c, n, chunk, c->queryRays.p, rays, sizeof(RtRay), c->queryHits.p, hits, sizeof(RtRayHit),
                       [&](int, int m) { return traceLocal(c, c->queryRays.p, c->queryHits.p, m, flags); });
}

int rtTraceRaysDevice(RtContext* c, const void* dRays, void* dHits, int n, int flags)
{
    if (!c) return RT_E_INVALID;
    int rc = traceArgs(c, "rtTraceRaysDevice", dRays, dHits, n, flags); if (rc != RT_OK) return rc;
    if (((uintptr_t)dRays & 3u) || ((uintptr_t)dHits & 15u)) return fail(c, RT_E_INVALID, "rtTraceRaysDevice: dRays must be 4-byte and dHits 16-byte aligned");
    if (n == 0) return RT_OK;
    CK(cudaSetDevice(c->device));
    return traceLocal(c, (const RtRay*)dRays, (RtRayHit*)dHits, n, flags);
}

// The segments travel in queryHits (28 of its 48 bytes per record) and the answers in queryRays (1 of 24), so an occlusion batch needs
// no memory beyond what a closest-hit batch of the same size keeps.
int rtTraceOcclusion(RtContext* c, const RtRaySegment* segs, int n, uint8_t* occluded, int flags)
{
    if (!c) return RT_E_INVALID;
    int rc = traceArgs(c, "rtTraceOcclusion", segs, occluded, n, flags); if (rc != RT_OK) return rc;
    if (n == 0) return RT_OK;
    CK(cudaSetDevice(c->device));
    const int chunk = n < RT_TRACE_CHUNK_RAYS ? n : RT_TRACE_CHUNK_RAYS;
    if ((rc = queryBuffers(c, chunk)) != RT_OK) return rc;
    RtRaySegment* dSegs = reinterpret_cast<RtRaySegment*>(c->queryHits.p);
    unsigned char* dOccluded = reinterpret_cast<unsigned char*>(c->queryRays.p);
    return hostBatches(c, n, chunk, dSegs, segs, sizeof(RtRaySegment), dOccluded, occluded, 1,
                       [&](int, int m) { return occlusionLocal(c, dSegs, dOccluded, m, flags); });
}

int rtTraceOcclusionDevice(RtContext* c, const void* dSegs, void* dOccluded, int n, int flags)
{
    if (!c) return RT_E_INVALID;
    int rc = traceArgs(c, "rtTraceOcclusionDevice", dSegs, dOccluded, n, flags); if (rc != RT_OK) return rc;
    if ((uintptr_t)dSegs & 3u) return fail(c, RT_E_INVALID, "rtTraceOcclusionDevice: dSegs must be 4-byte aligned");
    if (n == 0) return RT_OK;
    CK(cudaSetDevice(c->device));
    return occlusionLocal(c, (const RtRaySegment*)dSegs, (unsigned char*)dOccluded, n, flags);
}

// ---- radiance along caller-supplied rays (rtTracePaths, k_trace_paths in rt_kernel_query.cuh) ------------------------------------------
// What both forms of rtTracePaths and rtBakeProbes check; `items` names the input pointer ("rays", "positions")
static int batchArgs(RtContext* c, const char* what, const char* items, const void* in, const void* out, int n, int samples)
{
    int rc = refuseMember(c, what); if (rc != RT_OK) return rc;
    if (n < 0 || (n > 0 && (!in || !out))) return fail(c, RT_E_INVALID, std::string(what) + ": bad argument (n < 0, or " + items + " / out NULL)");
    if (samples < 1 || samples > RT_MAX_BATCH_SAMPLES) return fail(c, RT_E_INVALID, std::string(what) + ": samples must be 1 .. RT_MAX_BATCH_SAMPLES");
    return RT_OK;
}

// A kernel-1-style loop traces one segment even with a negative bound, where the reference's loop (HL:484) traces none
static int bounceLimit(RtContext* c, const char* what)
{
    if (c->P.MaxBounceCount < 0 || c->P.MaxBounceCount > 200) return fail(c, RT_E_STATE, std::string(what) + ": MaxBounceCount must be 0 .. 200 (as rtDispatch)");
    return RT_OK;
}

// n rays in device memory of this context's GPU -> n radiances; asynchronous on the context's stream.  RtStats.rays grows by the
// segments traced, through the kernel's counters; no timing events, so dispatches / kernelMs stay the camera kernels'.
static int pathsLocal(RtContext* c, const RtPathRay* dRays, RtPathRadiance* dOut, int n, int samples)
{
    int rc = bounceLimit(c, "rtTracePaths"); if (rc != RT_OK) return rc;
    if ((rc = prepareQueryScene(c, "rtTracePaths")) != RT_OK) return rc;
    const DevParams P = queryParams(c);
    PathParams Q = {};
    Q.rays = dRays; Q.out = dOut; Q.n = (unsigned int)n; Q.samples = samples;
    Q.box = sceneBounds(c);
    cudaError_t e = paths_launch(P, Q, c->numSMs, c->stream);
    if (e != cudaSuccess) return failCuda(c, e, "rtTracePaths launch");
    return RT_OK;
}

// The rays travel in queryHits (28 of its 48 bytes per record) and the results in queryRays (16 of 24), so a path batch needs no
// memory beyond what a closest-hit batch of the same size keeps.
int rtTracePaths(RtContext* c, const RtPathRay* rays, int n, int samples, RtPathRadiance* out)
{
    if (!c) return RT_E_INVALID;
    int rc = batchArgs(c, "rtTracePaths", "rays", rays, out, n, samples); if (rc != RT_OK) return rc;
    if (n == 0) return RT_OK;
    CK(cudaSetDevice(c->device));
    const int chunk = n < RT_TRACE_CHUNK_RAYS ? n : RT_TRACE_CHUNK_RAYS;
    if ((rc = queryBuffers(c, chunk)) != RT_OK) return rc;
    RtPathRay* dRays = reinterpret_cast<RtPathRay*>(c->queryHits.p);
    RtPathRadiance* dOut = reinterpret_cast<RtPathRadiance*>(c->queryRays.p);
    return hostBatches(c, n, chunk, dRays, rays, sizeof(RtPathRay), dOut, out, sizeof(RtPathRadiance),
                       [&](int, int m) { return pathsLocal(c, dRays, dOut, m, samples); });
}

int rtTracePathsDevice(RtContext* c, const void* dRays, void* dOut, int n, int samples)
{
    if (!c) return RT_E_INVALID;
    int rc = batchArgs(c, "rtTracePathsDevice", "rays", dRays, dOut, n, samples); if (rc != RT_OK) return rc;
    if (((uintptr_t)dRays & 3u) || ((uintptr_t)dOut & 15u)) return fail(c, RT_E_INVALID, "rtTracePathsDevice: dRays must be 4-byte and dOut 16-byte aligned");
    if (n == 0) return RT_OK;
    CK(cudaSetDevice(c->device));
    return pathsLocal(c, (const RtPathRay*)dRays, (RtPathRadiance*)dOut, n, samples);
}

// ---- light probes (rtBakeProbes, rt_kernel_probes.cuh) -------------------------------------------------------------------------------
// The probes of one launch: as many as RT_PROBE_SCRATCH_CHUNKS chunk records hold
static int probesPerLaunch(int samples)
{
    return RT_PROBE_SCRATCH_CHUNKS / ((samples + (int)RT_PROBE_CHUNK - 1) / (int)RT_PROBE_CHUNK);
}

// n probes in device memory of this context's GPU, the first of them probe p0 of the call -> n RtProbeSH, in launches of at most
// probesPerLaunch probes; asynchronous on the context's stream.  The scratch is allocated (or grown) here and nothing else is.
static int probesLocal(RtContext* c, const float* dPositions, RtProbeSH* dOut, int n, int samples, uint32_t seed, unsigned int p0)
{
    int rc = bounceLimit(c, "rtBakeProbes"); if (rc != RT_OK) return rc;
    if ((rc = prepareQueryScene(c, "rtBakeProbes")) != RT_OK) return rc;
    const unsigned int chunks = ((unsigned int)samples + RT_PROBE_CHUNK - 1) / RT_PROBE_CHUNK;
    const int per = probesPerLaunch(samples);
    const int first = n < per ? n : per;
    if (c->probeScratch.cap < (size_t)first * chunks * PROBE_WORDS) CK(c->probeScratch.ensure((size_t)first * chunks * PROBE_WORDS));
    const DevParams P = queryParams(c);
    ProbeParams Q = {};
    Q.scratch = c->probeScratch.p; Q.chunks = chunks; Q.samples = samples; Q.seed = seed;
    Q.box = sceneBounds(c);
    for (int i0 = 0; i0 < n; i0 += per)
    {
        Q.positions = dPositions + 3 * (size_t)i0; Q.out = dOut + i0;
        Q.n = (unsigned int)(n - i0 < per ? n - i0 : per); Q.p0 = p0 + (unsigned int)i0;
        cudaError_t e = probes_launch(P, Q, c->numSMs, c->stream);
        if (e != cudaSuccess) return failCuda(c, e, "rtBakeProbes launch");
    }
    return RT_OK;
}

int rtBakeProbes(RtContext* c, const float* positions, int n, int samples, uint32_t seed, RtProbeSH* out)
{
    if (!c) return RT_E_INVALID;
    int rc = batchArgs(c, "rtBakeProbes", "positions", positions, out, n, samples); if (rc != RT_OK) return rc;
    if (n == 0) return RT_OK;
    CK(cudaSetDevice(c->device));
    const int per = probesPerLaunch(samples);
    const int chunk = n < per ? n : per;
    if (c->probeOut.cap < (size_t)chunk) { CK(c->probePositions.ensure(3 * (size_t)chunk)); CK(c->probeOut.ensure((size_t)chunk)); }
    return hostBatches(c, n, chunk, c->probePositions.p, positions, 3 * sizeof(float), c->probeOut.p, out, sizeof(RtProbeSH),
                       [&](int i0, int m) { return probesLocal(c, c->probePositions.p, c->probeOut.p, m, samples, seed, (unsigned int)i0); });
}

int rtBakeProbesDevice(RtContext* c, const void* dPositions, void* dOut, int n, int samples, uint32_t seed)
{
    if (!c) return RT_E_INVALID;
    int rc = batchArgs(c, "rtBakeProbesDevice", "positions", dPositions, dOut, n, samples); if (rc != RT_OK) return rc;
    if (((uintptr_t)dPositions & 3u) || ((uintptr_t)dOut & 15u)) return fail(c, RT_E_INVALID, "rtBakeProbesDevice: dPositions must be 4-byte and dOut 16-byte aligned");
    if (n == 0) return RT_OK;
    CK(cudaSetDevice(c->device));
    return probesLocal(c, (const float*)dPositions, (RtProbeSH*)dOut, n, samples, seed, 0u);
}

// ---- reflection probes (rtBakeCubemaps, rt_kernel_cubemaps.cuh) -------------------------------------------------------------------
// The texels of one launch: as many as RT_CUBE_SCRATCH_CHUNKS chunk records hold
static int texelsPerLaunch(int samples)
{
    return RT_CUBE_SCRATCH_CHUNKS / ((samples + (int)RT_PROBE_CHUNK - 1) / (int)RT_PROBE_CHUNK);
}

// What both forms check beyond batchArgs; *texels gets n * 6 * faceSize^2
static int cubemapArgs(RtContext* c, const char* what, const void* positions, const void* out, int n, int faceSize, int samples, int* texels)
{
    int rc = batchArgs(c, what, "positions", positions, out, n, samples); if (rc != RT_OK) return rc;
    if (faceSize < 1 || faceSize > RT_CUBE_MAX_FACE) return fail(c, RT_E_INVALID, std::string(what) + ": faceSize must be 1 .. RT_CUBE_MAX_FACE");
    const long long t = (long long)n * 6 * faceSize * faceSize;
    if (t > 0x7fffffffLL) return fail(c, RT_E_INVALID, std::string(what) + ": n * 6 * faceSize^2 must be at most 2^31 - 1 texels");
    *texels = (int)t;
    return RT_OK;
}

// Texels t0 .. t0 + n - 1 of a cube-map or lightmap call (Q: the call's parameters, with Q.points, if set, at texel t0's point) -> dOut,
// in device memory of this context's GPU, in launches of at most texelsPerLaunch texels; asynchronous on the context's stream.  The
// scratch is allocated (or grown) here and nothing else is.
static int texelLaunches(RtContext* c, const char* what, CubeParams Q, RtCubeTexel* dOut, int n, unsigned int t0)
{
    int rc = bounceLimit(c, what); if (rc != RT_OK) return rc;
    if ((rc = prepareQueryScene(c, what)) != RT_OK) return rc;
    const unsigned int chunks = ((unsigned int)Q.samples + RT_PROBE_CHUNK - 1) / RT_PROBE_CHUNK;
    const int per = texelsPerLaunch(Q.samples);
    const int first = n < per ? n : per;
    if (c->probeScratch.cap < (size_t)first * chunks * CUBE_WORDS) CK(c->probeScratch.ensure((size_t)first * chunks * CUBE_WORDS));
    const DevParams P = queryParams(c);
    const RtSurfacePoint* points = Q.points;
    Q.scratch = c->probeScratch.p; Q.chunks = chunks;
    Q.box = sceneBounds(c);
    for (int i0 = 0; i0 < n; i0 += per)
    {
        Q.out = dOut + i0; Q.n = (unsigned int)(n - i0 < per ? n - i0 : per); Q.t0 = t0 + (unsigned int)i0;
        if (points) Q.points = points + i0;
        cudaError_t e = cubemaps_launch(P, Q, c->numSMs, c->stream);
        if (e != cudaSuccess) return failCuda(c, e, (std::string(what) + " launch").c_str());
    }
    return RT_OK;
}

// Texels t0 .. t0 + n - 1 of the call (dPositions: the call's probes; dOut: texel t0's record)
static int cubemapsLocal(RtContext* c, const float* dPositions, RtCubeTexel* dOut, int n, unsigned int t0, int faceSize, int samples, uint32_t seed)
{
    CubeParams Q = {};
    Q.positions = dPositions; Q.faceSize = (unsigned int)faceSize; Q.samples = samples; Q.seed = seed;
    return texelLaunches(c, "rtBakeCubemaps", Q, dOut, n, t0);
}

// The positions go to the device once; the texels come back a launch at a time
int rtBakeCubemaps(RtContext* c, const float* positions, int n, int faceSize, int samples, uint32_t seed, RtCubeTexel* out)
{
    if (!c) return RT_E_INVALID;
    int texels = 0;
    int rc = cubemapArgs(c, "rtBakeCubemaps", positions, out, n, faceSize, samples, &texels); if (rc != RT_OK) return rc;
    if (n == 0) return RT_OK;
    CK(cudaSetDevice(c->device));
    const int per = texelsPerLaunch(samples);
    const int chunk = texels < per ? texels : per;
    if (c->probePositions.cap < 3 * (size_t)n) CK(c->probePositions.ensure(3 * (size_t)n));
    if (c->cubeOut.cap < (size_t)chunk) CK(c->cubeOut.ensure((size_t)chunk));
    if ((rc = stagedH2D(c, c->probePositions.p, positions, 3 * sizeof(float) * (size_t)n)) != RT_OK) return rc;
    return hostBatches(c, texels, chunk, nullptr, nullptr, 0, c->cubeOut.p, out, sizeof(RtCubeTexel),
                       [&](int i0, int m) { return cubemapsLocal(c, c->probePositions.p, c->cubeOut.p, m, (unsigned int)i0, faceSize, samples, seed); });
}

int rtBakeCubemapsDevice(RtContext* c, const void* dPositions, void* dOut, int n, int faceSize, int samples, uint32_t seed)
{
    if (!c) return RT_E_INVALID;
    int texels = 0;
    int rc = cubemapArgs(c, "rtBakeCubemapsDevice", dPositions, dOut, n, faceSize, samples, &texels); if (rc != RT_OK) return rc;
    if (((uintptr_t)dPositions & 3u) || ((uintptr_t)dOut & 15u)) return fail(c, RT_E_INVALID, "rtBakeCubemapsDevice: dPositions must be 4-byte and dOut 16-byte aligned");
    if (n == 0) return RT_OK;
    CK(cudaSetDevice(c->device));
    return cubemapsLocal(c, (const float*)dPositions, (RtCubeTexel*)dOut, texels, 0u, faceSize, samples, seed);
}

// ---- lightmaps (rtBakeLightmap: surface texels of k_bake_cubemaps, rt_kernel_cubemaps.cuh) ---------------------------------------------
// Texels p0 .. p0 + n - 1 of the call (dPoints, dOut: texel p0's point and record); the checks, scratch and launches of rtBakeCubemaps
static int lightmapLocal(RtContext* c, const RtSurfacePoint* dPoints, RtCubeTexel* dOut, int n, unsigned int p0, int samples, uint32_t seed)
{
    CubeParams Q = {};
    Q.points = dPoints; Q.samples = samples; Q.seed = seed;
    return texelLaunches(c, "rtBakeLightmap", Q, dOut, n, p0);
}

// The points travel in queryRays (24 of its 24 bytes per record) and the texels in queryHits (16 of 48), so a lightmap batch needs no
// memory beyond what a closest-hit batch of the same size keeps.
int rtBakeLightmap(RtContext* c, const RtSurfacePoint* points, int n, int samples, uint32_t seed, RtCubeTexel* out)
{
    if (!c) return RT_E_INVALID;
    int rc = batchArgs(c, "rtBakeLightmap", "points", points, out, n, samples); if (rc != RT_OK) return rc;
    if (n == 0) return RT_OK;
    CK(cudaSetDevice(c->device));
    const int chunk = n < RT_TRACE_CHUNK_RAYS ? n : RT_TRACE_CHUNK_RAYS;
    if ((rc = queryBuffers(c, chunk)) != RT_OK) return rc;
    RtSurfacePoint* dPoints = reinterpret_cast<RtSurfacePoint*>(c->queryRays.p);
    RtCubeTexel* dOut = reinterpret_cast<RtCubeTexel*>(c->queryHits.p);
    return hostBatches(c, n, chunk, dPoints, points, sizeof(RtSurfacePoint), dOut, out, sizeof(RtCubeTexel),
                       [&](int i0, int m) { return lightmapLocal(c, dPoints, dOut, m, (unsigned int)i0, samples, seed); });
}

int rtBakeLightmapDevice(RtContext* c, const void* dPoints, void* dOut, int n, int samples, uint32_t seed)
{
    if (!c) return RT_E_INVALID;
    int rc = batchArgs(c, "rtBakeLightmapDevice", "points", dPoints, dOut, n, samples); if (rc != RT_OK) return rc;
    if (((uintptr_t)dPoints & 3u) || ((uintptr_t)dOut & 15u)) return fail(c, RT_E_INVALID, "rtBakeLightmapDevice: dPoints must be 4-byte and dOut 16-byte aligned");
    if (n == 0) return RT_OK;
    CK(cudaSetDevice(c->device));
    return lightmapLocal(c, (const RtSurfacePoint*)dPoints, (RtCubeTexel*)dOut, n, 0u, samples, seed);
}

// ---- first-hit feature images and the camera's own rays (rtDispatchFeatures, rtCameraRays, rt_kernel_features.cuh) ---------------------
// The image a camera call works on: rtResize done, "Resolution" equal to it, within the kernels' coordinate range
static int cameraImage(RtContext* c, const char* what)
{
    if (c->width == 0) return fail(c, RT_E_STATE, std::string(what) + ": rtResize has not been called");
    if ((int)c->P.W != c->width || (int)c->P.H != c->height) return fail(c, RT_E_STATE, std::string(what) + ": Resolution does not match the render textures");
    if (c->P.W > 65535u || c->P.H > 65535u) return fail(c, RT_E_STATE, std::string(what) + ": a resolution above 65535 is not supported");
    return RT_OK;
}

int rtDispatchFeatures(RtContext* c, int gx, int gy, int gz)
{
    if (!c) return RT_E_INVALID;
    if (gx < 0 || gy < 0 || gz < 0) return fail(c, RT_E_INVALID, "rtDispatchFeatures: bad argument");
    int rc = refuseGroup(c, "rtDispatchFeatures"); if (rc != RT_OK) return rc;
    if ((rc = cameraImage(c, "rtDispatchFeatures")) != RT_OK) return rc;
    CK(cudaSetDevice(c->device));
    const unsigned W = c->P.W, H = c->P.H;
    if (!c->featureFrame.p)                                    // the first call allocates the three images, zero-filled
    {
        const size_t n = (size_t)W * H;
        if ((rc = allocateZeroed(c, c->featureFrame, n)) != RT_OK || (rc = allocateZeroed(c, c->accumAlbedo, n)) != RT_OK ||
            (rc = allocateZeroed(c, c->accumNormal, n)) != RT_OK) return rc;
    }
    unsigned limX, limY;
    groupLimits(gx, gy, gz, W, H, limX, limY);
    if (limX == 0 || limY == 0) return RT_OK;
    if ((rc = prepareQueryScene(c, "rtDispatchFeatures")) != RT_OK) return rc;
    DevParams P = queryParams(c);
    P.limX = limX; P.limY = limY;
    P.tileRank = c->tileRank; P.tileWorld = c->tileWorld; P.bandRows = c->bandRows;
    P.zeroDefocus = 0;
    FeatureParams F = {};
    F.features = c->featureFrame.p; F.accumAlbedo = c->accumAlbedo.p; F.accumNormal = c->accumNormal.p;
    cudaError_t e = features_launch(P, F, c->numSMs, c->stream);
    if (e != cudaSuccess) return failCuda(c, e, "rtDispatchFeatures launch");
    return RT_OK;
}

// What both forms of rtCameraRays check before anything is allocated or launched
static int cameraRaysArgs(RtContext* c, const char* what, const void* rays, size_t bytes)
{
    int rc = refuseMember(c, what); if (rc != RT_OK) return rc;
    if (!rays) return fail(c, RT_E_INVALID, std::string(what) + ": rays is NULL");
    if ((rc = cameraImage(c, what)) != RT_OK) return rc;
    if (bytes != (size_t)c->width * c->height * sizeof(RtPathRay)) return fail(c, RT_E_INVALID, std::string(what) + ": bytes must equal W*H*28");
    return RT_OK;
}

// W*H rays of the whole image into device memory; asynchronous on the context's stream
static int cameraRaysLocal(RtContext* c, RtPathRay* dRays)
{
    DevParams P = c->P;
    P.limX = P.W; P.limY = P.H;
    P.tileRank = 0; P.tileWorld = 1; P.bandRows = 1;          // the whole image: a query about the camera, not a render
    P.zeroDefocus = 0;
    FeatureParams F = {};
    F.rays = dRays;
    cudaError_t e = camera_rays_launch(P, F, c->stream);
    if (e != cudaSuccess) return failCuda(c, e, "rtCameraRays launch");
    return RT_OK;
}

int rtCameraRays(RtContext* c, RtPathRay* rays, size_t bytes)
{
    if (!c) return RT_E_INVALID;
    int rc = cameraRaysArgs(c, "rtCameraRays", rays, bytes); if (rc != RT_OK) return rc;
    CK(cudaSetDevice(c->device));
    CK(c->cameraRays.ensure((size_t)c->width * c->height));
    if ((rc = cameraRaysLocal(c, c->cameraRays.p)) != RT_OK) return rc;
    if ((rc = stagedD2H(c, rays, c->cameraRays.p, bytes)) != RT_OK) return rc;
    CK(cudaStreamSynchronize(c->stream));
    return RT_OK;
}

int rtCameraRaysDevice(RtContext* c, void* dRays, size_t bytes)
{
    if (!c) return RT_E_INVALID;
    int rc = cameraRaysArgs(c, "rtCameraRaysDevice", dRays, bytes); if (rc != RT_OK) return rc;
    if ((uintptr_t)dRays & 3u) return fail(c, RT_E_INVALID, "rtCameraRaysDevice: dRays must be 4-byte aligned");
    CK(cudaSetDevice(c->device));
    return cameraRaysLocal(c, (RtPathRay*)dRays);
}

// ---- the a-trous denoiser (rtDenoise, rt_kernel_denoise.cuh) --------------------------------------------------------------------------
static bool finiteAbove0(float v) { return v > 0.0f && v < INFINITY; }

// The passes of the a-trous filter: pass k reads the image pass k - 1 wrote, 2^k pixels apart, with the colour weight cK0 * 4^k
static void passSchedule(int iterations, float cK0, DenoisePass* passes)
{
    for (int k = 0; k < iterations; k++)
    {
        passes[k].cK = cK0 * (float)(1u << (2 * k));
        passes[k].rd1 = 1.0f / (float)(1u << k); passes[k].rd2 = 1.0f / (float)(2u << k);
        passes[k].step = 1 << k; passes[k].src = k & 1; passes[k].last = k == iterations - 1;
    }
}

int rtDenoise(RtContext* c, int useAccumulated, int iterations, float sigmaColour, float sigmaNormal, float sigmaDepth)
{
    if (!c) return RT_E_INVALID;
    if (useAccumulated != 0 && useAccumulated != 1) return fail(c, RT_E_INVALID, "rtDenoise: useAccumulated must be 0 or 1");
    if (iterations < 1 || iterations > RT_DENOISE_MAX_ITERATIONS) return fail(c, RT_E_INVALID, "rtDenoise: iterations must be 1 .. RT_DENOISE_MAX_ITERATIONS");
    if (!finiteAbove0(sigmaColour) || !finiteAbove0(sigmaNormal) || !finiteAbove0(sigmaDepth)) return fail(c, RT_E_INVALID, "rtDenoise: every sigma must be finite and > 0");
    // the constants of include/rt_b200.h, one binary32 operation each
    const float invC = 1.0f / (sigmaColour * sigmaColour), invN = 1.0f / (sigmaNormal * sigmaNormal), invZ = 1.0f / sigmaDepth;
    DenoisePass passes[RT_DENOISE_MAX_ITERATIONS];
    passSchedule(iterations, invC, passes);
    if (!(passes[iterations - 1].cK < INFINITY) || !(invN < INFINITY) || !(invZ < INFINITY))
        return fail(c, RT_E_INVALID, "rtDenoise: a sigma too small: invC * 4^(iterations-1), 1 / sigmaNormal^2 or 1 / sigmaDepth is not finite");
    int rc = refuseGroup(c, "rtDenoise"); if (rc != RT_OK) return rc;
    if ((rc = cameraImage(c, "rtDenoise")) != RT_OK) return rc;
    if (!c->featureFrame.p) return fail(c, RT_E_STATE, "rtDenoise: no rtDispatchFeatures yet");
    if (c->tileWorld > 1) return fail(c, RT_E_STATE, "rtDenoise: the images of a context with rtSetTile world > 1 hold its own bands only");
    CK(cudaSetDevice(c->device));
    const size_t n = (size_t)c->width * c->height;
    CK(c->denoised.ensure(n)); CK(c->denoiseScratch.ensure(3 * n));
    DenoiseParams P = {};
    P.colour = useAccumulated ? c->accum.p : c->frame.p;
    P.albedo = c->accumAlbedo.p; P.normal = c->accumNormal.p; P.features = c->featureFrame.p;
    P.e[0] = c->denoiseScratch.p; P.e[1] = c->denoiseScratch.p + n; P.guide = c->denoiseScratch.p + 2 * n;
    P.out = c->denoised.p;
    P.W = c->width; P.H = c->height; P.useAccumulated = useAccumulated;
    P.invN = invN; P.invZ = invZ;
    cudaError_t e = denoise_launch(P, passes, iterations, c->stream);
    if (e != cudaSuccess) return failCuda(c, e, "rtDenoise launch");
    return RT_OK;
}

// ---- the temporal denoiser (rtDenoiseTemporal, rt_kernel_temporal.cuh) ------------------------------------------------------------------
// The previous camera's inverse affine map as include/rt_b200.h states it: adjugate / determinant in float64, each entry rounded once
static void temporalInverse(const float* m, float inv[12])
{
    const double a00 = m[0], a01 = m[4], a02 = m[8], a10 = m[1], a11 = m[5], a12 = m[9], a20 = m[2], a21 = m[6], a22 = m[10];
    const double t[3] = {m[12], m[13], m[14]};
    const double c00 = a11 * a22 - a12 * a21, c01 = a12 * a20 - a10 * a22, c02 = a10 * a21 - a11 * a20;
    const double c10 = a02 * a21 - a01 * a22, c11 = a00 * a22 - a02 * a20, c12 = a01 * a20 - a00 * a21;
    const double c20 = a01 * a12 - a02 * a11, c21 = a02 * a10 - a00 * a12, c22 = a00 * a11 - a01 * a10;
    const double det = (a00 * c00 + a01 * c01) + a02 * c02;
    const double R[3][3] = {{c00 / det, c10 / det, c20 / det}, {c01 / det, c11 / det, c21 / det}, {c02 / det, c12 / det, c22 / det}};
    for (int r = 0; r < 3; r++)
    {
        for (int k = 0; k < 3; k++) inv[4 * r + k] = (float)R[r][k];
        inv[4 * r + 3] = (float)-((R[r][0] * t[0] + R[r][1] * t[1]) + R[r][2] * t[2]);
    }
}

int rtDenoiseTemporal(RtContext* c, int iterations, float sigmaLuminance, float sigmaNormal, float sigmaDepth, float alpha, int resetHistory)
{
    if (!c) return RT_E_INVALID;
    if (iterations < 1 || iterations > RT_DENOISE_MAX_ITERATIONS) return fail(c, RT_E_INVALID, "rtDenoiseTemporal: iterations must be 1 .. RT_DENOISE_MAX_ITERATIONS");
    if (!finiteAbove0(sigmaLuminance) || !finiteAbove0(sigmaNormal) || !finiteAbove0(sigmaDepth)) return fail(c, RT_E_INVALID, "rtDenoiseTemporal: every sigma must be finite and > 0");
    if (!(alpha > 0.0f && alpha <= 1.0f)) return fail(c, RT_E_INVALID, "rtDenoiseTemporal: alpha must be in (0, 1]");
    if (resetHistory != 0 && resetHistory != 1) return fail(c, RT_E_INVALID, "rtDenoiseTemporal: resetHistory must be 0 or 1");
    const float invN = 1.0f / (sigmaNormal * sigmaNormal), invZ = 1.0f / sigmaDepth, invL = 1.0f / sigmaLuminance;
    if (!(invN < INFINITY) || !(invZ < INFINITY) || !(invL < INFINITY))
        return fail(c, RT_E_INVALID, "rtDenoiseTemporal: a sigma too small: 1 / sigmaNormal^2, 1 / sigmaDepth or 1 / sigmaLuminance is not finite");
    int rc = refuseGroup(c, "rtDenoiseTemporal"); if (rc != RT_OK) return rc;
    if ((rc = cameraImage(c, "rtDenoiseTemporal")) != RT_OK) return rc;
    if (!c->featureFrame.p) return fail(c, RT_E_STATE, "rtDenoiseTemporal: no rtDispatchFeatures yet");
    if (c->tileWorld > 1) return fail(c, RT_E_STATE, "rtDenoiseTemporal: the images of a context with rtSetTile world > 1 hold its own bands only");
    CK(cudaSetDevice(c->device));
    const size_t n = (size_t)c->width * c->height;
    if (!c->temporalHist.p) c->temporalHistory = false;
    CK(c->denoised.ensure(n)); CK(c->denoiseScratch.ensure(3 * n)); CK(c->temporalFrame.ensure(n)); CK(c->temporalHist.ensure(6 * n));
    DenoisePass passes[RT_DENOISE_MAX_ITERATIONS];
    passSchedule(iterations, 0.0f, passes);                                        // no colour weight: the variance guides instead
    const int cur = c->temporalSet ^ 1;
    float4* const set[2] = {c->temporalHist.p, c->temporalHist.p + 3 * n};       // guide, moments, colour history
    TemporalParams T = {};
    T.colour = c->frame.p; T.features = c->featureFrame.p;
    T.e = c->denoiseScratch.p; T.out = c->denoised.p; T.frame = c->temporalFrame.p;
    T.guide = set[cur]; T.mom = set[cur] + n;
    T.prevGuide = set[cur ^ 1]; T.prevMom = set[cur ^ 1] + n; T.prevColour = set[cur ^ 1] + 2 * n;
    T.W = c->width; T.H = c->height;
    T.alpha = alpha; T.invN = invN; T.invZ = invZ; T.invL = invL;
    T.mode = TEMPORAL_NONE;
    if (c->temporalHistory && !resetHistory)
    {
        if (memcmp(c->temporalCam, c->P.cam, sizeof(c->temporalCam)) == 0 && memcmp(c->temporalVP, c->P.ViewParams, sizeof(c->temporalVP)) == 0)
            T.mode = TEMPORAL_STATIC;
        else
        {
            T.mode = TEMPORAL_REPROJECT;
            temporalInverse(c->temporalCam, T.inv);
            T.prevOrigin[0] = c->temporalCam[12]; T.prevOrigin[1] = c->temporalCam[13]; T.prevOrigin[2] = c->temporalCam[14];
            T.kx = c->temporalVP[2] / c->temporalVP[0]; T.ky = c->temporalVP[2] / c->temporalVP[1];
        }
    }
    TemporalPassParams Pp = {};
    Pp.e[0] = c->denoiseScratch.p; Pp.e[1] = c->denoiseScratch.p + n; Pp.guide = T.guide; Pp.out = c->denoised.p;
    Pp.W = c->width; Pp.H = c->height; Pp.invN = invN; Pp.invZ = invZ;
    Pp.hist = set[cur] + 2 * n; Pp.sigmaL = sigmaLuminance;
    Pp.gv = reinterpret_cast<float*>(c->denoiseScratch.p + 2 * n);                // rtDenoise's guide slot, unused here
    cudaError_t e = temporal_launch(T, c->P, Pp, passes, iterations, c->stream);
    if (e != cudaSuccess) return failCuda(c, e, "rtDenoiseTemporal launch");
    c->temporalSet = cur; c->temporalHistory = true;
    memcpy(c->temporalCam, c->P.cam, sizeof(c->temporalCam)); memcpy(c->temporalVP, c->P.ViewParams, sizeof(c->temporalVP));
    return RT_OK;
}

int rtDisplayDenoised(RtContext* c, uint8_t* dst, size_t bytes)
{
    if (!c || !dst) return fail(c, RT_E_INVALID, "rtDisplayDenoised: bad argument");
    if (!c->denoised.p) return fail(c, RT_E_STATE, "rtDisplayDenoised: no rtDenoise yet");
    if (bytes != (size_t)c->width * c->height * 4) return fail(c, RT_E_INVALID, "rtDisplayDenoised: bytes must equal W*H*4");
    return displayTo(c, [&](size_t n) { encodeDisplay(c, c->denoised.p, n, 1.0f); return RT_OK; }, dst, bytes);      // t / 1 is exact
}

int rtExchangeTiles(RtContext* c)
{
    if (!c) return RT_E_INVALID;
    if (c->leader) return fail(c, RT_E_STATE, "rtExchangeTiles: call it on the context rtCreateMulti returned");
    if (c->tileWorld <= 1) return RT_OK;
    if (!c->comm && c->followers.empty()) return fail(c, RT_E_STATE, "rtExchangeTiles: no communicator (rtCommInit / rtCreateMulti)");
    return exchangeGroup(c);
}

int rtGetUniqueId(void* id, size_t bytes)
{
    if (!id || bytes != RT_UNIQUE_ID_BYTES) return fail(nullptr, RT_E_INVALID, "rtGetUniqueId: id must hold 128 bytes");
    std::string why;
    NcclApi* api = NcclApi::get(why);
    if (!api) return fail(nullptr, RT_E_STATE, "rtGetUniqueId: " + why);
    NcclApi::UniqueId u;
    const int r = api->GetUniqueId(&u);
    if (r != NcclApi::Success) return ncclFail(nullptr, api, r, "ncclGetUniqueId");
    memcpy(id, &u, RT_UNIQUE_ID_BYTES);
    return RT_OK;
}

static void destroyComm(RtContext* c)
{
    if (!c->comm) return;
    std::string why;
    NcclApi* api = NcclApi::get(why);
    cudaSetDevice(c->device);
    cudaStreamSynchronize(c->stream);
    if (api) api->CommDestroy(c->comm);
    c->comm = nullptr; c->commRank = 0; c->commWorld = 1;
}

int rtCommInit(RtContext* c, const void* id, size_t bytes, int rank, int world)
{
    if (!c || !id || bytes != RT_UNIQUE_ID_BYTES || world < 1 || rank < 0 || rank >= world) return fail(c, RT_E_INVALID, "rtCommInit: bad argument");
    if (c->leader || !c->followers.empty()) return fail(c, RT_E_STATE, "rtCommInit: the context belongs to a single-process group (rtCreateMulti), which has its communicator");
    std::string why;
    NcclApi* api = NcclApi::get(why);
    if (!api) return fail(c, RT_E_STATE, "rtCommInit: " + why);
    CK(cudaSetDevice(c->device));
    destroyComm(c);
    NcclApi::UniqueId u; memcpy(&u, id, RT_UNIQUE_ID_BYTES);
    const int r = api->CommInitRank(&c->comm, world, u, rank);
    if (r != NcclApi::Success) { c->comm = nullptr; return ncclFail(c, api, r, "ncclCommInitRank"); }
    c->commRank = rank; c->commWorld = world;
    return rtSetTile(c, rank, world, c->tileWorld == world && c->tileRank == rank ? c->bandRows : 8);
}

int rtCommDestroy(RtContext* c)
{
    if (!c) return RT_E_INVALID;
    if (c->leader || !c->followers.empty()) return fail(c, RT_E_STATE, "rtCommDestroy: a group's communicator lives as long as the group (rtDestroy)");
    destroyComm(c);
    return rtSetTile(c, 0, 1, c->bandRows);
}

int rtCreateMulti(RtContext** out, const int* devices, int nDevices)
{
    if (!out) return fail(nullptr, RT_E_INVALID, "rtCreateMulti: out is NULL");
    *out = nullptr;
    if (nDevices < 1 || nDevices > 64) return fail(nullptr, RT_E_INVALID, "rtCreateMulti: between 1 and 64 devices");
    for (int i = 0; i < nDevices; i++) for (int j = 0; j < i; j++)
        if (devices && devices[i] == devices[j]) return fail(nullptr, RT_E_INVALID, "rtCreateMulti: a device is listed twice (NCCL needs one rank per GPU)");
    std::vector<RtContext*> cs;
    auto undo = [&](int code) { for (RtContext* m : cs) { destroyComm(m); m->leader = nullptr; m->followers.clear(); rtDestroy(m); } return code; };
    for (int i = 0; i < nDevices; i++)
    {
        RtContext* m = nullptr;
        const int rc = rtCreate(&m, devices ? devices[i] : i);
        if (rc != RT_OK) return undo(rc);
        cs.push_back(m);
    }
    if (nDevices > 1)
    {
#ifndef RT_SIMT_EMU
        std::string why;
        NcclApi* api = NcclApi::get(why);
        if (!api) { fail(nullptr, RT_E_STATE, "rtCreateMulti: " + why); return undo(RT_E_STATE); }
        NcclApi::UniqueId u;
        int r = api->GetUniqueId(&u);
        if (r == NcclApi::Success) r = api->GroupStart();
        for (int i = 0; i < nDevices && r == NcclApi::Success; i++)
        {
            cudaSetDevice(cs[i]->device);
            r = api->CommInitRank(&cs[i]->comm, nDevices, u, i);
        }
        if (r == NcclApi::Success) r = api->GroupEnd();
        if (r != NcclApi::Success) { ncclFail(nullptr, api, r, "rtCreateMulti: NCCL communicator"); return undo(RT_E_CUDA); }
#endif
        for (int i = 0; i < nDevices; i++)
        {
            cs[i]->commRank = i; cs[i]->commWorld = nDevices;
            cs[i]->tileRank = i; cs[i]->tileWorld = nDevices; cs[i]->bandRows = 8;
            if (i) { cs[i]->leader = cs[0]; cs[0]->followers.push_back(cs[i]); }
        }
        cudaSetDevice(cs[0]->device);
    }
    *out = cs[0];
    return RT_OK;
}

int rtGetDevicePointer(RtContext* c, const char* name, void** devPtr, size_t* bytes)
{
    if (!c || !name || !devPtr || !bytes) return fail(c, RT_E_INVALID, "rtGetDevicePointer: bad argument");
    CK(cudaSetDevice(c->device));
    if (const NamedImage* img = findImage(name))
    {
        int rc = imageReady(c, *img, "rtGetDevicePointer"); if (rc != RT_OK) return rc;
        *devPtr = img->buf.p(c); *bytes = img->buf.count(c) * img->buf.element;
        return RT_OK;
    }
    // the tile staging buffers follow the tile pattern (rtSetTile), not the image alone
    const std::string n(name);
    if (n != "TileSend" && n != "TileRecv") return fail(c, RT_E_UNKNOWN_NAME, std::string("rtGetDevicePointer: unknown object ") + name);
    int rc = ensureTileBuffers(c); if (rc != RT_OK) return rc;
    const DevBuf<float4>& b = n == "TileSend" ? c->tileSend : c->tileRecv;
    *devPtr = b.p; *bytes = b.count * 16;
    return RT_OK;
}

// One exported image: the IPC handle of the allocation that contains it + its byte offset inside that allocation
// (cudaMalloc may sub-allocate small buffers from a larger block; the handle always names the whole block).
struct RtIpcImage { cudaIpcMemHandle_t handle; unsigned long long offset; };
static_assert(sizeof(RtIpcImage) == 72, "IPC blob layout");

static cudaError_t allocationBase(const void* p, unsigned long long* offset)
{
    typedef int (*GetRangeFn)(unsigned long long*, size_t*, unsigned long long);
    static GetRangeFn fn = nullptr;
    if (!fn)
    {
        void* sym = nullptr; cudaDriverEntryPointQueryResult qr;
        cudaError_t e = cudaGetDriverEntryPoint("cuMemGetAddressRange", &sym, cudaEnableDefault, &qr);
        if (e != cudaSuccess) return e;
        if (!sym) return cudaErrorNotSupported;
        fn = (GetRangeFn)sym;
    }
    unsigned long long base = 0; size_t size = 0;
    if (fn(&base, &size, (unsigned long long)(uintptr_t)p) != 0) return cudaErrorInvalidValue;
    *offset = (unsigned long long)(uintptr_t)p - base;
    return cudaSuccess;
}

int rtGetIpcHandles(RtContext* c, void* handles, size_t bytes)
{
    if (!c || !handles || bytes != 2 * sizeof(RtIpcImage)) return fail(c, RT_E_INVALID, "rtGetIpcHandles: handles must hold 2 x 72 bytes");
    if (!c->frame.p || !c->accum.p) return fail(c, RT_E_STATE, "rtGetIpcHandles: rtResize has not been called");
    CK(cudaSetDevice(c->device));
    RtIpcImage h[2];
    memset(h, 0, sizeof(h));
    CK(cudaIpcGetMemHandle(&h[0].handle, c->frame.p));
    CK(allocationBase(c->frame.p, &h[0].offset));
    CK(cudaIpcGetMemHandle(&h[1].handle, c->accum.p));
    CK(allocationBase(c->accum.p, &h[1].offset));
    memcpy(handles, h, sizeof(h));
    return RT_OK;
}

int rtSetPeers(RtContext* c, int nPeers, const void* handles, size_t bytes)
{
    if (!c || nPeers < 0 || nPeers > RT_MAX_PEERS) return fail(c, RT_E_INVALID, "rtSetPeers: at most 7 peers");
    if (nPeers > 0 && (!handles || bytes != (size_t)nPeers * 2 * sizeof(RtIpcImage))) return fail(c, RT_E_INVALID, "rtSetPeers: handles must hold nPeers x 2 x 72 bytes");
    CK(cudaSetDevice(c->device));
    CK(cudaStreamSynchronize(c->stream));
    closePeers(c);
    const RtIpcImage* h = (const RtIpcImage*)handles;
    for (int k = 0; k < nPeers; k++)
    {
        void* base[2] = {nullptr, nullptr};
        for (int j = 0; j < 2; j++)
        {
            // both images of a peer may live in the same allocation: open every distinct handle once
            if (j == 1 && memcmp(&h[2 * k].handle, &h[2 * k + 1].handle, sizeof(cudaIpcMemHandle_t)) == 0) { base[1] = base[0]; continue; }
            CK(cudaIpcOpenMemHandle(&base[j], h[2 * k + j].handle, cudaIpcMemLazyEnablePeerAccess));
            c->peerBase.push_back(base[j]);
        }
        c->peerFrame[k] = (float4*)((char*)base[0] + h[2 * k].offset);
        c->peerAccum[k] = (float4*)((char*)base[1] + h[2 * k + 1].offset);
    }
    c->nPeers = nPeers;
    return RT_OK;
}

// Host <-> device copies of large caller-owned (pageable) arrays through two pinned chunks: the CPU copies chunk k + 1 into / out of
// pinned memory while the DMA engine moves chunk k, instead of the driver's own slower staging of pageable memory.
// memcpy of one staging chunk on a few host threads: one core moves 5-10 GB/s (less into pages that are touched for the first time),
// the DMA engine 25-50 GB/s
static void hostCopy(void* dst, const void* src, size_t n)
{
#ifndef RT_SIMT_EMU
    const unsigned hw = std::thread::hardware_concurrency();
    const int parts = n < (1u << 20) || hw < 4 ? 1 : 4;
    if (parts > 1)
    {
        std::thread th[3];
        const size_t each = ((n / parts) + 4095) & ~(size_t)4095;
        for (int k = 1; k < parts; k++)
        {
            const size_t off = each * k, len = off >= n ? 0 : (k == parts - 1 ? n - off : (each < n - off ? each : n - off));
            th[k - 1] = std::thread([=]() { if (len) memcpy((unsigned char*)dst + off, (const unsigned char*)src + off, len); });
        }
        memcpy(dst, src, each < n ? each : n);
        for (int k = 1; k < parts; k++) th[k - 1].join();
        return;
    }
#endif
    memcpy(dst, src, n);
}

static int stagingReady(RtContext* c)
{
    for (int k = 0; k < 2; k++)
    {
        if (!c->stageBuf[k]) CK(cudaMallocHost((void**)&c->stageBuf[k], RtContext::STAGE_BYTES));
        if (!c->stageEv[k]) CK(cudaEventCreateWithFlags(&c->stageEv[k], cudaEventDisableTiming));
    }
    return RT_OK;
}
static int stagedH2D(RtContext* c, void* dst, const void* src, size_t bytes)
{
    int rc = stagingReady(c); if (rc != RT_OK) return rc;
    size_t off = 0; int k = 0;
    while (off < bytes)
    {
        const size_t n = bytes - off < RtContext::STAGE_BYTES ? bytes - off : RtContext::STAGE_BYTES;
        CK(cudaEventSynchronize(c->stageEv[k]));                                   // the copy that last used this chunk has read it
        hostCopy(c->stageBuf[k], (const unsigned char*)src + off, n);
        CK(cudaMemcpyAsync((unsigned char*)dst + off, c->stageBuf[k], n, cudaMemcpyHostToDevice, c->stream));
        CK(cudaEventRecord(c->stageEv[k], c->stream));
        off += n; k ^= 1;
    }
    return RT_OK;
}
static int stagedD2H(RtContext* c, void* dst, const void* src, size_t bytes)
{
    int rc = stagingReady(c); if (rc != RT_OK) return rc;
    CK(cudaEventSynchronize(c->stageEv[0])); CK(cudaEventSynchronize(c->stageEv[1]));
    size_t off = 0, prevOff = 0, prevN = 0; int k = 0;
    while (off < bytes || prevN)
    {
        size_t n = 0;
        if (off < bytes)
        {
            n = bytes - off < RtContext::STAGE_BYTES ? bytes - off : RtContext::STAGE_BYTES;
            CK(cudaMemcpyAsync(c->stageBuf[k], (const unsigned char*)src + off, n, cudaMemcpyDeviceToHost, c->stream));
            CK(cudaEventRecord(c->stageEv[k], c->stream));
        }
        if (prevN)                                                                  // while chunk k travels, hand chunk k ^ 1 to the caller
        {
            CK(cudaEventSynchronize(c->stageEv[k ^ 1]));
            hostCopy((unsigned char*)dst + prevOff, c->stageBuf[k ^ 1], prevN);
        }
        prevOff = off; prevN = n; off += n; k ^= 1;
    }
    return RT_OK;
}

// BVH(verts, indices, normals, quality) of the reference (BVH.cs:26, called per mesh from RayComputeManager.cs:209-232), built on the GPU:
// the same Nodes / Triangles the host builder returns (rt_bvh_build.cuh).  Host arrays in, host arrays out.
int rtBuildBVH(RtContext* c, const float* verts, int vertCount, const int* indices, int indexCount, const float* normals, int quality,
               RtTriangle* outTris, RtNode* outNodes, int nodeCapacity, int* outNodeCount)
{
    if (!c || !verts || !indices || !normals || !outTris || !outNodes || !outNodeCount) return fail(c, RT_E_INVALID, "rtBuildBVH: bad argument");
    if (quality < 0 || quality > 2) return fail(c, RT_E_INVALID, "rtBuildBVH: quality must be 0 (Low), 1 (High) or 2 (Disabled)");
    if (indexCount <= 0 || indexCount % 3 != 0) return fail(c, RT_E_INVALID, "rtBuildBVH: index count must be a positive multiple of 3");
    if (vertCount <= 0) return fail(c, RT_E_INVALID, "rtBuildBVH: no vertices");
    for (int i = 0; i < indexCount; i++)
        if (indices[i] < 0 || indices[i] >= vertCount) return fail(c, RT_E_INVALID, "rtBuildBVH: vertex index out of range");
    const int triCount = indexCount / 3;
    if (nodeCapacity < 2 * triCount + 1) return fail(c, RT_E_INVALID, "rtBuildBVH: outNodes must hold 2 * triangles + 1 entries");
    CK(cudaSetDevice(c->device));
    // ONE device allocation for inputs, outputs and the build's temporaries, kept by the context between builds (grow-only;
    // RayComputeManager builds every mesh of a scene in turn), and two pinned staging chunks for the host <-> device copies.
    const bool timing = getenv("RT_B200_BVH_TIMING") != nullptr;
    const auto t0 = std::chrono::steady_clock::now();
    auto ms = [&](std::chrono::steady_clock::time_point a) { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - a).count(); };
    const size_t bV = BvhScratch::align((size_t)vertCount * 12), bI = BvhScratch::align((size_t)indexCount * 4),
                 bNodes = BvhScratch::align(((size_t)2 * triCount + 1) * sizeof(RtNode)), bTris = BvhScratch::align((size_t)triCount * sizeof(RtTriangle));
    const size_t need = 2 * bV + bI + bNodes + bTris + BvhScratch::bytesFor(triCount);
    if (need > c->buildArena.count) { CK(cudaStreamSynchronize(c->stream)); CK(c->buildArena.ensure(need)); }
    unsigned char* base = c->buildArena.p;
    float* dV = reinterpret_cast<float*>(base); float* dN = reinterpret_cast<float*>(base + bV); int* dI = reinterpret_cast<int*>(base + 2 * bV);
    RtNode* dNodes = reinterpret_cast<RtNode*>(base + 2 * bV + bI); RtTriangle* dTris = reinterpret_cast<RtTriangle*>(base + 2 * bV + bI + bNodes);
    BvhScratch scratch; scratch.base = base + 2 * bV + bI + bNodes + bTris; scratch.cap = c->buildArena.count - (2 * bV + bI + bNodes + bTris);
    const double tAlloc = ms(t0);
    const auto t1 = std::chrono::steady_clock::now();
    int rc;
    if ((rc = stagedH2D(c, dV, verts, (size_t)vertCount * 12)) != RT_OK || (rc = stagedH2D(c, dN, normals, (size_t)vertCount * 12)) != RT_OK ||
        (rc = stagedH2D(c, dI, indices, (size_t)indexCount * 4)) != RT_OK) return rc;
    const double tUp = ms(t1);
    const auto t2 = std::chrono::steady_clock::now();
    BvhBuildResult res; std::string msg;
    cudaError_t e = bvh_build_device(dV, dN, dI, triCount, quality, dNodes, dTris, c->stream, res, msg, scratch);
    if (e != cudaSuccess) return msg.empty() ? failCuda(c, e, "rtBuildBVH") : fail(c, RT_E_STATE, "rtBuildBVH: " + msg);
    const double tBuild = ms(t2);
    const auto t3 = std::chrono::steady_clock::now();
    if ((rc = stagedD2H(c, outNodes, dNodes, (size_t)res.nodeCount * sizeof(RtNode))) != RT_OK || (rc = stagedD2H(c, outTris, dTris, (size_t)triCount * sizeof(RtTriangle))) != RT_OK) return rc;
    if (timing) fprintf(stderr, "[rtBuildBVH] %d triangles, %d nodes, %d levels: arena %.2f ms, upload %.2f ms (%.1f MB), build %.2f ms, download %.2f ms (%.1f MB), total %.2f ms\n",
                        triCount, res.nodeCount, res.levels, tAlloc, tUp, ((size_t)vertCount * 24 + (size_t)indexCount * 4) / 1e6, tBuild, ms(t3),
                        ((size_t)res.nodeCount * sizeof(RtNode) + (size_t)triCount * sizeof(RtTriangle)) / 1e6, ms(t0));
    *outNodeCount = res.nodeCount;
    return RT_OK;
}

/* Device-free test hook (not part of include/rt_b200.h): the breadth-first pair layout the upload would build.
 * pairsOut: capacity pairCap records of 64 bytes; rootsOut: 2 ints (start, count) per model.  Returns the number of pair
 * records, or a negative RT_E_* code with the reason in msg. */
int rtxPlanPairsOrdered(const RtNode* nodes, int nodeCount, const RtModel* models, int modelCount, int triCount, int smemBudget, int treeletDepth,
                        void* pairsOut, int pairCap, int* smemPairsOut, int* rootsOut, char* msg, int msgCap);
int rtxPlanPairs(const RtNode* nodes, int nodeCount, const RtModel* models, int modelCount, int triCount, int smemBudget,
                 void* pairsOut, int pairCap, int* smemPairsOut, int* rootsOut, char* msg, int msgCap)
{
    return rtxPlanPairsOrdered(nodes, nodeCount, models, modelCount, triCount, smemBudget, 0, pairsOut, pairCap, smemPairsOut, rootsOut, msg, msgCap);
}
int rtxPlanPairsOrdered(const RtNode* nodes, int nodeCount, const RtModel* models, int modelCount, int triCount, int smemBudget, int treeletDepth,
                        void* pairsOut, int pairCap, int* smemPairsOut, int* rootsOut, char* msg, int msgCap)
{
    if (!nodes || !models || nodeCount <= 0 || modelCount < 0 || !pairsOut || !rootsOut) return RT_E_INVALID;
    std::vector<RtNode> n(nodes, nodes + nodeCount);
    std::vector<RtModel> m(models, models + modelCount);
    for (int i = 0; i < modelCount; i++)
        if (m[i].nodeOffset < 0 || m[i].nodeOffset >= nodeCount) { if (msg && msgCap > 0) snprintf(msg, msgCap, "model nodeOffset out of range"); return RT_E_STATE; }
    RepackState st;
    std::vector<NodePair> out; std::string why;
    st.planScene(n, m, modelCount, (size_t)triCount, smemBudget, out, why, treeletDepth);
    if (!why.empty()) { if (msg && msgCap > 0) snprintf(msg, msgCap, "%s", why.c_str()); return RT_E_STATE; }
    if ((int)out.size() > pairCap) return RT_E_INVALID;
    if (!out.empty()) memcpy(pairsOut, out.data(), out.size() * sizeof(NodePair));
    if (smemPairsOut) *smemPairsOut = st.smemPairs;
    for (int i = 0; i < modelCount; i++)
    {
        const MeshRoot& r = st.roots[std::make_pair(m[i].nodeOffset, m[i].triOffset)];
        rootsOut[2 * i] = r.rootStart; rootsOut[2 * i + 1] = r.rootCount;
    }
    return (int)out.size();
}

#ifdef RT_POOL_CLOCKS
/* Cycle account of the pooled kernel (RT_POOL_CLOCKS variant builds only, not part of include/rt_b200.h): copies the 3 x CK_KINDS
 * counters ([cycles, steps, lanes] per step kind, rt_kernel_pool.cuh) of the current device into out (n >= 3 * CK_KINDS), then zeroes
 * them if reset != 0.  Returns the number of counters or a negative RT_E_* code. */
int rtxPoolClocks(unsigned long long* out, int n, int reset)
{
    if (!out || n < 3 * CK_KINDS) return RT_E_INVALID;
    if (cudaDeviceSynchronize() != cudaSuccess) return RT_E_CUDA;
    if (cudaMemcpyFromSymbol(out, g_poolClocks, sizeof(g_poolClocks)) != cudaSuccess) return RT_E_CUDA;
    if (reset)
    {
        static const unsigned long long zero[3 * CK_KINDS] = {};
        if (cudaMemcpyToSymbol(g_poolClocks, zero, sizeof(zero)) != cudaSuccess) return RT_E_CUDA;
    }
    return 3 * CK_KINDS;
}
#endif

/* Device-free test hook (not part of include/rt_b200.h): the TLAS the upload would build over `modelCount` world boxes
 * (6 floats each: min xyz, max xyz).  pairsOut: capacity pairCap records of 64 bytes; leavesOut: modelCount model indices in leaf
 * order; rootOut: 2 ints (start, count).  Returns the number of pair records or a negative RT_E_* code. */
int rtxPlanTlas(const float* boxes, int modelCount, void* pairsOut, int pairCap, int* leavesOut, int* rootOut)
{
    if (!boxes || modelCount < 1 || modelCount > RT_TLAS_MAX_MODELS || !pairsOut || !leavesOut || !rootOut) return RT_E_INVALID;
    std::vector<DevModel> dm(modelCount);
    for (int i = 0; i < modelCount; i++)
    {
        memset(&dm[i], 0, sizeof(DevModel));
        dm[i].wmin[0] = boxes[6 * i]; dm[i].wmin[1] = boxes[6 * i + 1]; dm[i].wmin[2] = boxes[6 * i + 2];
        dm[i].wmaxx = boxes[6 * i + 3]; dm[i].wmaxy = boxes[6 * i + 4]; dm[i].wmaxz = boxes[6 * i + 5];
    }
    std::vector<NodePair> out; std::vector<int> order;
    RepackState::planTlas(dm, modelCount, out, order, rootOut[0], rootOut[1]);
    if ((int)out.size() > pairCap) return RT_E_INVALID;
    if (!out.empty()) memcpy(pairsOut, out.data(), out.size() * sizeof(NodePair));
    memcpy(leavesOut, order.data(), order.size() * sizeof(int));
    return (int)out.size();
}

/* Device-free test hook: the sphere accelerator's tree the upload would build over n spheres (4 floats each: centre xyz, radius) for
 * ray origins in originBox (min xyz, max xyz).  Outputs as rtxPlanTlas; leavesOut holds n sphere indices. */
int rtxPlanSpheres(const float* spheres, int n, const float* originBox, void* pairsOut, int pairCap, int* leavesOut, int* rootOut)
{
    if (!spheres || n < 1 || !originBox || !pairsOut || !leavesOut || !rootOut) return RT_E_INVALID;
    std::vector<RtSphere> sp(n);
    for (int i = 0; i < n; i++)
    {
        memset(&sp[i], 0, sizeof(RtSphere));
        for (int a = 0; a < 3; a++) sp[i].centre[a] = spheres[4 * i + a];
        sp[i].radius = spheres[4 * i + 3];
    }
    std::vector<NodePair> out; std::vector<int> order;
    RepackState::planSpheres(sp.data(), (size_t)n, originBox, originBox + 3, order, out, rootOut[0], rootOut[1]);
    if ((int)out.size() > pairCap) return RT_E_INVALID;
    if (!out.empty()) memcpy(pairsOut, out.data(), out.size() * sizeof(NodePair));
    memcpy(leavesOut, order.data(), order.size() * sizeof(int));
    return (int)out.size();
}

/* Device-free test hook: for a tree over n items (which = 0: the sphere accelerator, 1: the TLAS), the surface-area levels the host
 * builds, the most stack entries a walk of that tree can need (SplitTreeStackBound) and the entries the device walk keeps. */
int rtxTreeStackLimits(int which, long long n, int* sahDepthOut, int* boundOut, int* stackOut)
{
    if (n < 1 || !sahDepthOut || !boundOut || !stackOut) return RT_E_INVALID;
    if (which == 0) { *sahDepthOut = RepackState::sphereSahDepth(n); *stackOut = RT_SPHERE_STACK; }
    else if (which == 1 && n <= RT_TLAS_MAX_MODELS) { *sahDepthOut = RT_TLAS_SAH_DEPTH; *stackOut = RT_TLAS_STACK; }
    else return RT_E_INVALID;
    *boundOut = SplitTreeStackBound(n, *sahDepthOut);
    return RT_OK;
}

static int one_rtGetStats(RtContext* c, RtStats* out);
int rtGetStats(RtContext* c, RtStats* out)
{
    // a group reports the work of all its GPUs: counters summed, times = the slowest GPU's (they run side by side)
    int rc = one_rtGetStats(c, out);
    if (rc != RT_OK || !c) return rc;
    for (RtContext* m : c->followers)
    {
        RtStats s;
        if ((rc = one_rtGetStats(m, &s)) != RT_OK) return fail(c, rc, "GPU " + std::to_string(m->device) + ": " + m->err);
        out->rays += s.rays; out->boxTests += s.boxTests; out->triTests += s.triTests; out->sphereTests += s.sphereTests; out->sphereBoxTests += s.sphereBoxTests;
        if (s.kernelMs > out->kernelMs) out->kernelMs = s.kernelMs;
        if (s.exchangeMs > out->exchangeMs) out->exchangeMs = s.exchangeMs;
    }
    if (!c->followers.empty()) CK(cudaSetDevice(c->device));
    return RT_OK;
}
static int one_rtGetStats(RtContext* c, RtStats* out)
{
    if (!c || !out) return fail(c, RT_E_INVALID, "rtGetStats: bad argument");
    CK(cudaSetDevice(c->device));
    CK(cudaStreamSynchronize(c->stream));
    int rc = drainEvents(c); if (rc != RT_OK) return rc;
    unsigned long long h[5];
    CK(cudaMemcpy(h, c->dCounters, sizeof(h), cudaMemcpyDeviceToHost));
    c->stats.rays = h[0]; c->stats.boxTests = h[1]; c->stats.triTests = h[2]; c->stats.sphereTests = h[3]; c->stats.sphereBoxTests = h[4];
    *out = c->stats;
    return RT_OK;
}

static int one_rtResetStats(RtContext* c);
int rtResetStats(RtContext* c)
{
    int rc = forGroup(c, one_rtResetStats);
    if (rc != RT_OK || !c) return rc;
    if (!c->followers.empty()) CK(cudaSetDevice(c->device));
    return RT_OK;
}
static int one_rtResetStats(RtContext* c)
{
    if (!c) return RT_E_INVALID;
    CK(cudaSetDevice(c->device));
    CK(cudaStreamSynchronize(c->stream));
    int rc = drainEvents(c); if (rc != RT_OK) return rc;
    CK(cudaMemset(c->dCounters, 0, 8 * sizeof(unsigned long long)));
    if (c->pixelStats.p) CK(cudaMemset(c->pixelStats.p, 0, c->pixelStats.count * sizeof(RtPixelStats)));
    memset(&c->stats, 0, sizeof(c->stats));
    return RT_OK;
}

// ---- per-pixel counters ("PixelStats") ----------------------------------------------------------------------------------------
static int pixelStatsReady(RtContext* c, const char* what)
{
    int rc = refuseGroup(c, what); if (rc != RT_OK) return rc;
    if (!c->pixelStats.p) return fail(c, RT_E_STATE, std::string(what) + ": no counting dispatch yet (rtSetOption(\"countStats\", 1))");
    return RT_OK;
}

int rtReadbackPixelStats(RtContext* c, RtPixelStats* dst, size_t bytes)
{
    if (!c || !dst) return fail(c, RT_E_INVALID, "rtReadbackPixelStats: bad argument");
    int rc = pixelStatsReady(c, "rtReadbackPixelStats"); if (rc != RT_OK) return rc;
    if (bytes != c->pixelStats.count * sizeof(RtPixelStats)) return fail(c, RT_E_INVALID, "rtReadbackPixelStats: bytes must equal W*H*20");
    CK(cudaSetDevice(c->device));
    CK(cudaMemcpyAsync(dst, c->pixelStats.p, bytes, cudaMemcpyDeviceToHost, c->stream));
    CK(cudaStreamSynchronize(c->stream));
    return RT_OK;
}

int rtDisplayPixelStats(RtContext* c, int visMode, float debugVisScale, uint8_t* dst, size_t bytes)
{
    if (!c || !dst) return fail(c, RT_E_INVALID, "rtDisplayPixelStats: bad argument");
    if (visMode < 1 || visMode > 4) return fail(c, RT_E_INVALID, "rtDisplayPixelStats: visMode must be 1 (box tests), 2 (triangle tests), 3 (sphere tests) or 4 (rays)");
    if (!std::isfinite(debugVisScale) || !(debugVisScale > 0.0f)) return fail(c, RT_E_INVALID, "rtDisplayPixelStats: debugVisScale must be finite and > 0");
    int rc = pixelStatsReady(c, "rtDisplayPixelStats"); if (rc != RT_OK) return rc;
    if (bytes != c->pixelStats.count * 4) return fail(c, RT_E_INVALID, "rtDisplayPixelStats: bytes must equal W*H*4");
    return displayTo(c, [&](size_t n)
    {
        RT_LAUNCH((unsigned)((n + 255) / 256), 256, 0, c->stream, k_pixel_stats_display, c->pixelStats.p, c->display.p, n, visMode, debugVisScale);
        return RT_OK;
    }, dst, bytes);
}

} // extern "C"
