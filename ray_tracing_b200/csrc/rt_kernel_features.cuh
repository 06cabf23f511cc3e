// rt_kernel_features.cuh — rtDispatchFeatures: the first-hit feature images a denoiser is guided by (albedo, shading normal, depth,
// object id) for the camera ray every pixel's path of the current Frame starts with; rtCameraRays: those rays themselves.
//
// The feature ray of a pixel is SetupPixel + one GenerateCameraRay (HL:547-576, rt_device.cuh): the pixel's own seed for the current
// Frame and renderSeed, four draws of jitter.  It is the first sample's ray of an rtDispatch of the same frame — with NumRaysPerPixel
// = 1 the only one.  (Later samples of a pixel start from the RNG state the whole path before them left behind, HL:563-579: only the
// render kernels can know them.)
//
// k_camera_features has the shape of the queries (rt_kernel_query.cuh: a persistent grid, spheres staged in shared memory, no tree
// tops) and the work order of wave_body (rt_kernel_wave.cuh): one atomicAdd per warp reserves an 8x4-pixel tile, mapped through this
// context's row bands, so a warp's 32 rays start from neighbouring pixels and walk the same nodes.  Each lane traces its ray through
// the camera kernels' Intersect, evaluates the material and stores a 32-byte RtPixelFeatures as two 16-byte stores; when accumulating
// it adds into two float4 images (one thread owns a pixel: no atomics).  Camera rays start inside the box of origins the model
// records, the TLAS and the sphere accelerator were padded for (fitOriginPadding, rt_api.cu), so the per-ray test of the queries is
// not made; Intersect's QUERY form is used only for what it reports, the winner's kind and index.
#pragma once
#include "rt_kernel_query.cuh"

namespace rtd {

struct FeatureParams
{
    RtPixelFeatures* features;                   // "FeatureFrame": W*H records, [y][x]
    float4* accumAlbedo;                         // "AccumulatedAlbedo" += (albedo, 1) on a hit
    float4* accumNormal;                         // "AccumulatedNormal" += (normal, dst) on a hit
    RtPathRay* rays;                             // k_camera_rays: W*H records, [y][x] (4-byte aligned)
    unsigned int totalJobs, tilesX, ownedRows;   // 32 jobs per 8x4-pixel tile, as camera_jobs counts them
};

// job -> pixel, as wave_body maps it: tile job >> 5, lane job & 31; rows counted through this rank's bands.  false = outside the image
RT_DI bool FeaturePixel(const DevParams& P, const FeatureParams& F, unsigned int job, unsigned int& x, unsigned int& y)
{
    const unsigned int tile = job >> 5, l = job & 31u;
    x = (tile % F.tilesX) * 8u + (l & 7u);
    const unsigned int r = (tile / F.tilesX) * 4u + (l >> 3);
    if (x >= P.limX || r >= F.ownedRows) return false;
    y = ((r / (unsigned int)P.bandRows) * (unsigned int)P.tileWorld + (unsigned int)P.tileRank) * (unsigned int)P.bandRows + (r % (unsigned int)P.bandRows);
    return true;
}

template <bool STATS, bool EXT, bool TLAS>
__global__ void __launch_bounds__(WAVE_THREADS, RT_WAVE_MINBLOCKS) k_camera_features(const __grid_constant__ DevParams P, const __grid_constant__ FeatureParams F)
{
    RT_DYNAMIC_SMEM(smemRaw);
    const DevSphere* smemSpheres = StageSpheres(P, smemRaw);

    const unsigned int lane = threadIdx.x & 31u;
    Counters cnt; cnt.rays = cnt.box = cnt.tri = cnt.sph = cnt.sbox = 0;
    for (;;)
    {
        unsigned int base = 0;
        if (lane == 0) base = atomicAdd(P.workCounter, 32u);
        base = __shfl_sync(0xffffffffu, base, 0);
        if (base >= F.totalJobs) break;
        unsigned int x, y;
        if (!FeaturePixel(P, F, base + lane, x, y)) continue;

        const PixelSetup px = SetupPixel(P, x, y);
        uint32_t rngState = px.rngState;
        PathState ray;
        GenerateCameraRay(P, px, rngState, ray);
        QueryRay q;
        q.modelsExact = q.spheresExact = true; q.noCull = false;         // a camera ray: HL:487
        const Hit h = Intersect<STATS, EXT, TLAS, true>(P, nullptr, smemSpheres, ray.pos, ray.dir, cnt, &q);

        const size_t o = (size_t)y * P.W + x;
        float4* out = reinterpret_cast<float4*>(F.features + o);
        if (q.kind == RT_HIT_NONE)
        {
            out[0] = make_float4(0.0f, 0.0f, 0.0f, h.dst);
            out[1] = make_float4(0.0f, 0.0f, 0.0f, __int_as_float(-1));
            continue;
        }
        // a transmissive surface shows what lies behind it: white, the usual convention; anything else its diffuse colour (HL:450-466)
        const f3 albedo = h.material->flag == RT_MATERIAL_GLASS ? splat3(1.0f) : GetMaterialColour(h.material, h.pos, h.normal, false);
        const int object = q.kind == RT_HIT_SPHERE ? -2 - q.index : q.index;
        out[0] = make_float4(albedo.x, albedo.y, albedo.z, h.dst);
        out[1] = make_float4(h.normal.x, h.normal.y, h.normal.z, __int_as_float(object));
        if (P.accumulate)
        {
            float4 a = F.accumAlbedo[o], n = F.accumNormal[o];
            a.x += albedo.x; a.y += albedo.y; a.z += albedo.z; a.w += 1.0f;
            n.x += h.normal.x; n.y += h.normal.y; n.z += h.normal.z; n.w += h.dst;
            F.accumAlbedo[o] = a; F.accumNormal[o] = n;
        }
    }

    FlushCounters<STATS>(P, cnt);
}

// The feature ray of every pixel of the image and the RNG state after its four draws: what rtTracePaths takes.  One thread per job.
__global__ void __launch_bounds__(WAVE_THREADS) k_camera_rays(const __grid_constant__ DevParams P, const __grid_constant__ FeatureParams F)
{
    const unsigned int job = blockIdx.x * WAVE_THREADS + threadIdx.x;
    unsigned int x, y;
    if (job >= F.totalJobs || !FeaturePixel(P, F, job, x, y)) return;
    const PixelSetup px = SetupPixel(P, x, y);
    uint32_t rngState = px.rngState;
    PathState ray;
    GenerateCameraRay(P, px, rngState, ray);
    float* out = reinterpret_cast<float*>(F.rays + ((size_t)y * P.W + x));
    out[0] = ray.pos.x; out[1] = ray.pos.y; out[2] = ray.pos.z;
    out[3] = ray.dir.x; out[4] = ray.dir.y; out[5] = ray.dir.z;
    out[6] = __uint_as_float(rngState);
}

// this rank's jobs over the dispatched region, counted as the camera kernels count them
inline cudaError_t features_jobs(const DevParams& P, FeatureParams& F)
{
    CameraJobs J;
    if (!camera_jobs(FORM_PLAIN, P, 0u, J)) return cudaErrorInvalidValue;
    F.totalJobs = J.total; F.tilesX = J.tilesX; F.ownedRows = J.ownedRows;
    return cudaSuccess;
}

inline cudaError_t features_launch(const DevParams& P, FeatureParams& F, int numSMs, cudaStream_t stream)
{
    cudaError_t e = features_jobs(P, F);
    if (e != cudaSuccess || F.totalJobs == 0) return e;
    return with_persistent_kernel(P, [&](auto S, auto X, auto T) {
        return persistent_launch(k_camera_features<S, X, T>, QUERY_SMEM_BYTES, F.totalJobs / 32u, P, F, numSMs, stream);
    });
}

inline cudaError_t camera_rays_launch(const DevParams& P, FeatureParams& F, cudaStream_t stream)
{
    cudaError_t e = features_jobs(P, F);
    if (e != cudaSuccess || F.totalJobs == 0) return e;
    RT_LAUNCH((F.totalJobs + WAVE_THREADS - 1) / WAVE_THREADS, WAVE_THREADS, 0, stream, k_camera_rays, P, F);
    return cudaGetLastError();
}

} // namespace rtd
