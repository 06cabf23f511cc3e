// rt_kernel_query.cuh — rtTraceRays: the closest hit of caller-supplied rays (picking, autofocus, line of sight, visibility baking);
// rtTraceOcclusion: whether anything lies on caller-supplied segments (shadow and ambient-occlusion rays, line of sight);
// rtTracePaths: the path tracer's radiance along caller-supplied rays (custom cameras, probe baking; k_trace_paths at the end).
//
// Each lane traces one ray through the camera kernels' own Intersect (rt_kernel_wave.cuh), so a query returns the bits the path tracer
// computes for the same ray.  Shape: a persistent grid (a multiple of the SM count); every warp reserves 32 consecutive rays with one
// atomicAdd, each lane traces one of them and writes its 48-byte RtRayHit as three 16-byte stores.  Spheres are staged in shared
// memory as in wave_body; tree tops are not (smemPairs = 0).  k_trace_occlusion has the same shape: each lane walks its segment through
// Intersect<..., ANY = true> (from tMax, ended by the first hit) and stores one byte.
//
// Model skipping, the TLAS and the sphere accelerator are exact only for origins inside the box their records were padded for (the
// camera with its defocus disc and all geometry, RepackState::buildModels / buildSpheres).  Camera rays are inside by construction;
// a query ray is tested per lane: componentwise lo <= o <= hi (a NaN fails), and a ray outside walks every model and tests every
// sphere in buffer order — the reference's own loop.
//
// The padding is also sized for the reference's rounding error with every intermediate of RaySphere / the world -> local transform / the
// slab test a normal float, as it is for unit-length camera rays.  That argument is scale-invariant in the direction's length only while
// dot(dir, dir), b * b, 4ac and the transformed directions stay normal and finite: for |dir| near 1e-21 the discriminant of the
// reference is mostly rounding and it reports hits (at dst ~ 1e22) that the padded boxes prune.  So the skips are also restricted to
// directions with QUERY_DIR2_MIN <= dot(dir, dir) <= QUERY_DIR2_MAX (NaN fails): |dir| within a factor 2^10 of a camera ray's, which
// keeps every squared term within 2^+-20 of what unit-length rays produce.  Any other direction takes the linear loop as well.
#pragma once
#include "rt_kernel_wave.cuh"

namespace rtd {

struct QueryParams
{
    const RtRay* rays;
    RtRayHit* hits;
    unsigned int n;
    int noCull;                                  // RT_TRACE_NO_CULL: forceDontCullBack (HL:356)
    float modelLo[3], modelHi[3];                // origins the model records (world boxes, TLAS) were padded for
    float sphLo[3], sphHi[3];                    // origins the sphere accelerator was padded for
    const RtRaySegment* segs;                    // rtTraceOcclusion: the segments and their answers (rays / hits unused)
    unsigned char* occluded;
};

constexpr float QUERY_DIR2_MIN = 9.5367431640625e-07f;      // 2^-20: |dir| >= 2^-10
constexpr float QUERY_DIR2_MAX = 1048576.0f;                 // 2^20:  |dir| <= 2^10

RT_DI bool OriginInside(f3 o, const float lo[3], const float hi[3])
{
    return lo[0] <= o.x && o.x <= hi[0] && lo[1] <= o.y && o.y <= hi[1] && lo[2] <= o.z && o.z <= hi[2];
}

RT_DI bool DirectionInRange(f3 d)
{
    const float dd = dot3(d, d);
    return dd >= QUERY_DIR2_MIN && dd <= QUERY_DIR2_MAX;
}

// One persistent grid over Q.n rays (ANY = false: RtRay -> RtRayHit) or segments (ANY = true: RtRaySegment -> one byte, 1 = occluded)
template <bool STATS, bool EXT, bool TLAS, bool ANY>
RT_DI void query_body(const DevParams& P, const QueryParams& Q)
{
    RT_DYNAMIC_SMEM(smemRaw);
    DevSphere* smemSpheres = reinterpret_cast<DevSphere*>(smemRaw);
    {
        const int nS = P.sphereCount < WAVE_MAX_SMEM_SPHERES ? P.sphereCount : WAVE_MAX_SMEM_SPHERES;
        for (int i = threadIdx.x; i < nS; i += WAVE_THREADS) smemSpheres[i] = P.spheres[i];
    }
    __syncthreads();

    const unsigned int lane = threadIdx.x & 31u;
    Counters cnt; cnt.rays = cnt.box = cnt.tri = cnt.sph = cnt.sbox = 0;
    for (;;)
    {
        unsigned int base = 0;
        if (lane == 0) base = atomicAdd(P.workCounter, 32u);
        base = __shfl_sync(0xffffffffu, base, 0);
        if (base >= Q.n) break;
        const unsigned int i = base + lane;
        if (i < Q.n)
        {
            const float* r = ANY ? reinterpret_cast<const float*>(Q.segs + i) : reinterpret_cast<const float*>(Q.rays + i);
            const f3 o = make_f3(__ldg(r), __ldg(r + 1), __ldg(r + 2));
            const f3 d = make_f3(__ldg(r + 3), __ldg(r + 4), __ldg(r + 5));
            QueryRay q;
            const bool dirOk = DirectionInRange(d);
            q.modelsExact = dirOk && OriginInside(o, Q.modelLo, Q.modelHi);
            q.spheresExact = dirOk && OriginInside(o, Q.sphLo, Q.sphHi);
            q.noCull = Q.noCull != 0;
            if constexpr (ANY)
            {
                q.tMax = __ldg(r + 6);
                Intersect<STATS, EXT, TLAS, true, true>(P, nullptr, smemSpheres, o, d, cnt, &q);
                Q.occluded[i] = q.kind != RT_HIT_NONE ? 1 : 0;
            }
            else
            {
                const Hit h = Intersect<STATS, EXT, TLAS, true>(P, nullptr, smemSpheres, o, d, cnt, &q);
                float4* out = reinterpret_cast<float4*>(Q.hits + i);
                out[0] = make_float4(h.dst, h.pos.x, h.pos.y, h.pos.z);
                out[1] = make_float4(h.normal.x, h.normal.y, h.normal.z, __int_as_float(h.isBackface ? 1 : 0));
                out[2] = make_float4(__int_as_float(q.kind), __int_as_float(q.index), 0.0f, 0.0f);
            }
        }
    }

    unsigned int r = __reduce_add_sync(0xffffffffu, cnt.rays);
    if (lane == 0) atomicAdd(P.counters + 0, (unsigned long long)r);
    if (STATS)
    {
        const unsigned int b = __reduce_add_sync(0xffffffffu, cnt.box), t = __reduce_add_sync(0xffffffffu, cnt.tri), s = __reduce_add_sync(0xffffffffu, cnt.sph), sb = __reduce_add_sync(0xffffffffu, cnt.sbox);
        if (lane == 0) { atomicAdd(P.counters + 1, (unsigned long long)b); atomicAdd(P.counters + 2, (unsigned long long)t); atomicAdd(P.counters + 3, (unsigned long long)s); atomicAdd(P.counters + 4, (unsigned long long)sb); }
    }
}

template <bool STATS, bool EXT, bool TLAS>
__global__ void __launch_bounds__(WAVE_THREADS, RT_WAVE_MINBLOCKS) k_trace_rays(const __grid_constant__ DevParams P, const __grid_constant__ QueryParams Q)
{
    query_body<STATS, EXT, TLAS, false>(P, Q);
}

template <bool STATS, bool EXT, bool TLAS>
__global__ void __launch_bounds__(WAVE_THREADS, RT_WAVE_MINBLOCKS) k_trace_occlusion(const __grid_constant__ DevParams P, const __grid_constant__ QueryParams Q)
{
    query_body<STATS, EXT, TLAS, true>(P, Q);
}

template <bool S, bool X, bool T, bool ANY> inline cudaError_t query_launch_one(const DevParams& P, const QueryParams& Q, int numSMs, cudaStream_t stream)
{
    auto kernel = ANY ? k_trace_occlusion<S, X, T> : k_trace_rays<S, X, T>;
    const size_t smemBytes = (size_t)WAVE_MAX_SMEM_SPHERES * sizeof(DevSphere);
    int ctasPerSM = 0;
    cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctasPerSM, kernel, WAVE_THREADS, smemBytes);
    if (e != cudaSuccess) return e;
    if (ctasPerSM < 1) return cudaErrorInvalidConfiguration;
    unsigned int grid = (unsigned int)(numSMs * ctasPerSM);                  // persistent: a multiple of the SM count
    const unsigned int warpsNeeded = (Q.n + 31u) / 32u;
    const unsigned int ctasNeeded = (warpsNeeded + (WAVE_THREADS / 32) - 1) / (WAVE_THREADS / 32);
    if (grid > ctasNeeded) grid = ctasNeeded ? ctasNeeded : 1;
    if ((e = cudaMemsetAsync(P.workCounter, 0, sizeof(unsigned int), stream)) != cudaSuccess) return e;
    RT_LAUNCH(grid, WAVE_THREADS, smemBytes, stream, kernel, P, Q);
    return cudaGetLastError();
}

// The instantiation follows the scene the way wave_launch chooses a camera kernel: the counting build walks every model; the TLAS
// kernel when the scene has a TLAS and skipping is on; the extension family with the sphere accelerator (or "extInstantiation").
// ANY: the occlusion kernels, chosen by the same rules.
template <bool ANY = false>
inline cudaError_t query_launch(const DevParams& P, const QueryParams& Q, int numSMs, cudaStream_t stream)
{
    const bool ext = P.sphBvh != 0 || P.forceExt != 0;
    if (P.countStats) return ext ? query_launch_one<true, true, false, ANY>(P, Q, numSMs, stream) : query_launch_one<true, false, false, ANY>(P, Q, numSMs, stream);
    if (P.tlas && P.modelSkip) return query_launch_one<false, true, true, ANY>(P, Q, numSMs, stream);
    return ext ? query_launch_one<false, true, false, ANY>(P, Q, numSMs, stream) : query_launch_one<false, false, false, ANY>(P, Q, numSMs, stream);
}

// ---- rtTracePaths: the radiance along caller-supplied rays ------------------------------------------------------------------------
// A lane keeps its ray for all Q.samples paths (one RNG chain) and runs them segment by segment: Intersect<..., QUERY = true> with the
// per-segment gate, then ShadeSegment — HL:479-542 as the camera kernels run it.  Paths of a ray take 1 .. MaxBounceCount + 1 segments
// each, so a warp that took 32 rays at once would wait for its longest chain; instead, as in kernel 1 (wave_body), every iteration
// first refills the lanes whose ray has ended (ballot, one atomicAdd per warp, rays handed out by popcount rank), then traces one
// segment on every lane that has a ray.
struct PathParams
{
    const RtPathRay* rays;
    RtPathRadiance* out;
    unsigned int n;
    int samples;                                 // 1 .. RT_MAX_BATCH_SAMPLES
    float modelLo[3], modelHi[3];                // as QueryParams
    float sphLo[3], sphHi[3];
};

template <bool STATS, bool EXT, bool TLAS>
RT_DI void paths_body(const DevParams& P, const PathParams& Q)
{
    RT_DYNAMIC_SMEM(smemRaw);
    DevSphere* smemSpheres = reinterpret_cast<DevSphere*>(smemRaw);
    {
        const int nS = P.sphereCount < WAVE_MAX_SMEM_SPHERES ? P.sphereCount : WAVE_MAX_SMEM_SPHERES;
        for (int i = threadIdx.x; i < nS; i += WAVE_THREADS) smemSpheres[i] = P.spheres[i];
    }
    __syncthreads();

    const unsigned int lane = threadIdx.x & 31u;
    const unsigned int laneMaskLt = (1u << lane) - 1u;
    Counters cnt; cnt.rays = cnt.box = cnt.tri = cnt.sph = cnt.sbox = 0;
    bool exhausted = false, haveRay = false;
    unsigned int i = 0;                          // the lane's ray
    uint32_t rngState = 0;
    f3 total = splat3(0.0f);
    int sample = 0, bounce = 0;
    PathState ray; ray.pos = ray.dir = ray.transmittance = ray.totalLight = splat3(0.0f);

    for (;;)
    {
        // [refill] lanes without a ray take the next ones (ballot + one atomic per warp)
        const bool need = !haveRay && !exhausted;
        const unsigned int needMask = __ballot_sync(0xffffffffu, need);
        if (needMask)
        {
            unsigned int base = 0;
            const int leader = __ffs(needMask) - 1;
            if ((int)lane == leader) base = atomicAdd(P.workCounter, (unsigned int)__popc(needMask));
            base = __shfl_sync(0xffffffffu, base, leader);
            if (need)
            {
                i = base + (unsigned int)__popc(needMask & laneMaskLt);
                if (i >= Q.n) exhausted = true;
                else
                {
                    rngState = __ldg(&Q.rays[i].rngState);
                    total = splat3(0.0f);
                    sample = 0;
                    bounce = -1;                 // a path starts below
                    haveRay = true;
                }
            }
        }
        // every lane now holds a ray or has run out of them
        if (__ballot_sync(0xffffffffu, haveRay) == 0u) break;

        if (haveRay)
        {
            if (bounce < 0)
            {
                // CreateRay(origin, dir, 1, 0) (HL:439-448), for every sample from the caller's record
                const float* r = reinterpret_cast<const float*>(Q.rays + i);
                ray.pos = make_f3(__ldg(r), __ldg(r + 1), __ldg(r + 2));
                ray.dir = make_f3(__ldg(r + 3), __ldg(r + 4), __ldg(r + 5));
                ray.transmittance = splat3(1.0f);
                ray.totalLight = splat3(0.0f);
                bounce = 0;
            }
            // [intersect] the segment, with rtTraceRays' gate on its own origin and direction
            QueryRay q;
            const bool dirOk = DirectionInRange(ray.dir);
            q.modelsExact = dirOk && OriginInside(ray.pos, Q.modelLo, Q.modelHi);
            q.spheresExact = dirOk && OriginInside(ray.pos, Q.sphLo, Q.sphHi);
            q.noCull = false;                    // HL:487
            const Hit hit = Intersect<STATS, EXT, TLAS, true>(P, nullptr, smemSpheres, ray.pos, ray.dir, cnt, &q);
            // [shade]
            const bool cont = ShadeSegment(P, hit, ray, rngState);
            bounce++;
            if (!cont || bounce > P.MaxBounceCount)
            {
                total = total + ray.totalLight;                      // HL:578
                bounce = -1;
                if (++sample >= Q.samples)
                {
                    const f3 c = total / __int2float_rn(Q.samples);  // HL:581
                    reinterpret_cast<float4*>(Q.out)[i] = make_float4(c.x, c.y, c.z, __uint_as_float(rngState));
                    haveRay = false;
                }
            }
        }
    }

    unsigned int r = __reduce_add_sync(0xffffffffu, cnt.rays);
    if (lane == 0) atomicAdd(P.counters + 0, (unsigned long long)r);
    if (STATS)
    {
        const unsigned int b = __reduce_add_sync(0xffffffffu, cnt.box), t = __reduce_add_sync(0xffffffffu, cnt.tri), s = __reduce_add_sync(0xffffffffu, cnt.sph), sb = __reduce_add_sync(0xffffffffu, cnt.sbox);
        if (lane == 0) { atomicAdd(P.counters + 1, (unsigned long long)b); atomicAdd(P.counters + 2, (unsigned long long)t); atomicAdd(P.counters + 3, (unsigned long long)s); atomicAdd(P.counters + 4, (unsigned long long)sb); }
    }
}

template <bool STATS, bool EXT, bool TLAS>
__global__ void __launch_bounds__(WAVE_THREADS, RT_WAVE_MINBLOCKS) k_trace_paths(const __grid_constant__ DevParams P, const __grid_constant__ PathParams Q)
{
    paths_body<STATS, EXT, TLAS>(P, Q);
}

template <bool S, bool X, bool T> inline cudaError_t paths_launch_one(const DevParams& P, const PathParams& Q, int numSMs, cudaStream_t stream)
{
    auto kernel = k_trace_paths<S, X, T>;
    const size_t smemBytes = (size_t)WAVE_MAX_SMEM_SPHERES * sizeof(DevSphere);
    int ctasPerSM = 0;
    cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctasPerSM, kernel, WAVE_THREADS, smemBytes);
    if (e != cudaSuccess) return e;
    if (ctasPerSM < 1) return cudaErrorInvalidConfiguration;
    unsigned int grid = (unsigned int)(numSMs * ctasPerSM);                  // persistent: a multiple of the SM count
    const unsigned int warpsNeeded = (Q.n + 31u) / 32u;
    const unsigned int ctasNeeded = (warpsNeeded + (WAVE_THREADS / 32) - 1) / (WAVE_THREADS / 32);
    if (grid > ctasNeeded) grid = ctasNeeded ? ctasNeeded : 1;
    if ((e = cudaMemsetAsync(P.workCounter, 0, sizeof(unsigned int), stream)) != cudaSuccess) return e;
    RT_LAUNCH(grid, WAVE_THREADS, smemBytes, stream, kernel, P, Q);
    return cudaGetLastError();
}

// The five instantiations of query_launch, chosen by the same rules
inline cudaError_t paths_launch(const DevParams& P, const PathParams& Q, int numSMs, cudaStream_t stream)
{
    const bool ext = P.sphBvh != 0 || P.forceExt != 0;
    if (P.countStats) return ext ? paths_launch_one<true, true, false>(P, Q, numSMs, stream) : paths_launch_one<true, false, false>(P, Q, numSMs, stream);
    if (P.tlas && P.modelSkip) return paths_launch_one<false, true, true>(P, Q, numSMs, stream);
    return ext ? paths_launch_one<false, true, false>(P, Q, numSMs, stream) : paths_launch_one<false, false, false>(P, Q, numSMs, stream);
}

} // namespace rtd
