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

// The boxes of origins the model records (world boxes, TLAS) and the sphere accelerator were padded for
struct OriginBox { float modelLo[3], modelHi[3], sphLo[3], sphHi[3]; };

struct QueryParams
{
    const RtRay* rays;
    RtRayHit* hits;
    unsigned int n;
    int noCull;                                  // RT_TRACE_NO_CULL: forceDontCullBack (HL:356)
    OriginBox box;
    const RtRaySegment* segs;                    // rtTraceOcclusion: the segments and their answers (rays / hits unused)
    unsigned char* occluded;
};

constexpr float QUERY_DIR2_MIN = 9.5367431640625e-07f;      // 2^-20: |dir| >= 2^-10
constexpr float QUERY_DIR2_MAX = 1048576.0f;                 // 2^20:  |dir| <= 2^10
constexpr size_t QUERY_SMEM_BYTES = (size_t)WAVE_MAX_SMEM_SPHERES * sizeof(DevSphere);

RT_DI bool OriginInside(f3 o, const float lo[3], const float hi[3])
{
    return lo[0] <= o.x && o.x <= hi[0] && lo[1] <= o.y && o.y <= hi[1] && lo[2] <= o.z && o.z <= hi[2];
}

RT_DI bool DirectionInRange(f3 d)
{
    const float dd = dot3(d, d);
    return dd >= QUERY_DIR2_MIN && dd <= QUERY_DIR2_MAX;
}

// The first WAVE_MAX_SMEM_SPHERES spheres into the CTA's dynamic shared memory, as wave_body stages them (no tree tops)
RT_DI DevSphere* StageSpheres(const DevParams& P, unsigned char* smem)
{
    DevSphere* smemSpheres = reinterpret_cast<DevSphere*>(smem);
    const int nS = P.sphereCount < WAVE_MAX_SMEM_SPHERES ? P.sphereCount : WAVE_MAX_SMEM_SPHERES;
    for (int i = threadIdx.x; i < nS; i += WAVE_THREADS) smemSpheres[i] = P.spheres[i];
    __syncthreads();
    return smemSpheres;
}

// One persistent grid over Q.n rays (ANY = false: RtRay -> RtRayHit) or segments (ANY = true: RtRaySegment -> one byte, 1 = occluded)
template <bool STATS, bool EXT, bool TLAS, bool ANY>
RT_DI void query_body(const DevParams& P, const QueryParams& Q)
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
        if (base >= Q.n) break;
        const unsigned int i = base + lane;
        if (i < Q.n)
        {
            const float* r = ANY ? reinterpret_cast<const float*>(Q.segs + i) : reinterpret_cast<const float*>(Q.rays + i);
            const f3 o = make_f3(__ldg(r), __ldg(r + 1), __ldg(r + 2));
            const f3 d = make_f3(__ldg(r + 3), __ldg(r + 4), __ldg(r + 5));
            // the per-ray gate (the header's conditions), as path_lanes has it per segment.  Written out in both: behind a function
            // the two flags are carried as bytes rather than predicates, and the query and path kernels spill more.
            QueryRay q;
            const bool dirOk = DirectionInRange(d);
            q.modelsExact = dirOk && OriginInside(o, Q.box.modelLo, Q.box.modelHi);
            q.spheresExact = dirOk && OriginInside(o, Q.box.sphLo, Q.box.sphHi);
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
    FlushCounters<STATS>(P, cnt);
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

// A persistent launch of the query family: persistent_grid's grid over the jobs of warpsNeeded warps; the work counter the warps draw
// from starts at 0
template <class Kernel, class Params>
inline cudaError_t persistent_launch(Kernel kernel, size_t smemBytes, unsigned int warpsNeeded, const DevParams& P, const Params& Q, int numSMs,
                                     cudaStream_t stream)
{
    unsigned int grid = 0;
    cudaError_t e = persistent_grid(kernel, smemBytes, warpsNeeded, numSMs, grid);
    if (e != cudaSuccess) return e;
    if ((e = cudaMemsetAsync(P.workCounter, 0, sizeof(unsigned int), stream)) != cudaSuccess) return e;
    RT_LAUNCH(grid, WAVE_THREADS, smemBytes, stream, kernel, P, Q);
    return cudaGetLastError();
}

// ANY: the occlusion kernels
template <bool ANY = false>
inline cudaError_t query_launch(const DevParams& P, const QueryParams& Q, int numSMs, cudaStream_t stream)
{
    return with_persistent_kernel(P, [&](auto S, auto X, auto T) {
        auto kernel = ANY ? k_trace_occlusion<S, X, T> : k_trace_rays<S, X, T>;
        return persistent_launch(kernel, QUERY_SMEM_BYTES, (Q.n + 31u) / 32u, P, Q, numSMs, stream);
    });
}

// ---- path lanes: the refill loop of rtTracePaths and rtBakeProbes --------------------------------------------------------------------
// Each lane runs its job sample by sample and segment by segment: Intersect<..., QUERY = true> with the per-segment gate, then
// ShadeSegment — HL:479-542 as the camera kernels run it.  A path takes 1 .. MaxBounceCount + 1 segments, so a warp that took 32 jobs
// at once would wait for its longest chain; instead, as in kernel 1 (wave_body), every iteration first refills the lanes whose job
// has ended (ballot, one atomicAdd per warp, jobs handed out by popcount rank), then traces one segment on every lane that has a job.
// What a job is comes from the policy J, per lane:
//   J.take(job, rng)      job < jobs becomes the lane's: load it or reset its sums
//   J.begin(ray, rng)     start the ray of the job's next sample
//   J.end(ray, rng)       the sample has ended: add it up; when it was the job's last, store the result and return true
template <bool STATS, bool EXT, bool TLAS, class Job>
RT_DI void path_lanes(const DevParams& P, Job& J, unsigned int jobs, const OriginBox& box)
{
    RT_DYNAMIC_SMEM(smemRaw);
    const DevSphere* smemSpheres = StageSpheres(P, smemRaw);

    const unsigned int lane = threadIdx.x & 31u;
    const unsigned int laneMaskLt = (1u << lane) - 1u;
    Counters cnt; cnt.rays = cnt.box = cnt.tri = cnt.sph = cnt.sbox = 0;
    bool exhausted = false, haveJob = false;
    uint32_t rngState = 0;
    int bounce = 0;
    PathState ray; ray.pos = ray.dir = ray.transmittance = ray.totalLight = splat3(0.0f);

    for (;;)
    {
        // [refill] lanes without a job take the next ones (ballot + one atomic per warp)
        const bool need = !haveJob && !exhausted;
        const unsigned int needMask = __ballot_sync(0xffffffffu, need);
        if (needMask)
        {
            unsigned int base = 0;
            const int leader = __ffs(needMask) - 1;
            if ((int)lane == leader) base = atomicAdd(P.workCounter, (unsigned int)__popc(needMask));
            base = __shfl_sync(0xffffffffu, base, leader);
            if (need)
            {
                const unsigned int job = base + (unsigned int)__popc(needMask & laneMaskLt);
                if (job >= jobs) exhausted = true;
                else
                {
                    J.take(job, rngState);
                    bounce = -1;                 // a path starts below
                    haveJob = true;
                }
            }
        }
        // every lane now holds a job or has run out of them
        if (__ballot_sync(0xffffffffu, haveJob) == 0u) break;

        if (haveJob)
        {
            if (bounce < 0)
            {
                J.begin(ray, rngState);
                bounce = 0;
            }
            // [intersect] the segment, with rtTraceRays' gate on its own origin and direction (written out as in query_body)
            QueryRay q;
            const bool dirOk = DirectionInRange(ray.dir);
            q.modelsExact = dirOk && OriginInside(ray.pos, box.modelLo, box.modelHi);
            q.spheresExact = dirOk && OriginInside(ray.pos, box.sphLo, box.sphHi);
            q.noCull = false;                    // HL:487
            const Hit hit = Intersect<STATS, EXT, TLAS, true>(P, nullptr, smemSpheres, ray.pos, ray.dir, cnt, &q);
            // [shade]
            const bool cont = ShadeSegment(P, hit, ray, rngState);
            bounce++;
            if (!cont || bounce > P.MaxBounceCount)
            {
                bounce = -1;
                if (J.end(ray, rngState)) haveJob = false;
            }
        }
    }
    FlushCounters<STATS>(P, cnt);
}

// ---- rtTracePaths: the radiance along caller-supplied rays ------------------------------------------------------------------------
// A job is one caller ray: all Q.samples paths of it, on one RNG chain.
struct PathParams
{
    const RtPathRay* rays;
    RtPathRadiance* out;
    unsigned int n;
    int samples;                                 // 1 .. RT_MAX_BATCH_SAMPLES
    OriginBox box;
};

struct PathJob
{
    const PathParams& Q;
    unsigned int i = 0;                          // the lane's ray
    int sample = 0;
    f3 total = splat3(0.0f);

    RT_DI void take(unsigned int job, uint32_t& rngState)
    {
        i = job;
        rngState = __ldg(&Q.rays[i].rngState);
        total = splat3(0.0f);
        sample = 0;
    }
    // CreateRay(origin, dir, 1, 0) (HL:439-448), for every sample from the caller's record
    RT_DI void begin(PathState& ray, uint32_t&) const
    {
        const float* r = reinterpret_cast<const float*>(Q.rays + i);
        ray.pos = make_f3(__ldg(r), __ldg(r + 1), __ldg(r + 2));
        ray.dir = make_f3(__ldg(r + 3), __ldg(r + 4), __ldg(r + 5));
        ray.transmittance = splat3(1.0f);
        ray.totalLight = splat3(0.0f);
    }
    RT_DI bool end(const PathState& ray, uint32_t rngState)
    {
        total = total + ray.totalLight;                          // HL:578
        if (++sample < Q.samples) return false;
        const f3 c = total / __int2float_rn(Q.samples);          // HL:581
        reinterpret_cast<float4*>(Q.out)[i] = make_float4(c.x, c.y, c.z, __uint_as_float(rngState));
        return true;
    }
};

template <bool STATS, bool EXT, bool TLAS>
__global__ void __launch_bounds__(WAVE_THREADS, RT_WAVE_MINBLOCKS) k_trace_paths(const __grid_constant__ DevParams P, const __grid_constant__ PathParams Q)
{
    PathJob J{Q};
    path_lanes<STATS, EXT, TLAS>(P, J, Q.n, Q.box);
}

inline cudaError_t paths_launch(const DevParams& P, const PathParams& Q, int numSMs, cudaStream_t stream)
{
    return with_persistent_kernel(P, [&](auto S, auto X, auto T) {
        return persistent_launch(k_trace_paths<S, X, T>, QUERY_SMEM_BYTES, (Q.n + 31u) / 32u, P, Q, numSMs, stream);
    });
}

} // namespace rtd
