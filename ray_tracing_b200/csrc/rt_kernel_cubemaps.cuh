// rt_kernel_cubemaps.cuh — rtBakeCubemaps: HDR cube maps of path-traced radiance at probe positions (reflection probes), and
// rtBakeLightmap: cosine-weighted path-traced lighting at surface texels.  A lightmap texel is a second kind of texel of the same two
// kernels: only its origin and the direction of each sample differ (CubeJob::begin), chosen by CubeParams::points, which is uniform
// across a launch.
//
// Two launches per batch of texels (include/rt_b200.h states the contract):
//   k_bake_cubemaps  the path tracer's samples.  A job is one (texel, chunk) pair: RT_PROBE_CHUNK consecutive samples of one texel,
//                    each along its own direction through an R2 point of the texel's area, run in rtTracePaths' path lanes
//                    (path_lanes, rt_kernel_query.cuh).  The chunk's 3 sums and its rejected count stay in registers: unlike
//                    rtBakeProbes' 27 sums, they are PathJob's running total plus one word (DESIGN.md §7d''''''''''' has the
//                    -Xptxas -v figures).  A finished chunk writes one 16-byte record of the scratch.
//   k_cube_sums      one thread per (texel, word): rtBakeProbes' tree (ChunkTree, rt_kernel_probes.cuh), then the division by S.
#pragma once
#include "rt_kernel_probes.cuh"

namespace rtd {

constexpr int CUBE_WORDS = 4;                    // a chunk record: rgb as RtCubeTexel lays it out, then the rejected count

struct CubeParams
{
    const float* positions;                      // the call's probes, 3 floats each
    float* scratch;                              // n * chunks records of CUBE_WORDS words, texel-major
    RtCubeTexel* out;                            // the launch's first texel
    unsigned int n;                              // texels in this launch
    unsigned int t0;                             // the call's index of the launch's first texel
    unsigned int chunks;                         // ceil(samples / RT_PROBE_CHUNK)
    unsigned int faceSize;                       // N: 1 .. RT_CUBE_MAX_FACE
    int samples;                                 // 1 .. RT_MAX_BATCH_SAMPLES
    uint32_t seed;
    OriginBox box;
    const RtSurfacePoint* points;                // rtBakeLightmap: the launch's first texel's point; nullptr for cube maps
};

// The direction of sample k of texel (x, y) of face f, one binary32 operation at a time (the contract in include/rt_b200.h)
RT_DI f3 CubeDirection(unsigned int f, unsigned int x, unsigned int y, unsigned int k, unsigned int N)
{
    const float u = __uint2float_rn(k * 3242174889u + 2147483648u) * 2.3283064365386963e-10f;     // R2, RandomValue's conversion
    const float v = __uint2float_rn(k * 2447445414u + 2147483648u) * 2.3283064365386963e-10f;
    const float n = __uint2float_rn(N);
    const float a = ((__uint2float_rn(x) + u) / n) * 2.0f - 1.0f;
    const float b = ((__uint2float_rn(y) + v) / n) * 2.0f - 1.0f;
    f3 w;
    switch (f)
    {
    case 0:  w = make_f3(1.0f, -b, -a); break;
    case 1:  w = make_f3(-1.0f, -b, a); break;
    case 2:  w = make_f3(a, 1.0f, b); break;
    case 3:  w = make_f3(a, -1.0f, -b); break;
    case 4:  w = make_f3(a, -b, 1.0f); break;
    default: w = make_f3(-a, -b, -1.0f); break;
    }
    return normalize3(w);
}

// Sample k of a lightmap texel at (position P, normal M), one binary32 operation at a time (the contract in include/rt_b200.h): the
// origin P + n * 0.001 and a cosine-weighted direction about n = normalize(M) through the R2 point (u, v), in Duff et al.'s frame
RT_DI void SurfaceRay(f3 P, f3 M, unsigned int k, f3& origin, f3& dir)
{
    const float u = __uint2float_rn(k * 3242174889u + 2147483648u) * 2.3283064365386963e-10f;     // R2, as CubeDirection
    const float v = __uint2float_rn(k * 2447445414u + 2147483648u) * 2.3283064365386963e-10f;
    const f3 n = normalize3(M);
    const float sg = copysignf(1.0f, n.z);
    const float a = -1.0f / (sg + n.z);
    const float b = (n.x * n.y) * a;
    const f3 T = make_f3(1.0f + ((sg * n.x) * n.x) * a, sg * b, -(sg * n.x));
    const f3 B = make_f3(b, sg + (n.y * n.y) * a, -n.y);
    const float r = sqrtf(u);
    float s, c; sincos_rt(v * 6.28318548f, s, c);
    const float x = r * c, y = r * s, z = sqrtf(fmaxf(1.0f - u, 0.0f));
    dir = normalize3(make_f3((T.x * x + B.x * y) + n.x * z, (T.y * x + B.y * y) + n.y * z, (T.z * x + B.z * y) + n.z * z));
    origin = make_f3(P.x + n.x * 0.001f, P.y + n.y * 0.001f, P.z + n.z * 0.001f);
}

// A job is one (texel, chunk) pair: samples k .. kEnd - 1 of texel tau = t0 + job / Q.chunks, each from CreateRay(origin, d, 1, 0)
// (HL:439-448) with state H(H(seed + tau) + k), summed into the lane's registers.  The origin is the probe's position (cube maps) or
// the surface point lifted off its surface (lightmaps).
struct CubeJob
{
    const CubeParams& Q;
    unsigned int job = 0, k = 0, kEnd = 0, rejected = 0;    // the lane's (texel, chunk) job, its current sample, the chunk's end
    uint32_t texelKey = 0;                                  // H(seed + tau)
    f3 sum = splat3(0.0f);

    RT_DI unsigned int tau() const { return Q.t0 + job / Q.chunks; }
    RT_DI void take(unsigned int j, uint32_t&)
    {
        job = j;
        k = (job - (job / Q.chunks) * Q.chunks) * PROBE_CHUNK;
        kEnd = k + PROBE_CHUNK < (unsigned int)Q.samples ? k + PROBE_CHUNK : (unsigned int)Q.samples;
        texelKey = ProbeHash(Q.seed + tau());
        sum = splat3(0.0f);
        rejected = 0;
    }
    RT_DI void begin(PathState& ray, uint32_t& rngState) const
    {
        if (Q.points)                                       // a lightmap texel: point job / chunks of the launch
        {
            const float* s = reinterpret_cast<const float*>(Q.points + job / Q.chunks);
            SurfaceRay(make_f3(__ldg(s), __ldg(s + 1), __ldg(s + 2)), make_f3(__ldg(s + 3), __ldg(s + 4), __ldg(s + 5)), k, ray.pos, ray.dir);
        }
        else
        {
            const unsigned int N = Q.faceSize, t = tau();
            const unsigned int row = t / N, x = t - row * N, face = row / N, y = row - face * N, p = face / 6u, f = face - p * 6u;
            const float* o = Q.positions + 3u * p;
            ray.pos = make_f3(__ldg(o), __ldg(o + 1), __ldg(o + 2));
            ray.dir = CubeDirection(f, x, y, k, N);
        }
        ray.transmittance = splat3(1.0f);
        ray.totalLight = splat3(0.0f);
        rngState = ProbeHash(texelKey + k);
    }
    RT_DI bool end(const PathState& ray, uint32_t)
    {
        const f3 L = ray.totalLight;
        if (Finite3(L)) sum = sum + L;
        else rejected++;
        if (++k < kEnd) return false;
        reinterpret_cast<float4*>(Q.scratch)[job] = make_float4(sum.x, sum.y, sum.z, __uint_as_float(rejected));
        return true;
    }
};

template <bool STATS, bool EXT, bool TLAS>
__global__ void __launch_bounds__(WAVE_THREADS, RT_WAVE_MINBLOCKS) k_bake_cubemaps(const __grid_constant__ DevParams P, const __grid_constant__ CubeParams Q)
{
    CubeJob J{Q};
    path_lanes<STATS, EXT, TLAS>(P, J, Q.n * Q.chunks, Q.box);
}

// The texel's mean: the tree over S, one IEEE division as rtTracePaths divides its total
__global__ void __launch_bounds__(PROBE_SUM_THREADS) k_cube_sums(const __grid_constant__ CubeParams Q)
{
    ChunkTree<CUBE_WORDS>(Q.scratch, Q.out, Q.n, Q.chunks,
                          [&](float r) { return r / __int2float_rn(Q.samples); });
}

// k_bake_cubemaps over the launch's n * chunks jobs, then k_cube_sums over its records
inline cudaError_t cubemaps_launch(const DevParams& P, const CubeParams& Q, int numSMs, cudaStream_t stream)
{
    cudaError_t e = with_persistent_kernel(P, [&](auto S, auto X, auto T) {
        return persistent_launch(k_bake_cubemaps<S, X, T>, QUERY_SMEM_BYTES, (Q.n * Q.chunks + 31u) / 32u, P, Q, numSMs, stream);
    });
    if (e != cudaSuccess) return e;
    RT_LAUNCH((Q.n * CUBE_WORDS + PROBE_SUM_THREADS - 1) / PROBE_SUM_THREADS, PROBE_SUM_THREADS, 0, stream, k_cube_sums, Q);
    return cudaGetLastError();
}

} // namespace rtd
