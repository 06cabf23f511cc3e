// rt_kernel_probes.cuh — rtBakeProbes: path-traced radiance around probe positions, projected onto L2 spherical harmonics.
//
// Two launches per batch of probes (include/rt_b200.h states the contract):
//   k_bake_probes  the path tracer's samples.  A job is one (probe, chunk) pair: RT_PROBE_CHUNK consecutive samples of one probe, so
//                  the grid fills from n * ceil(S / 32) jobs however few the probes are.  Each lane runs its job sample by sample and
//                  segment by segment in rtTracePaths' path lanes (path_lanes, rt_kernel_query.cuh: kernel 1's refill,
//                  Intersect<..., QUERY = true> with the per-segment gate and ShadeSegment), and adds L * Y_i into the chunk's 27
//                  sums.  The sums live in shared memory, one column per lane (sums[v * WAVE_THREADS + threadIdx.x]: no bank
//                  conflicts), not in registers: k_trace_paths already spills at the 80-register cap, and 27 more live floats
//                  across Intersect would all go to local memory (DESIGN.md §7d''''''''' has the -Xptxas -v figures).  A finished
//                  chunk writes its 27 sums and its rejected count as one 112-byte record of the scratch.
//   k_probe_sums   one thread per (probe, word): the tree over the probe's chunk records, the scale, the store into RtProbeSH
//                  (ChunkTree, which rtBakeCubemaps' k_cube_sums shares).
#pragma once
#include "rt_kernel_query.cuh"

namespace rtd {

constexpr unsigned int PROBE_CHUNK = RT_PROBE_CHUNK;
constexpr int PROBE_WORDS = 28;                  // a chunk record: sh[3][9] as RtProbeSH lays it out, then the rejected count
constexpr int PROBE_SUM_THREADS = 256;

struct ProbeParams
{
    const float* positions;                      // the launch's probes, 3 floats each
    float* scratch;                              // n * chunks records of PROBE_WORDS words, probe-major
    RtProbeSH* out;
    unsigned int n;                              // probes in this launch
    unsigned int p0;                             // the call's index of the launch's first probe
    unsigned int chunks;                         // ceil(samples / RT_PROBE_CHUNK)
    int samples;                                 // 1 .. RT_MAX_BATCH_SAMPLES
    uint32_t seed;
    OriginBox box;
};

// Sample k of S: a spherical Fibonacci set, one binary32 operation at a time (the contract in include/rt_b200.h)
RT_DI f3 ProbeDirection(unsigned int k, int samples)
{
    const float t = __uint2float_rn(k * 2654435769u) * 2.3283064365386963e-10f;     // RandomValue's conversion
    const float phi = t * 6.28318548f;
    float s, c; sincos_rt(phi, s, c);
    const float z = 1.0f - __uint2float_rn(2u * k + 1u) / __int2float_rn(samples);
    const float r = sqrtf(fmaxf(1.0f - z * z, 0.0f));
    return make_f3(r * c, r * s, z);
}

// H(x): the value NextRandom returns from state x
RT_DI uint32_t ProbeHash(uint32_t x) { return NextRandom(x); }

RT_DI bool Finite3(f3 v)
{
    return fabsf(v.x) <= 3.40282347e38f && fabsf(v.y) <= 3.40282347e38f && fabsf(v.z) <= 3.40282347e38f;
}

// The nine real L2 basis functions at d, in Unity's order (l, then m = -l .. l)
RT_DI void ProbeBasis(f3 d, float Y[9])
{
    Y[0] = 0.282094792f;
    Y[1] = 0.488602512f * d.y; Y[2] = 0.488602512f * d.z; Y[3] = 0.488602512f * d.x;
    Y[4] = 1.09254843f * (d.x * d.y); Y[5] = 1.09254843f * (d.y * d.z);
    Y[6] = 0.315391565f * ((3.0f * (d.z * d.z)) - 1.0f);
    Y[7] = 1.09254843f * (d.x * d.z);
    Y[8] = 0.546274215f * ((d.x * d.x) - (d.y * d.y));
}

// A job is one (probe, chunk) pair: samples k .. kEnd - 1 of probe job / Q.chunks, each from CreateRay(position, d_k, 1, 0)
// (HL:439-448) with state H(H(seed + p) + k), projected onto the basis at d_k into the lane's column of the shared sums.
struct ProbeJob
{
    const ProbeParams& Q;
    float* sums;                                 // this lane's column of 27 (sums[v * WAVE_THREADS])
    unsigned int job = 0, k = 0, kEnd = 0, rejected = 0;    // the lane's (probe, chunk) job, its current sample, the chunk's end
    uint32_t probeKey = 0;                                  // H(seed + p)

    RT_DI void take(unsigned int j, uint32_t&)
    {
        job = j;
        const unsigned int p = job / Q.chunks, chunk = job - p * Q.chunks;
        k = chunk * PROBE_CHUNK;
        kEnd = k + PROBE_CHUNK < (unsigned int)Q.samples ? k + PROBE_CHUNK : (unsigned int)Q.samples;
        probeKey = ProbeHash(Q.seed + Q.p0 + p);
        for (int v = 0; v < 27; v++) sums[v * WAVE_THREADS] = 0.0f;
        rejected = 0;
    }
    RT_DI void begin(PathState& ray, uint32_t& rngState) const
    {
        const float* o = Q.positions + 3u * (job / Q.chunks);
        ray.pos = make_f3(__ldg(o), __ldg(o + 1), __ldg(o + 2));
        ray.dir = ProbeDirection(k, Q.samples);
        ray.transmittance = splat3(1.0f);
        ray.totalLight = splat3(0.0f);
        rngState = ProbeHash(probeKey + k);
    }
    RT_DI bool end(const PathState& ray, uint32_t)
    {
        // [project] the sample's Trace result onto the basis at its direction (recomputed: fewer live registers)
        const f3 L = ray.totalLight;
        if (Finite3(L))
        {
            float Y[9]; ProbeBasis(ProbeDirection(k, Q.samples), Y);
#pragma unroll
            for (int i = 0; i < 9; i++)
            {
                sums[i * WAVE_THREADS] = sums[i * WAVE_THREADS] + L.x * Y[i];
                sums[(9 + i) * WAVE_THREADS] = sums[(9 + i) * WAVE_THREADS] + L.y * Y[i];
                sums[(18 + i) * WAVE_THREADS] = sums[(18 + i) * WAVE_THREADS] + L.z * Y[i];
            }
        }
        else rejected++;
        if (++k < kEnd) return false;
        float4* rec = reinterpret_cast<float4*>(Q.scratch + (size_t)job * PROBE_WORDS);
#pragma unroll
        for (int w = 0; w < 6; w++)
            rec[w] = make_float4(sums[(4 * w) * WAVE_THREADS], sums[(4 * w + 1) * WAVE_THREADS], sums[(4 * w + 2) * WAVE_THREADS], sums[(4 * w + 3) * WAVE_THREADS]);
        rec[6] = make_float4(sums[24 * WAVE_THREADS], sums[25 * WAVE_THREADS], sums[26 * WAVE_THREADS], __uint_as_float(rejected));
        return true;
    }
};

// The sums follow the staged spheres in the dynamic shared memory
template <bool STATS, bool EXT, bool TLAS>
__global__ void __launch_bounds__(WAVE_THREADS, RT_WAVE_MINBLOCKS) k_bake_probes(const __grid_constant__ DevParams P, const __grid_constant__ ProbeParams Q)
{
    RT_DYNAMIC_SMEM(smemRaw);
    ProbeJob J{Q, reinterpret_cast<float*>(smemRaw + QUERY_SMEM_BYTES) + threadIdx.x};
    path_lanes<STATS, EXT, TLAS>(P, J, Q.n * Q.chunks, Q.box);
}

// Word v of item p (a probe, a cube-map texel): the item's chunk records (WORDS words each, item-major; the last word the rejected
// count) combined by the full binary tree over the chunk count padded to a power of two with +0 chunks, adjacent chunks paired, then
// finished by fin (the scale or the division by S).  The tree is built left to right on a stack: after chunk c the stack holds the
// complete subtrees of the first c + 1 chunks (one per set bit of c + 1, largest first), and the padded root is their right fold:
// a subtree made only of padding is +0, and x + +0 = x for every value a sum from +0 can take (never -0).  The rejected counts add
// as integers.  out holds n items (Item: WORDS words laid out as the records are).
template <int WORDS, class Item, class Finish>
RT_DI void ChunkTree(const float* scratch, Item* out, unsigned int n, unsigned int chunks, Finish fin)
{
    const unsigned int t = blockIdx.x * PROBE_SUM_THREADS + threadIdx.x;
    if (t >= n * WORDS) return;
    const unsigned int p = t / WORDS, v = t - p * WORDS;
    const float* rec = scratch + (size_t)p * chunks * WORDS + v;
    float* o = reinterpret_cast<float*>(out + p) + v;
    if (v == WORDS - 1)
    {
        unsigned int r = 0;
        for (unsigned int c = 0; c < chunks; c++) r += __float_as_uint(rec[(size_t)c * WORDS]);
        *o = __uint_as_float(r);
        return;
    }
    float stack[16];                             // chunks <= 2^15: at most 16 complete subtrees
    int top = 0;
    for (unsigned int c = 0; c < chunks; c++)
    {
        float s = rec[(size_t)c * WORDS];
        for (unsigned int m = c + 1u; (m & 1u) == 0u; m >>= 1) s = stack[--top] + s;
        stack[top++] = s;
    }
    float r = stack[--top];
    while (top > 0) r = stack[--top] + r;
    *o = fin(r);
}

// The probe's SH coefficients: the tree scaled by 4 pi / S
__global__ void __launch_bounds__(PROBE_SUM_THREADS) k_probe_sums(const __grid_constant__ ProbeParams Q)
{
    ChunkTree<PROBE_WORDS>(Q.scratch, Q.out, Q.n, Q.chunks,
                           [&](float r) { return r * (12.566371f / __int2float_rn(Q.samples)); });
}

// k_bake_probes over the launch's n * chunks jobs, then k_probe_sums over its records
inline cudaError_t probes_launch(const DevParams& P, const ProbeParams& Q, int numSMs, cudaStream_t stream)
{
    cudaError_t e = with_persistent_kernel(P, [&](auto S, auto X, auto T) {
        return persistent_launch(k_bake_probes<S, X, T>, QUERY_SMEM_BYTES + (size_t)27 * WAVE_THREADS * sizeof(float), (Q.n * Q.chunks + 31u) / 32u,
                                 P, Q, numSMs, stream);
    });
    if (e != cudaSuccess) return e;
    RT_LAUNCH((Q.n * PROBE_WORDS + PROBE_SUM_THREADS - 1) / PROBE_SUM_THREADS, PROBE_SUM_THREADS, 0, stream, k_probe_sums, Q);
    return cudaGetLastError();
}

} // namespace rtd
