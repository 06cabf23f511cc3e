// rt_kernel_adaptive.cuh — rtDispatchAdaptive's selection: which covered pixels still need frames (the criterion is stated bit for bit
// in include/rt_b200.h), stream-compacted into the pixel list the list-driven camera kernels take their jobs from; and rtDisplayMean's mean image.
//
// The selection runs in the camera kernels' own job order (8x4 tiles, tile rows over this context's row bands, rt_kernel_wave.cuh),
// so that a warp of the render takes a compact tile while most pixels are active.  Three launches, no atomics, a deterministic order:
//   k_adaptive_flags    one thread per job: the criterion on the pixel's moments (16 B read), one ballot word per 32-job tile and
//                       the active count of each 256-job block;
//   k_adaptive_scan     one CTA: exclusive scan of the block counts, the total into `count`;
//   k_adaptive_scatter  one thread per job again: the active ones write (y << 16) | x at block offset + warp offset + rank in the ballot.
#pragma once
#include "rt_device.cuh"

namespace rtd {

constexpr int ADAPTIVE_BLOCK = 256;          // jobs per selection block (8 tiles of 32)
constexpr int ADAPTIVE_SCAN_THREADS = 1024;

struct AdaptiveParams
{
    const float4* moments;                   // AdaptiveMoments, or nullptr before the first traced frame (all zero)
    unsigned int* masks;                     // one ballot word per tile of 32 jobs
    unsigned int* partials;                  // active pixels per block, then (k_adaptive_scan) their exclusive prefix
    unsigned int* list;                      // the active pixels, (y << 16) | x
    unsigned int* count;                     // their number
    unsigned int W, limX, ownedRows, tilesX, totalJobs, nBlocks;
    int tileRank, tileWorld, bandRows;
    float threshold, minFrames, maxFrames;
};

// The job's pixel (the mapping of the camera kernels' refill); false for the padding jobs of partial tiles
RT_DI bool AdaptiveJobPixel(const AdaptiveParams& A, unsigned int job, unsigned int& x, unsigned int& y)
{
    const unsigned int tile = job >> 5, l = job & 31u;
    x = (tile % A.tilesX) * 8u + (l & 7u);
    const unsigned int r = (tile / A.tilesX) * 4u + (l >> 3);
    if (job >= A.totalJobs || x >= A.limX || r >= A.ownedRows) return false;
    y = ((r / (unsigned int)A.bandRows) * (unsigned int)A.tileWorld + (unsigned int)A.tileRank) * (unsigned int)A.bandRows + (r % (unsigned int)A.bandRows);
    return true;
}

// include/rt_b200.h, rtDispatchAdaptive: binary32, one operation each in the order written (-fmad=false), NaN-ignoring max
RT_DI bool AdaptiveActive(const float4 m, float threshold, float minFrames, float maxFrames)
{
    const float n = m.z;
    const float mu = m.x / n;
    const float v = fmaxf(m.y / n - mu * mu, 0.0f);
    return n < minFrames || (n < maxFrames && v > ((threshold * threshold) * n) * (mu * mu + RT_ADAPTIVE_EPSILON));
}

__global__ void __launch_bounds__(ADAPTIVE_BLOCK) k_adaptive_flags(const __grid_constant__ AdaptiveParams A)
{
    __shared__ unsigned int warpCount[ADAPTIVE_BLOCK / 32];
    const unsigned int job = blockIdx.x * (unsigned int)ADAPTIVE_BLOCK + threadIdx.x;
    const unsigned int lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    unsigned int x = 0, y = 0;
    bool active = false;
    if (AdaptiveJobPixel(A, job, x, y))
    {
        const float4 m = A.moments ? A.moments[(size_t)y * A.W + x] : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        active = AdaptiveActive(m, A.threshold, A.minFrames, A.maxFrames);
    }
    const unsigned int mask = __ballot_sync(0xffffffffu, active);
    if (lane == 0)
    {
        if (job < A.totalJobs) A.masks[job >> 5] = mask;          // totalJobs is a multiple of 32: a warp is all in or all out
        warpCount[warp] = (unsigned int)__popc(mask);
    }
    __syncthreads();
    if (threadIdx.x == 0)
    {
        unsigned int s = 0;
        for (int w = 0; w < ADAPTIVE_BLOCK / 32; w++) s += warpCount[w];
        A.partials[blockIdx.x] = s;
    }
}

__global__ void __launch_bounds__(ADAPTIVE_SCAN_THREADS) k_adaptive_scan(const __grid_constant__ AdaptiveParams A)
{
    __shared__ unsigned int warpSum[ADAPTIVE_SCAN_THREADS / 32];
    __shared__ unsigned int carry;
    const unsigned int lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (unsigned int base = 0; base < A.nBlocks; base += ADAPTIVE_SCAN_THREADS)
    {
        const unsigned int i = base + threadIdx.x;
        const unsigned int v = i < A.nBlocks ? A.partials[i] : 0u;
        unsigned int incl = v;                                    // inclusive scan within the warp
        for (unsigned int d = 1; d < 32u; d <<= 1)
        {
            const unsigned int t = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= d) incl += t;
        }
        if (lane == 31u) warpSum[warp] = incl;
        __syncthreads();
        if (warp == 0)
        {
            unsigned int w = warpSum[lane], wincl = w;
            for (unsigned int d = 1; d < 32u; d <<= 1)
            {
                const unsigned int t = __shfl_up_sync(0xffffffffu, wincl, d);
                if (lane >= d) wincl += t;
            }
            warpSum[lane] = wincl - w;                            // exclusive prefix of the warps
        }
        __syncthreads();
        const unsigned int c = carry;
        if (i < A.nBlocks) A.partials[i] = c + warpSum[warp] + (incl - v);
        __syncthreads();
        if (threadIdx.x == ADAPTIVE_SCAN_THREADS - 1) carry = c + warpSum[warp] + incl;
        __syncthreads();
    }
    if (threadIdx.x == 0) *A.count = carry;
}

__global__ void __launch_bounds__(ADAPTIVE_BLOCK) k_adaptive_scatter(const __grid_constant__ AdaptiveParams A)
{
    __shared__ unsigned int warpBase[ADAPTIVE_BLOCK / 32];
    const unsigned int job = blockIdx.x * (unsigned int)ADAPTIVE_BLOCK + threadIdx.x;
    const unsigned int lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    const unsigned int mask = job < A.totalJobs ? A.masks[job >> 5] : 0u;
    if (lane == 0) warpBase[warp] = (unsigned int)__popc(mask);
    __syncthreads();
    if (threadIdx.x == 0)
    {
        unsigned int s = A.partials[blockIdx.x];
        for (int w = 0; w < ADAPTIVE_BLOCK / 32; w++) { const unsigned int c = warpBase[w]; warpBase[w] = s; s += c; }
    }
    __syncthreads();
    if (mask & (1u << lane))
    {
        unsigned int x = 0, y = 0;
        AdaptiveJobPixel(A, job, x, y);
        A.list[warpBase[warp] + (unsigned int)__popc(mask & ((1u << lane) - 1u))] = (y << 16) | x;
    }
}

inline cudaError_t adaptive_select(const AdaptiveParams& A, cudaStream_t stream)
{
    if (A.nBlocks == 0) return cudaMemsetAsync(A.count, 0, sizeof(unsigned int), stream);
    RT_LAUNCH(A.nBlocks, ADAPTIVE_BLOCK, 0, stream, k_adaptive_flags, A);
    RT_LAUNCH(1, ADAPTIVE_SCAN_THREADS, 0, stream, k_adaptive_scan, A);
    RT_LAUNCH(A.nBlocks, ADAPTIVE_BLOCK, 0, stream, k_adaptive_scatter, A);
    return cudaGetLastError();
}

// rtDisplayMean's first step: the per-pixel mean A / A.w, (0, 0, 0, 1) where no frame was accumulated; rtDisplay's own k_display
// then encodes it with Frame = 1 (q / 1 is exact), so that the encode stays one kernel's code
__global__ void k_mean_image(const float4* __restrict__ tex, float4* __restrict__ out, size_t n)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 t = tex[i];
    out[i] = t.w == 0.0f ? make_float4(0.0f, 0.0f, 0.0f, 1.0f) : make_float4(t.x / t.w, t.y / t.w, t.z / t.w, t.w / t.w);
}

} // namespace rtd
