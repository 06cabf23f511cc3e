// rt_kernel_mega.cuh — kernel variant 0: the reference-shaped per-pixel megakernel.
//
// One thread per pixel, 8x8 thread groups, the reference's own buffer layouts (32-byte nodes, 72-byte
// triangles, 224-byte models) and its loop structure (RC:10-24, HL:234-287,335-374,479-582).  It exists
// (a) as the simplest statement of the arithmetic on the device, parity-checked against the CPU oracle,
// and (b) as the baseline the persistent wavefront kernel (variant 1) is measured against.
#pragma once
#include "rt_device.cuh"

namespace rtd {

// HL:234-287 on the reference layout (node re-read on pop, push-time culling only)
RT_DI void RayTriangleBVH_ref(const DevParams& P, f3 pos, f3 dir, f3 invDir, float rayLength, int nodeOffset, int triOffset,
                              bool cullBackface, float& bestDst, int& bestTri, float& bestU, float& bestV, float& bestDet,
                              Counters& cnt)
{
    bestDst = rayLength; bestTri = -1;
    int stack[64];
    int stackCount = 0;
    stack[stackCount++] = nodeOffset;
    while (stackCount > 0)
    {
        const RtNode node = P.Nodes[stack[--stackCount]];
        if (node.triangleCount > 0)
        {
            for (int i = 0; i < node.triangleCount; i++)
            {
                const int t = triOffset + node.startIndex + i;
                const RtTriangle* tri = P.Triangles + t;
                const f3 A = load3(tri->posA), B = load3(tri->posB), C = load3(tri->posC);
                const f3 edgeAB = B - A, edgeAC = C - A;
                float dst, u, v, det;
                const bool didHit = RayTriangleCore(pos, dir, A, edgeAB, edgeAC, cross3(edgeAB, edgeAC), cullBackface, dst, u, v, det);
                cnt.tri++;
                if (didHit && dst < bestDst) { bestDst = dst; bestTri = t; bestU = u; bestV = v; bestDet = det; }
            }
        }
        else
        {
            const int childIndexA = nodeOffset + node.startIndex;
            const int childIndexB = childIndexA + 1;
            const RtNode childA = P.Nodes[childIndexA];
            const RtNode childB = P.Nodes[childIndexB];
            const float dstA = RayBoundingBoxDst(pos, invDir, load3(childA.boundsMin), load3(childA.boundsMax));
            const float dstB = RayBoundingBoxDst(pos, invDir, load3(childB.boundsMin), load3(childB.boundsMax));
            cnt.box += 2;
            const bool isNearestA = dstA <= dstB;
            const float dstNear = isNearestA ? dstA : dstB;
            const float dstFar = isNearestA ? dstB : dstA;
            const int childIndexNear = isNearestA ? childIndexA : childIndexB;
            const int childIndexFar = isNearestA ? childIndexB : childIndexA;
            if (dstFar < bestDst && stackCount < 64) stack[stackCount++] = childIndexFar;
            if (dstNear < bestDst && stackCount < 64) stack[stackCount++] = childIndexNear;
        }
    }
}

// HL:335-374 (+ sphere extension before the model loop)
RT_DI Hit CalculateRayCollision_ref(const DevParams& P, f3 rayPos, f3 rayDir, Counters& cnt)
{
    Hit result;
    result.dst = inf32(); result.isBackface = false; result.normal = splat3(0.0f); result.pos = splat3(0.0f); result.material = nullptr;
    cnt.rays++;

    if (P.sphBvh)
    {
        int idx = 0x7fffffff, flag = 0; bool inside = false;
        TraverseSpheres(P, rayPos, rayDir, result.dst, idx, inside, flag, cnt, true);
        if (idx != 0x7fffffff)
        {
            const RtSphere* sp = P.Spheres + idx;
            result.isBackface = inside;
            result.pos = rayPos + rayDir * result.dst;
            result.normal = normalize3(result.pos - load3(sp->centre)) * (inside ? -1.0f : 1.0f);
            result.material = &sp->material;
        }
    }
    else
    for (int i = 0; i < P.sphereCount; i++)
    {
        const RtSphere* sp = P.Spheres + i;
        const f3 centre = load3(sp->centre);
        float dst; bool inside;
        cnt.sph++;
        if (RaySphereCore(rayPos, rayDir, centre, sp->radius * sp->radius, dst, inside) && dst < result.dst)
        {
            result.dst = dst; result.isBackface = inside;
            result.pos = rayPos + rayDir * dst;
            result.normal = normalize3(result.pos - centre) * (inside ? -1.0f : 1.0f);
            result.material = &sp->material;
        }
    }

    for (int i = 0; i < P.modelCount; i++)
    {
        const RtModel* model = P.ModelInfo + i;
        const f3 localPos = mul_cm(model->worldToLocal, rayPos, 1.0f);
        const f3 localDir = mul_cm(model->worldToLocal, rayDir, 0.0f);
        const f3 invDir = rcp3(localDir);
        const bool cullBackface = model->material.flag != RT_MATERIAL_GLASS;
        float dst, u, v, det; int tri;
        RayTriangleBVH_ref(P, localPos, localDir, invDir, result.dst, model->nodeOffset, model->triOffset, cullBackface, dst, tri, u, v, det, cnt);
        if (dst < result.dst)
        {
            const RtTriangle* t = P.Triangles + tri;
            const f3 n = TriangleSmoothNormal(load3(t->normA), load3(t->normB), load3(t->normC), u, v, det);
            result.isBackface = det < 0.0f;
            result.dst = dst;
            result.normal = normalize3(mul_cm(model->localToWorld, n, 0.0f));
            result.pos = rayPos + rayDir * dst;
            result.material = &model->material;
        }
    }
    return result;
}

RT_DI void FlushCounters(const DevParams& P, const Counters& cnt)
{
    // warp-aggregate, then one atomic per warp per counter
    unsigned int r = cnt.rays, b = cnt.box, t = cnt.tri, s = cnt.sph, sb = cnt.sbox;
    const unsigned int m = __activemask();
    r = __reduce_add_sync(m, r);
    if (P.countStats) { b = __reduce_add_sync(m, b); t = __reduce_add_sync(m, t); s = __reduce_add_sync(m, s); sb = __reduce_add_sync(m, sb); }
    const int lane = (threadIdx.x + threadIdx.y * blockDim.x) & 31;
    if (lane == (__ffs(m) - 1))
    {
        atomicAdd(P.counters + 0, (unsigned long long)r);
        if (P.countStats)
        {
            atomicAdd(P.counters + 1, (unsigned long long)b);
            atomicAdd(P.counters + 2, (unsigned long long)t);
            atomicAdd(P.counters + 3, (unsigned long long)s);
            atomicAdd(P.counters + 4, (unsigned long long)sb);
        }
    }
}

// RC:10-24
__global__ void __launch_bounds__(64) k_raytrace_mega(const __grid_constant__ DevParams P)
{
    const unsigned int idx = blockIdx.x * 8u + threadIdx.x;
    const unsigned int idy = blockIdx.y * 8u + threadIdx.y;
    if (idx >= P.limX || idy >= P.limY) return;
    if ((int)((idy / (unsigned int)P.bandRows) % (unsigned int)P.tileWorld) != P.tileRank) return;

    Counters cnt; cnt.rays = cnt.box = cnt.tri = cnt.sph = cnt.sbox = 0;
    const PixelSetup px = SetupPixel(P, idx, idy);
    uint32_t rngState = px.rngState;
    f3 totalIncomingLight = splat3(0.0f);

    for (int rayIndex = 0; rayIndex < P.NumRaysPerPixel; rayIndex++)
    {
        PathState ray;
        GenerateCameraRay(P, px, rngState, ray);
        for (int i = 0; i <= P.MaxBounceCount; i++)
        {
            const Hit hit = CalculateRayCollision_ref(P, ray.pos, ray.dir, cnt);
            if (!ShadeSegment(P, hit, ray, rngState)) break;
        }
        totalIncomingLight = totalIncomingLight + ray.totalLight;
    }
    const f3 pixelCol = totalIncomingLight / __int2float_rn(P.NumRaysPerPixel);

    const size_t o = (size_t)idy * P.W + idx;
    WritePixel<true>(P, o, pixelCol.x, pixelCol.y, pixelCol.z);
    if (P.countStats) { Counters zero; zero.rays = zero.box = zero.tri = zero.sph = zero.sbox = 0; AddPixelStats(P, o, cnt, zero); }
    FlushCounters(P, cnt);
}

// rtDispatchFrames: k_raytrace_mega for frames Frame .. Frame + P.frames - 1 of the thread's pixel, one after the other, each written
// and accumulated as its own dispatch would.  (A kernel of its own: folding the frame loop into k_raytrace_mega changed that kernel's code.)
__global__ void __launch_bounds__(64) k_raytrace_mega_frames(const __grid_constant__ DevParams P)
{
    const unsigned int idx = blockIdx.x * 8u + threadIdx.x;
    const unsigned int idy = blockIdx.y * 8u + threadIdx.y;
    if (idx >= P.limX || idy >= P.limY) return;
    if ((int)((idy / (unsigned int)P.bandRows) % (unsigned int)P.tileWorld) != P.tileRank) return;

    Counters cnt; cnt.rays = cnt.box = cnt.tri = cnt.sph = cnt.sbox = 0;
    const PixelSetup px = SetupPixel(P, idx, idy);
    const size_t o = (size_t)idy * P.W + idx;
    for (int frame = 0; frame < P.frames; frame++)
    {
        uint32_t rngState = FrameSeed(px.rngState, (unsigned int)frame);
        f3 totalIncomingLight = splat3(0.0f);
        for (int rayIndex = 0; rayIndex < P.NumRaysPerPixel; rayIndex++)
        {
            PathState ray;
            GenerateCameraRay(P, px, rngState, ray);
            for (int i = 0; i <= P.MaxBounceCount; i++)
            {
                const Hit hit = CalculateRayCollision_ref(P, ray.pos, ray.dir, cnt);
                if (!ShadeSegment(P, hit, ray, rngState)) break;
            }
            totalIncomingLight = totalIncomingLight + ray.totalLight;
        }
        const f3 pixelCol = totalIncomingLight / __int2float_rn(P.NumRaysPerPixel);
        WritePixel<true>(P, o, pixelCol.x, pixelCol.y, pixelCol.z);
    }
    if (P.countStats) { Counters zero; zero.rays = zero.box = zero.tri = zero.sph = zero.sbox = 0; AddPixelStats(P, o, cnt, zero); }
    FlushCounters(P, cnt);
}

// rtDispatchAdaptive: k_raytrace_mega over the `count` pixels of the selection's list ((y << 16) | x each), a 1-D grid of BLOCK-thread
// blocks; the write also updates the pixel's moments.  (A kernel of its own, so that k_raytrace_mega keeps its code; and a template,
// instantiated where mega_launch launches it: defined here as a plain kernel, it moved ahead of the wavefront kernels in the module and
// the compiler then numbered the registers of the k_raytrace_wave_frames kernels differently.)
template <unsigned int BLOCK>
__global__ void __launch_bounds__(BLOCK) k_raytrace_mega_list(const __grid_constant__ DevParams P, const unsigned int count,
                                                              const unsigned int* __restrict__ list, float4* __restrict__ moments)
{
    const unsigned int job = blockIdx.x * BLOCK + threadIdx.x;
    if (job >= count) return;
    const unsigned int xy = list[job];
    const unsigned int idx = xy & 0xffffu, idy = xy >> 16;

    Counters cnt; cnt.rays = cnt.box = cnt.tri = cnt.sph = cnt.sbox = 0;
    const PixelSetup px = SetupPixel(P, idx, idy);
    uint32_t rngState = px.rngState;
    f3 totalIncomingLight = splat3(0.0f);

    for (int rayIndex = 0; rayIndex < P.NumRaysPerPixel; rayIndex++)
    {
        PathState ray;
        GenerateCameraRay(P, px, rngState, ray);
        for (int i = 0; i <= P.MaxBounceCount; i++)
        {
            const Hit hit = CalculateRayCollision_ref(P, ray.pos, ray.dir, cnt);
            if (!ShadeSegment(P, hit, ray, rngState)) break;
        }
        totalIncomingLight = totalIncomingLight + ray.totalLight;
    }
    const f3 pixelCol = totalIncomingLight / __int2float_rn(P.NumRaysPerPixel);

    const size_t o = (size_t)idy * P.W + idx;
    WritePixel<true, true>(P, o, pixelCol.x, pixelCol.y, pixelCol.z, moments);
    if (P.countStats) { Counters zero; zero.rays = zero.box = zero.tri = zero.sph = zero.sbox = 0; AddPixelStats(P, o, cnt, zero); }
    FlushCounters(P, cnt);
}

// Kernel 0 over one dispatch: 8 x 8-pixel groups over P's region, or (FORM_LIST) 64-thread blocks over the `count` pixels of `list`,
// between the timing events.  A launch error is left to the caller's cudaGetLastError.
inline cudaError_t mega_launch(CameraForm form, const DevParams& P, unsigned int count, const unsigned int* list, float4* moments,
                               cudaStream_t stream, cudaEvent_t evA, cudaEvent_t evB)
{
    const cudaError_t e = cudaEventRecord(evA, stream);
    if (e != cudaSuccess) return e;
    const dim3 grid((P.limX + 7) / 8, (P.limY + 7) / 8, 1), block(8, 8, 1);
    if (form == FORM_LIST) RT_LAUNCH((count + 63u) / 64u, 64, 0, stream, k_raytrace_mega_list<64>, P, count, list, moments);
    else if (form == FORM_FRAMES) RT_LAUNCH(grid, block, 0, stream, k_raytrace_mega_frames, P);
    else RT_LAUNCH(grid, block, 0, stream, k_raytrace_mega, P);
    return cudaEventRecord(evB, stream);
}

} // namespace rtd
