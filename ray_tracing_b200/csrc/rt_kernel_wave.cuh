// rt_kernel_wave.cuh — kernel variant 1: persistent threads, one path per lane (the default for sphere-only scenes; the
// pooled wavefront kernel, rt_kernel_pool.cuh, is the default when the scene has meshes).
//
// Shape (this implementation's own; the arithmetic per path is the reference's, see rt_device.cuh):
//   * persistent CTAs (a multiple of the SM count) pull pixel jobs from one global counter.  A lane that
//     finishes its pixel is refilled in place: the lanes that need work are found with a warp ballot, ONE
//     atomicAdd per warp reserves a contiguous job range, and the lanes take consecutive jobs by popcount
//     rank (warp-ballot compaction of the free slots).  Jobs are ordered in 8x4-pixel tiles so a freshly
//     filled warp traces a coherent 32-pixel block.
//   * a pixel's samples stay on one lane, in order, because the reference threads ONE rng state through all
//     NumRaysPerPixel samples of a pixel (HL:552,563-579) and sums them in order (HL:578): this keeps
//     results bit-identical while every lane always has a live path segment to intersect (no idle lanes
//     after early path termination, which is what the megakernel wastes).
//   * every loop iteration is one wavefront step for the warp: [refill] -> [generate] -> [intersect] ->
//     [shade]; all live lanes run the intersection phase together.
//   * the top of every BVH (the first `smemPairs` breadth-first NodePair records, contiguous by
//     construction) is staged into shared memory once per CTA by a TMA bulk copy (cp.async.bulk +
//     mbarrier complete_tx); deeper records and triangles are read with 128-bit vector loads from the
//     repacked 64-byte / 48-byte aligned streams.  Spheres are staged in shared memory too.
//   * traversal visits exactly the nodes and triangles the reference visits, in the same order, with the
//     same push-time-only culling (HL:243-283) — so closest hits, tie winners and the box/triangle test
//     counts equal the oracle's.  What is removed is the re-read of a popped node (the stack carries the
//     node's (start,count)) and the push/pop round trip of the near child.
#pragma once
#include <type_traits>
#include "rt_device.cuh"

namespace rtd {

constexpr int WAVE_THREADS = 128;
constexpr int WAVE_MAX_SMEM_SPHERES = 256;
constexpr int WAVE_STACK = 64;

struct WaveSmemHeader
{
    unsigned long long mbar;
    unsigned int pad[14];
};

#ifndef RT_SIMT_EMU      // (the test-only host build, tests/simt, supplies its own versions of these six helpers)
RT_DI uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

RT_DI void mbar_init(uint32_t mbar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(mbar), "r"(count) : "memory"); }
RT_DI void mbar_expect_tx(uint32_t mbar, uint32_t bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(mbar), "r"(bytes) : "memory"); }
RT_DI void tma_bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t mbar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"(dst), "l"(src), "r"(bytes), "r"(mbar) : "memory");
}
RT_DI bool mbar_try_wait(uint32_t mbar, uint32_t parity)
{
    uint32_t ok;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(mbar), "r"(parity) : "memory");
    return ok != 0;
}
RT_DI void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
#endif

struct NodeRef { int start, count; };

// RT_TREELET_PREFETCH (compiled out by default, it was slower; option "treeletPrefetch"): with records laid out as two-level
// treelets — [record of a node, records of its inner children] contiguous, "pairOrder" = 2 — a reference to a treelet's first
// record carries bit 30.  Fetching such a record also asks L1 for the one or two records behind it, i.e. for BOTH possible next
// steps of the descent, before the box tests have decided which one it is: every second level of a descent then finds its
// record in L1 instead of paying another trip to L2 — the dependent-fetch chain that stalls the mesh scenes is halved.
constexpr int TREELET_ROOT_BIT = 0x40000000;

// Fetch one 64-byte pair record: from the shared-memory copy of the tree tops (STAGED instantiations only: the test for it costs
// warp instructions in the plain pooled kernel, for an option that never paid off), or from L2 / HBM.
template <bool STAGED>
RT_DI void LoadPair(const DevParams& P, const float4* __restrict__ smemPairs, int idx, float4& q0, float4& q1, float4& q2, float4& q3)
{
#ifdef RT_TREELET_PREFETCH
    const bool treeletRoot = (idx & TREELET_ROOT_BIT) != 0;
    idx &= ~TREELET_ROOT_BIT;
#endif
    if (STAGED && idx < P.smemPairs)
    {
        const float4* p = smemPairs + (size_t)idx * 4;
        q0 = p[0]; q1 = p[1]; q2 = p[2]; q3 = p[3];
    }
    else
    {
        const float4* p = reinterpret_cast<const float4*>(P.pairs + idx);
        ldg_record64(p, q0, q1, q2, q3);
#if defined(RT_TREELET_PREFETCH) && !defined(RT_SIMT_EMU)
        if (treeletRoot)
        {
            asm volatile("prefetch.global.L1 [%0];" :: "l"(p + 4));      // the records of the inner children (or, for a one-child
            asm volatile("prefetch.global.L1 [%0];" :: "l"(p + 8));      // treelet, the start of the next treelet: harmless)
        }
#endif
    }
}

// HL:234-287 on the repacked streams.  Same visiting order and culling as the reference.  ANY (occlusion queries, rtTraceOcclusion):
// return right after the first triangle that hits closer than rayLength; bestDst < rayLength then says that there was one.
template <bool STATS, bool STAGED, bool ANY = false>
RT_DI void TraverseMesh(const DevParams& P, const float4* __restrict__ smemPairs, f3 pos, f3 dir, f3 invDir, float rayLength,
                        NodeRef root, bool cullBackface,
                        float& bestDst, int& bestTri, float& bestU, float& bestV, float& bestDet, Counters& cnt)
{
    bestDst = rayLength; bestTri = -1;
    NodeRef stack[WAVE_STACK];
    int stackCount = 0;
    NodeRef cur = root;
    for (;;)
    {
        if (cur.count > 0)
        {
            const float4* g = reinterpret_cast<const float4*>(P.triGeom + cur.start);
            for (int i = 0; i < cur.count; i++, g += TRI_GEOM_F4)
            {
                float4 g0, g1, g2;
                ldg_trigeom(g, g0, g1, g2);
                float dst, u, v, det;
                const bool didHit = RayTriangleCore(pos, dir, make_f3(g0.x, g0.y, g0.z), make_f3(g0.w, g1.x, g1.y), make_f3(g1.z, g1.w, g2.x),
                                                    make_f3(g2.y, g2.z, g2.w), cullBackface, dst, u, v, det);
                if (STATS) cnt.tri++;
                if (didHit && dst < bestDst)
                {
                    bestDst = dst; bestTri = cur.start + i; bestU = u; bestV = v; bestDet = det;
                    if (ANY) return;
                }
            }
            if (stackCount == 0) return;
            cur = stack[--stackCount];
        }
        else
        {
            float4 q0, q1, q2, q3;
            LoadPair<STAGED>(P, smemPairs, cur.start, q0, q1, q2, q3);
            const float dstA = RayBoundingBoxDst(pos, invDir, make_f3(q0.x, q0.y, q0.z), make_f3(q0.w, q1.x, q1.y));
            const float dstB = RayBoundingBoxDst(pos, invDir, make_f3(q2.x, q2.y, q2.z), make_f3(q2.w, q3.x, q3.y));
            if (STATS) cnt.box += 2;
            NodeRef a, b;
            a.start = __float_as_int(q1.z); a.count = __float_as_int(q1.w);
            b.start = __float_as_int(q3.z); b.count = __float_as_int(q3.w);
            const bool isNearestA = dstA <= dstB;
            const float dstNear = isNearestA ? dstA : dstB;
            const float dstFar = isNearestA ? dstB : dstA;
            const NodeRef nearRef = isNearestA ? a : b;
            const NodeRef farRef = isNearestA ? b : a;
            // reference: push far, push near, pop (= near).  Equivalent: push far, continue with near.
            if (dstFar < bestDst && stackCount < WAVE_STACK) stack[stackCount++] = farRef;
            if (dstNear < bestDst) cur = nearRef;
            else { if (stackCount == 0) return; cur = stack[--stackCount]; }
        }
    }
}

// A caller-supplied ray (rtTraceRays, rt_kernel_query.cuh).  In: whether its origin lies inside the box of origins the model records
// (modelsExact) and the sphere accelerator (spheresExact) were padded for — only then may the ray skip models, walk the TLAS or use
// the accelerator — and whether back faces count for every model (forceDontCullBack, HL:356).  Out: the winner's kind (RT_HIT_*) and
// its index in Spheres / ModelInfo.  Occlusion queries (ANY) also bring the segment's end, tMax, and get kind != RT_HIT_NONE back when
// something lies closer than it (kind then names the stage that found it; index stays -1).
struct QueryRay { bool modelsExact, spheresExact, noCull; int kind, index; float tMax; };

// HL:335-374 (+ sphere extension) on the repacked streams.  QUERY = rtTraceRays (q != nullptr); the camera kernels leave it false.
// ANY (with QUERY) = rtTraceOcclusion: the same walk with result.dst starting at q->tMax instead of +inf, ended by the first hit.  Before
// that hit the running bound is the constant tMax, so which boxes are entered and which primitives count does not depend on what was
// visited before: the first hit exists exactly when the full walk from tMax finds one.  No position, normal or winner is computed.
template <bool STATS, bool EXT, bool TLAS, bool QUERY = false, bool ANY = false>
RT_DI Hit Intersect(const DevParams& P, const float4* __restrict__ smemPairs, const DevSphere* __restrict__ smemSpheres,
                    f3 rayPos, f3 rayDir, Counters& cnt, QueryRay* q = nullptr)
{
    static_assert(QUERY || !ANY, "occlusion queries are queries");
    Hit result;
    result.dst = inf32(); result.isBackface = false; result.normal = splat3(0.0f); result.pos = splat3(0.0f); result.material = nullptr;
    if constexpr (ANY) result.dst = q->tMax;
    cnt.rays++;
    if constexpr (QUERY) { q->kind = RT_HIT_NONE; q->index = -1; }

    int bestSphere = -1; bool bestInside = false;
    if (EXT && P.sphBvh && (!QUERY || q->spheresExact))
    {
        int idx = 0x7fffffff, flag = 0;
        TraverseSpheres(P, rayPos, rayDir, result.dst, idx, bestInside, flag, cnt, STATS);
        // (queries: the accelerator's tie rule also keeps a "hit" at dst = +inf, which the reference's strict < never takes; such a hit
        // needs a direction so short or long that dot(dir, dir) leaves the float range — camera rays are unit length.  Occlusion
        // queries start from tMax, so the same rule keeps a sphere at exactly dst = tMax: it counts only below tMax.)
        bool keep = idx != 0x7fffffff;
        if constexpr (QUERY) keep = keep && result.dst < (ANY ? q->tMax : inf32());
        if (keep) bestSphere = idx;
    }
    else
    for (int i = 0; i < P.sphereCount; i++)
    {
        float cx, cy, cz, r2;
        if (i < WAVE_MAX_SMEM_SPHERES) { const DevSphere s = smemSpheres[i]; cx = s.cx; cy = s.cy; cz = s.cz; r2 = s.r2; }
        else { const float4 s0 = __ldg(reinterpret_cast<const float4*>(P.spheres + i)); cx = s0.x; cy = s0.y; cz = s0.z; r2 = __ldg(&P.spheres[i].r2); }
        float dst; bool inside;
        if (STATS) cnt.sph++;
        if (RaySphereCore(rayPos, rayDir, make_f3(cx, cy, cz), r2, dst, inside) && dst < result.dst)
        {
            result.dst = dst; bestSphere = i; bestInside = inside;
            if (ANY) break;
        }
    }
    if constexpr (ANY)
        if (bestSphere >= 0) { q->kind = RT_HIT_SPHERE; return result; }
    if (bestSphere >= 0)
    {
        // HL:319-320 for the winner only (position / normal of a sphere hit depend on nothing but the winner)
        f3 centre;
        if (bestSphere < WAVE_MAX_SMEM_SPHERES) { const DevSphere s = smemSpheres[bestSphere]; centre = make_f3(s.cx, s.cy, s.cz); }
        else centre = make_f3(P.spheres[bestSphere].cx, P.spheres[bestSphere].cy, P.spheres[bestSphere].cz);
        result.isBackface = bestInside;
        result.pos = rayPos + rayDir * result.dst;
        result.normal = normalize3(result.pos - centre) * (bestInside ? -1.0f : 1.0f);
        result.material = &P.Spheres[bestSphere].material;
        if constexpr (QUERY) { q->kind = RT_HIT_SPHERE; q->index = bestSphere; }
    }

    const f3 rayInv = rcp3(rayDir);
    // model skipping (the TLAS and the per-model box test) is exact only for origins inside the box the model records were padded for
    bool skipExact = true;
    if constexpr (QUERY) skipExact = q->modelsExact;
    // many-model scenes (<TLAS> kernels only): one walk of the TLAS marks the models this ray can reach at all; the loop below
    // then jumps from marked model to marked model, still in buffer order and still re-testing each against the running result
    unsigned int tlasMask[TLAS ? RT_TLAS_WORDS : 1];
    const bool useTlas = TLAS && !STATS && P.modelSkip && P.tlas && skipExact;
    if (useTlas) TlasCollect(P, rayPos, rayInv, result.dst, tlasMask);
    for (int i = 0; i < P.modelCount; i++)
    {
        if (useTlas) { i = TlasNext(tlasMask, i, P.modelCount); if (i >= P.modelCount) break; }
        const DevModel* m = P.models + i;
        const float4* mr = reinterpret_cast<const float4*>(m);
        // the instrumented build walks every model like the reference (identical test counts); otherwise models the ray cannot
        // reach before its current best hit are skipped — they could not have changed the result
        if (!STATS && P.modelSkip && skipExact && ModelOutOfReach(mr, rayPos, rayInv, result.dst)) continue;
        float w2l[12];
        {
            const float4 r0 = __ldg(mr), r1 = __ldg(mr + 1), r2 = __ldg(mr + 2);
            w2l[0] = r0.x; w2l[1] = r0.y; w2l[2] = r0.z; w2l[3] = r0.w;
            w2l[4] = r1.x; w2l[5] = r1.y; w2l[6] = r1.z; w2l[7] = r1.w;
            w2l[8] = r2.x; w2l[9] = r2.y; w2l[10] = r2.z; w2l[11] = r2.w;
        }
        const int4 meta = __ldg(reinterpret_cast<const int4*>(mr + 6));     // rootStart, rootCount, cullBackface, matIndex
        const f3 localPos = mul_rm(w2l, rayPos, 1.0f);
        const f3 localDir = mul_rm(w2l, rayDir, 0.0f);
        const f3 invDir = rcp3(localDir);
        NodeRef root; root.start = meta.x; root.count = meta.y;
        bool cullBackface = meta.z != 0;
        if constexpr (QUERY) cullBackface = cullBackface && !q->noCull;
        float dst, u, v, det; int tri;
        TraverseMesh<STATS, EXT, ANY>(P, smemPairs, localPos, localDir, invDir, result.dst, root, cullBackface, dst, tri, u, v, det, cnt);
        if constexpr (ANY)
            if (dst < result.dst) { q->kind = RT_HIT_MODEL; return result; }
        if (dst < result.dst)
        {
            const float4* nq = reinterpret_cast<const float4*>(P.triNormals + tri);
            const float4 n0 = ldg_tri(nq), n1 = ldg_tri(nq + 1), n2 = ldg_tri(nq + 2);
            const f3 n = TriangleSmoothNormal(make_f3(n0.x, n0.y, n0.z), make_f3(n0.w, n1.x, n1.y), make_f3(n1.z, n1.w, n2.x), u, v, det);
            float l2w[12];
            {
                const float4 r0 = __ldg(mr + 3), r1 = __ldg(mr + 4), r2 = __ldg(mr + 5);
                l2w[0] = r0.x; l2w[1] = r0.y; l2w[2] = r0.z; l2w[3] = r0.w;
                l2w[4] = r1.x; l2w[5] = r1.y; l2w[6] = r1.z; l2w[7] = r1.w;
                l2w[8] = r2.x; l2w[9] = r2.y; l2w[10] = r2.z; l2w[11] = r2.w;
            }
            result.isBackface = det < 0.0f;
            result.dst = dst;
            result.normal = normalize3(mul_rm(l2w, n, 0.0f));
            result.pos = rayPos + rayDir * dst;
            result.material = &P.ModelInfo[meta.w].material;
            if constexpr (QUERY) { q->kind = RT_HIT_MODEL; q->index = meta.w; }
        }
    }
    return result;
}

#if defined(RT_SIMT_PROFILE) && defined(RT_SIMT_EMU)
#define WAVE_PROF(i, v) do { if ((threadIdx.x & 31u) == 0) simt::prof_add(i, (unsigned long long)(v)); } while (0)
#define WAVE_PROF_LANES(i, pred) do { const unsigned m_ = __ballot_sync(0xffffffffu, (pred)); if ((threadIdx.x & 31u) == 0) { simt::prof_add(i, (unsigned long long)__popc(m_)); simt::prof_add((i) + 20, m_ ? 1u : 0u); } } while (0)
#define WAVE_PROF_LANE(i, pred) do { if (pred) simt::prof_add(i, 1); } while (0)
#else
#define WAVE_PROF(i, v) do { } while (0)
#define WAVE_PROF_LANES(i, pred) do { } while (0)
#define WAVE_PROF_LANE(i, pred) do { } while (0)
#endif
#ifndef RT_WAVE_MINBLOCKS
#define RT_WAVE_MINBLOCKS 6      // <= 85 registers: 24 warps per SM (faster than 16 warps on config 2)
#endif

// The end of a persistent kernel: the warp's counters summed, then added by lane 0 into P.counters (rays; with STATS the others too)
template <bool STATS>
RT_DI void FlushCounters(const DevParams& P, const Counters& cnt)
{
    const unsigned int lane = threadIdx.x & 31u;
    unsigned int r = __reduce_add_sync(0xffffffffu, cnt.rays);
    if (lane == 0) atomicAdd(P.counters + 0, (unsigned long long)r);
    if (STATS)
    {
        const unsigned int b = __reduce_add_sync(0xffffffffu, cnt.box), t = __reduce_add_sync(0xffffffffu, cnt.tri), s = __reduce_add_sync(0xffffffffu, cnt.sph), sb = __reduce_add_sync(0xffffffffu, cnt.sbox);
        if (lane == 0) { atomicAdd(P.counters + 1, (unsigned long long)b); atomicAdd(P.counters + 2, (unsigned long long)t); atomicAdd(P.counters + 3, (unsigned long long)s); atomicAdd(P.counters + 4, (unsigned long long)sb); }
    }
}

// The kernel body.  TLAS = the many-model instantiation (its own kernel, k_raytrace_wave_tlas, so that the kernels measured in
// round 1 keep their code: the TLAS walk and its mask exist only there).  FRAMES = the batch instantiations of rtDispatchFrames (never
// CHUNKED): a lane keeps its pixel for frames Frame .. Frame + P.frames - 1, writing and accumulating each frame when its samples end.
// LIST = the list-driven instantiations of rtDispatchAdaptive (never CHUNKED): job j < totalJobs is the pixel P.pixelList[j]
// ((y << 16) | x), and the write also updates the pixel's moments in P.adaptiveMoments.  (Both come in parameter slots of their own
// (rt_device.cuh), not as arguments: with two more arguments here the k_raytrace_wave_frames kernels compiled to other code.)
template <bool STATS, bool EXT, bool TLAS, bool CHUNKED, bool FRAMES = false, bool LIST = false>
RT_DI void wave_body(const DevParams& P, const unsigned int totalJobs, const unsigned int tilesX, const unsigned int ownedRows)
{
    RT_DYNAMIC_SMEM(smemRaw);
    WaveSmemHeader* hdr = reinterpret_cast<WaveSmemHeader*>(smemRaw);
    float4* smemPairs = reinterpret_cast<float4*>(smemRaw + sizeof(WaveSmemHeader));
    DevSphere* smemSpheres = reinterpret_cast<DevSphere*>(smemRaw + sizeof(WaveSmemHeader) + (size_t)P.smemPairs * sizeof(NodePair));

    // ---- stage the tree tops (TMA bulk copy) and the spheres ------------------------------------------------------------
    const uint32_t mbar = smem_u32(&hdr->mbar);
    if (threadIdx.x == 0)
    {
        mbar_init(mbar, 1);
        mbar_fence_init();
    }
    __syncthreads();
    if (P.smemPairs > 0 && threadIdx.x == 0)
    {
        const uint32_t bytes = (uint32_t)P.smemPairs * (uint32_t)sizeof(NodePair);
        mbar_expect_tx(mbar, bytes);
        // chunks of <= 32 KB; all complete on the same mbarrier phase
        uint32_t off = 0;
        while (off < bytes)
        {
            const uint32_t n = (bytes - off) < 32768u ? (bytes - off) : 32768u;
            tma_bulk_g2s(smem_u32(smemPairs) + off, reinterpret_cast<const unsigned char*>(P.pairs) + off, n, mbar);
            off += n;
        }
    }
    {
        const int nS = P.sphereCount < WAVE_MAX_SMEM_SPHERES ? P.sphereCount : WAVE_MAX_SMEM_SPHERES;
        for (int i = threadIdx.x; i < nS; i += WAVE_THREADS) smemSpheres[i] = P.spheres[i];
    }
    if (P.smemPairs > 0) { while (!mbar_try_wait(mbar, 0)) { } }
    __syncthreads();

    // ---- persistent wavefront loop ------------------------------------------------------------------------------------------
    const unsigned int lane = threadIdx.x & 31u;
    const unsigned int laneMaskLt = (1u << lane) - 1u;
    Counters cnt; cnt.rays = cnt.box = cnt.tri = cnt.sph = cnt.sbox = 0;
    Counters pixelStart = cnt;       // STATS: the counters when this lane took its pixel (or chunk); the difference goes to PixelStats

    bool exhausted = false;          // no more jobs for this lane
    bool havePixel = false;
    bool pathActive = false;
    PixelSetup px; px.camOrigin = px.focusPoint = px.camRight = px.camUp = splat3(0.0f); px.rngState = 0;
    uint32_t rngState = 0;
    f3 totalIncomingLight = splat3(0.0f);
    int sample = 0, bounce = 0;
    size_t pixelOffset = 0;
    PathState ray; ray.pos = ray.dir = ray.transmittance = ray.totalLight = splat3(0.0f);
    // Sample chunks (small tiles, P.chunks > 1).  A pixel's samples are one sequential chain, but the chain may change lanes between
    // samples: job j is chunk j / totalJobs of pixel job j % totalJobs — samples [c R / C, (c + 1) R / C) — so every chunk 0 is handed
    // out before any chunk 1, and the lane that finishes a chunk leaves the RNG state and the running sum for the lane that takes the
    // next one.  With 2.3 pixels per lane (8 GPUs, 1080p) the last round of whole pixels runs on a quarter-full machine; in chunks of
    // an eighth the same work is 18.2 rounds.  A lane whose predecessor chunk is still running holds its job and idles (it keeps
    // taking part in the warp's collectives); the predecessor was handed out a whole pass over the tile earlier, so that is rare.
    // (CHUNKED is a template parameter: with the hand-off code merely present the whole-pixel kernel ran slower on config 2)
    const int chunks = CHUNKED && P.chunks > 1 && totalJobs > 0u ? P.chunks : 1;
    const unsigned int chunkJobs = totalJobs * (unsigned int)chunks;
    int chunk = 0, sampleEnd = P.NumRaysPerPixel; unsigned int pixJob = 0; bool waiting = false;
    static_assert(!(FRAMES && CHUNKED), "a batch of frames runs whole pixels");
    static_assert(!(LIST && (CHUNKED || FRAMES)), "a pixel list runs whole pixels, one frame");
    unsigned int frame = 0;          // FRAMES: frame of the batch the lane's pixel is in
    (void)frame;

    for (;;)
    {
        // [refill] lanes without a pixel take the next jobs (ballot + one atomic per warp)
        const bool need = !havePixel && !exhausted;
        const unsigned int needMask = __ballot_sync(0xffffffffu, need);
        if (needMask)
        {
            unsigned int base = 0;
            const int leader = __ffs(needMask) - 1;
            if ((int)lane == leader) base = atomicAdd(P.workCounter, (unsigned int)__popc(needMask));
            base = __shfl_sync(0xffffffffu, base, leader);
            if (need)
            {
                const unsigned int jobAll = base + (unsigned int)__popc(needMask & laneMaskLt);
                if (jobAll >= chunkJobs) exhausted = true;
                else if constexpr (LIST)
                {
                    const unsigned int xy = P.pixelList[jobAll];
                    px = SetupPixel(P, xy & 0xffffu, xy >> 16);
                    rngState = px.rngState;
                    totalIncomingLight = splat3(0.0f);
                    sample = 0; sampleEnd = P.NumRaysPerPixel;
                    pixelOffset = (size_t)(xy >> 16) * P.W + (xy & 0xffffu);
                    havePixel = true; pathActive = false;
                    if (STATS) pixelStart = cnt;
                }
                else
                {
                    const unsigned int job = CHUNKED && chunks > 1 ? jobAll % totalJobs : jobAll;
                    const unsigned int tile = job >> 5, l = job & 31u;
                    const unsigned int x = (tile % tilesX) * 8u + (l & 7u);
                    const unsigned int r = (tile / tilesX) * 4u + (l >> 3);
                    if (x < P.limX && r < ownedRows)
                    {
                        const unsigned int y = ((r / (unsigned int)P.bandRows) * (unsigned int)P.tileWorld + (unsigned int)P.tileRank) * (unsigned int)P.bandRows
                                             + (r % (unsigned int)P.bandRows);
                        px = SetupPixel(P, x, y);
                        rngState = px.rngState;
                        totalIncomingLight = splat3(0.0f);
                        sample = 0; sampleEnd = P.NumRaysPerPixel;
                        pixelOffset = (size_t)y * P.W + x;
                        havePixel = true; pathActive = false;
                        if constexpr (FRAMES) frame = 0;
                        if (STATS) pixelStart = cnt;
                        if (CHUNKED && chunks > 1)
                        {
                            chunk = (int)(jobAll / totalJobs); pixJob = job;
                            sample = (int)(((long long)chunk * P.NumRaysPerPixel) / chunks);
                            sampleEnd = (int)(((long long)(chunk + 1) * P.NumRaysPerPixel) / chunks);
                            waiting = chunk > 0;          // the state at `sample` comes from the lane that ran the chunk before
                        }
                    }
                }
            }
        }
        if (__ballot_sync(0xffffffffu, havePixel) == 0u)
        {
            if (__ballot_sync(0xffffffffu, !exhausted) == 0u) break;
            continue;
        }
        if (CHUNKED && chunks > 1 && havePixel && waiting)
        {
            // four self-validating words: {tag, value} with tag = this dispatch's serial and the number of chunks completed
            const volatile unsigned long long* h = reinterpret_cast<const volatile unsigned long long*>(P.handoff + 4ull * pixJob);
            const unsigned long long w0 = h[0], w1 = h[1], w2 = h[2], w3 = h[3];
            const unsigned int tag = ((unsigned int)P.chunkSerial << 8) | (unsigned int)chunk;
            if ((unsigned int)(w0 >> 32) == tag && (unsigned int)(w1 >> 32) == tag && (unsigned int)(w2 >> 32) == tag && (unsigned int)(w3 >> 32) == tag)
            {
                rngState = (uint32_t)w0;
                totalIncomingLight = make_f3(__uint_as_float((unsigned int)w1), __uint_as_float((unsigned int)w2), __uint_as_float((unsigned int)w3));
                waiting = false;
            }
        }

        // (interpreter-only schedule profile, see rt_kernel_pool.cuh / tools/simt_schedule_profile.py)
        WAVE_PROF(20, 1); WAVE_PROF_LANES(21, havePixel && !pathActive && sample < P.NumRaysPerPixel); WAVE_PROF_LANES(22, pathActive || (havePixel && sample < P.NumRaysPerPixel));
        // [generate] start the pixel's next sample
        if (havePixel && !(CHUNKED && waiting) && !pathActive && sample < (CHUNKED ? sampleEnd : P.NumRaysPerPixel))
        {
            GenerateCameraRay(P, px, rngState, ray);
            bounce = 0;
            pathActive = true;
        }

        // [intersect] + [shade]
        if (pathActive)
        {
            const Hit hit = Intersect<STATS, EXT, TLAS>(P, smemPairs, smemSpheres, ray.pos, ray.dir, cnt);
            WAVE_PROF_LANE(23, !(hit.dst < inf32())); WAVE_PROF_LANE(24, hit.dst < inf32() && hit.material->flag == RT_MATERIAL_GLASS);
            const bool cont = ShadeSegment(P, hit, ray, rngState);
            bounce++;
            if (!cont || bounce > P.MaxBounceCount)
            {
                totalIncomingLight = totalIncomingLight + ray.totalLight;        // HL:578
                sample++;
                pathActive = false;
            }
        }

        // [write] pixel finished (RC:18-23) — or, in chunks, this part of its chain: leave the state for the next chunk's lane
        if (havePixel && !(CHUNKED && waiting) && !pathActive && sample >= (CHUNKED ? sampleEnd : P.NumRaysPerPixel))
        {
            if (!CHUNKED || sampleEnd >= P.NumRaysPerPixel)
            {
                const f3 pixelCol = totalIncomingLight / __int2float_rn(P.NumRaysPerPixel);
                if constexpr (LIST) WritePixel<EXT, true>(P, pixelOffset, pixelCol.x, pixelCol.y, pixelCol.z, P.adaptiveMoments);
                else WritePixel<EXT>(P, pixelOffset, pixelCol.x, pixelCol.y, pixelCol.z);
            }
            else
            {
                volatile unsigned long long* h = reinterpret_cast<volatile unsigned long long*>(P.handoff + 4ull * pixJob);
                const unsigned long long tag = (unsigned long long)(((unsigned int)P.chunkSerial << 8) | (unsigned int)(chunk + 1)) << 32;
                h[0] = tag | rngState; h[1] = tag | __float_as_uint(totalIncomingLight.x);
                h[2] = tag | __float_as_uint(totalIncomingLight.y); h[3] = tag | __float_as_uint(totalIncomingLight.z);
            }
            if constexpr (FRAMES)
            {
                if (++frame < (unsigned int)P.frames)
                {
                    // the pixel's next frame: reseeded, a fresh sum, the same lane (frames accumulate in order)
                    rngState = FrameSeed(px.rngState, frame);
                    totalIncomingLight = splat3(0.0f);
                    sample = 0;
                }
                else
                {
                    if (STATS) AddPixelStats(P, pixelOffset, cnt, pixelStart);      // all the pixel's frames
                    havePixel = false;
                }
            }
            else
            {
                if (STATS) AddPixelStats(P, pixelOffset, cnt, pixelStart);      // this lane's share: the whole pixel, or this chunk of it
                havePixel = false;
            }
        }
    }

    FlushCounters<STATS>(P, cnt);
}

template <bool STATS, bool EXT, bool CHUNKED = false>
__global__ void __launch_bounds__(WAVE_THREADS, RT_WAVE_MINBLOCKS) k_raytrace_wave(const __grid_constant__ DevParams P, const unsigned int totalJobs,
                                                               const unsigned int tilesX, const unsigned int ownedRows)
{
    wave_body<STATS, EXT, false, CHUNKED>(P, totalJobs, tilesX, ownedRows);
}

// many-model scenes: every extension + the TLAS walk (never instrumented: the counting build walks every model like the reference)
__global__ void __launch_bounds__(WAVE_THREADS, RT_WAVE_MINBLOCKS) k_raytrace_wave_tlas(const __grid_constant__ DevParams P, const unsigned int totalJobs,
                                                                    const unsigned int tilesX, const unsigned int ownedRows)
{
    wave_body<false, true, true, true>(P, totalJobs, tilesX, ownedRows);      // (the many-model kernel carries the chunk hand-off: it is never the Cornell-box kernel)
}

// rtDispatchFrames: P.frames frames of every pixel in one launch (kernels of their own, so that the kernels above keep their code)
template <bool STATS, bool EXT>
__global__ void __launch_bounds__(WAVE_THREADS, RT_WAVE_MINBLOCKS) k_raytrace_wave_frames(const __grid_constant__ DevParams P, const unsigned int totalJobs,
                                                                      const unsigned int tilesX, const unsigned int ownedRows)
{
    wave_body<STATS, EXT, false, false, true>(P, totalJobs, tilesX, ownedRows);
}

__global__ void __launch_bounds__(WAVE_THREADS, RT_WAVE_MINBLOCKS) k_raytrace_wave_tlas_frames(const __grid_constant__ DevParams P, const unsigned int totalJobs,
                                                                           const unsigned int tilesX, const unsigned int ownedRows)
{
    wave_body<false, true, true, false, true>(P, totalJobs, tilesX, ownedRows);
}

// rtDispatchAdaptive: the selection's pixel list (P.pixelList, totalJobs = its length), one frame per pixel (kernels of their own, so
// that the kernels above keep their code; TLAS = the many-model form, <false, true, true>).  Templates, instantiated where
// wave_kernel names them: a plain kernel defined here changed the register numbering of the k_raytrace_wave_frames kernels.
template <bool STATS, bool EXT, bool TLAS>
__global__ void __launch_bounds__(WAVE_THREADS, RT_WAVE_MINBLOCKS) k_raytrace_wave_list(const __grid_constant__ DevParams P, const unsigned int totalJobs)
{
    wave_body<STATS, EXT, TLAS, false, false, true>(P, totalJobs, 0u, 0u);
}

// "gridFit": a pixel's samples cannot be split (one RNG chain), so a persistent lane works through whole pixels.  When the image
// gives every lane only a few (8 GPUs, config 2: 2.3 pixels per lane) the last round runs with mostly empty warps.  With the
// option on, the grid is shrunk so that pixels / lanes is just under a whole number k = ceil(pixels / maxLanes): the same k
// rounds, every one of them with full warps, on fewer resident warps.  Scheduling only; off by default (slower than the full grid on whole images).
inline unsigned int fit_persistent_grid(int enabled, unsigned int grid, unsigned int lanesPerCta, unsigned int totalJobs)
{
    if (!enabled || grid == 0 || totalJobs == 0) return grid;
    const unsigned long long lanes = (unsigned long long)grid * lanesPerCta;
    const unsigned long long k = (totalJobs + lanes - 1) / lanes;                    // rounds at full size
    const unsigned long long fitLanes = (totalJobs + k - 1) / k;                     // lanes that keep k rounds full
    const unsigned long long fit = (fitLanes + lanesPerCta - 1) / lanesPerCta;
    return fit < grid ? (unsigned int)(fit ? fit : 1) : grid;
}

// Sample chunks per pixel for kernel 1 (wave_body): automatic = mesh scenes on tiles where whole pixels quantise badly — more than one and
// fewer than four pixels per resident lane — and then about eight chunk-rounds per launch.  forced > 0 overrides (tests); always <= samples.
inline int wave_chunks(int forced, int numSMs, unsigned long long pixels, int samples, int modelCount)
{
    if (samples < 2) return 1;
    int c = 1;
    if (forced > 0) c = forced;
    else if (forced < 0 && modelCount > 0)
    {
        // on a mesh scene with about two pixels per lane, chunked pixels beat whole ones (4 - 8 chunks best); on the sphere-only Cornell box
        // a sample is too cheap for the hand-off, so sphere-only scenes keep whole pixels.
        const double lanes = (double)numSMs * RT_WAVE_MINBLOCKS * WAVE_THREADS;
        const double perLane = (double)pixels / lanes;
        if (perLane > 1.0 && perLane < 4.0) { c = (int)(8.0 / perLane + 0.999); if (c > 8) c = 8; }
    }
    if (c > samples) c = samples;
    return c < 1 ? 1 : c;
}

// ---- choosing and launching a persistent kernel (kernels 1 and 2 here and in rt_kernel_pool.cuh, the query family in rt_kernel_query.cuh)

// The instantiation <STATS, EXT, TLAS> of a persistent kernel, chosen here and nowhere else: the counting build walks every model like the
// reference; the TLAS kernel when the scene has a TLAS and skipping is on; otherwise the extension family when an extension is active —
// peer stores, the sphere accelerator, "extInstantiation" or staged tree tops (the plain instantiation carries none of them).  The query
// family's launches come here with nPeers = smemPairs = 0 (queryParams), so for them ext is sphBvh || forceExt.  `launch` is called with
// three std::integral_constant<bool, ...>.
template <class Launch>
inline cudaError_t with_persistent_kernel(const DevParams& P, Launch launch)
{
    std::true_type Y;
    std::false_type N;
    const bool ext = P.nPeers > 0 || P.sphBvh != 0 || P.forceExt != 0 || P.smemPairs > 0;
    if (P.countStats) return ext ? launch(Y, Y, N) : launch(Y, N, N);
    if (P.tlas && P.modelSkip) return launch(N, Y, Y);
    return ext ? launch(N, Y, N) : launch(N, N, N);
}

// A camera kernel's variant: `launch` is called with the form and with_persistent_kernel's <STATS, EXT, TLAS>, all std::integral_constants
template <class Launch>
inline cudaError_t with_camera_kernel(CameraForm form, const DevParams& P, Launch launch)
{
    return with_persistent_kernel(P, [&](auto S, auto X, auto T) {
        if (form == FORM_LIST) return launch(std::integral_constant<CameraForm, FORM_LIST>(), S, X, T);
        if (form == FORM_FRAMES) return launch(std::integral_constant<CameraForm, FORM_FRAMES>(), S, X, T);
        return launch(std::integral_constant<CameraForm, FORM_PLAIN>(), S, X, T);
    });
}

// Every variant with_camera_kernel can choose (most of them more than once), for the *_configure functions: the rule is run on every
// combination of its inputs, so that no kernel a launch can pick is left without its shared-memory limit
template <class Launch>
inline cudaError_t for_each_camera_kernel(Launch launch)
{
    DevParams P = {};
    for (int in = 0; in < 24; in++)
    {
        P.countStats = in & 1; P.tlas = P.modelSkip = (in >> 1) & 1; P.forceExt = (in >> 2) & 1;
        const cudaError_t e = with_camera_kernel((CameraForm)(in >> 3), P, launch);
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

// The rows among the first limY that the bands of bandRows rows, dealt round-robin to tileWorld ranks, give to `rank`
inline unsigned int owned_rows(unsigned int limY, int bandRows, int tileWorld, int rank)
{
    unsigned int rows = 0;
    for (unsigned int y0 = 0, b = 0; y0 < limY; y0 += (unsigned int)bandRows, b++)
        if ((int)(b % (unsigned int)tileWorld) == rank) rows += limY - y0 < (unsigned int)bandRows ? limY - y0 : (unsigned int)bandRows;
    return rows;
}

// The camera kernels' jobs over limX x rows pixels: 32 per 8 x 4-pixel tile, tiles cut off at the region's edges included
inline unsigned long long tile_jobs(unsigned int limX, unsigned int rows)
{
    return (unsigned long long)((limX + 7u) / 8u) * ((rows + 3u) / 4u) * 32ull;
}

// The jobs of a launch of kernel 1 or 2: the `listCount` pixels of a list (FORM_LIST), or the tiles of P's region in this rank's bands.
// False when the tiles' jobs would not fit the 32-bit work counter, which every resident lane draws from once more after the last job.
struct CameraJobs { unsigned int total = 0, tilesX = 0, ownedRows = 0; };
inline bool camera_jobs(CameraForm form, const DevParams& P, unsigned int listCount, CameraJobs& J)
{
    if (form == FORM_LIST) { J.total = listCount; return true; }
    J.ownedRows = owned_rows(P.limY, P.bandRows, P.tileWorld, P.tileRank);
    J.tilesX = (P.limX + 7u) / 8u;
    const unsigned long long jobs = tile_jobs(P.limX, J.ownedRows);
    if (jobs >= 0xffff0000ull) return false;
    J.total = (unsigned int)jobs;
    return true;
}

// The grid of a persistent launch of kernel 1 or of the query family: as many CTAs as fit on every SM (a multiple of the SM count), but
// no more than warpsNeeded warps fill (at least one)
template <class Kernel>
inline cudaError_t persistent_grid(Kernel kernel, size_t smemBytes, unsigned int warpsNeeded, int numSMs, unsigned int& grid)
{
    int ctasPerSM = 0;
    const cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctasPerSM, kernel, WAVE_THREADS, smemBytes);
    if (e != cudaSuccess) return e;
    if (ctasPerSM < 1) return cudaErrorInvalidConfiguration;
    grid = (unsigned int)(numSMs * ctasPerSM);
    const unsigned int ctasNeeded = (warpsNeeded + (WAVE_THREADS / 32) - 1) / (WAVE_THREADS / 32);
    if (grid > ctasNeeded) grid = ctasNeeded ? ctasNeeded : 1;
    return cudaSuccess;
}

// Kernel 1's table: the __global__ of form F and <STATS, EXT, TLAS>.  CHUNKED: sample chunks (P.chunks > 1, the plain form only), which
// live in instantiations of their own, <STATS, true, false, CHUNKED>; the TLAS kernel carries the hand-off itself.
template <CameraForm F, bool S, bool X, bool T, bool CHUNKED>
inline auto wave_kernel()
{
    if constexpr (F == FORM_LIST) return k_raytrace_wave_list<S, X, T>;
    else if constexpr (F == FORM_FRAMES && T) return k_raytrace_wave_tlas_frames;
    else if constexpr (F == FORM_FRAMES) return k_raytrace_wave_frames<S, X>;
    else if constexpr (T) return k_raytrace_wave_tlas;
    else if constexpr (CHUNKED) return k_raytrace_wave<S, true, true>;
    else return k_raytrace_wave<S, X>;
}

inline cudaError_t wave_configure()
{
    return for_each_camera_kernel([](auto F, auto S, auto X, auto T) {
        const cudaError_t e = cudaFuncSetAttribute(wave_kernel<F, S, X, T, false>(), cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024 - 1024);
        return e != cudaSuccess ? e : cudaFuncSetAttribute(wave_kernel<F, S, X, T, true>(), cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024 - 1024);
    });
}

// Kernel 1 over one dispatch in `form`; FORM_LIST: over the `count` pixels of `list`, whose moments its writes update (both reach the
// kernel in P's parameter slots)
inline cudaError_t wave_launch(CameraForm form, DevParams P, int numSMs, unsigned int count, const unsigned int* list, float4* moments,
                               cudaStream_t stream, cudaEvent_t evA, cudaEvent_t evB)
{
    CameraJobs J;
    if (!camera_jobs(form, P, count, J)) return cudaErrorInvalidValue;
    if (form == FORM_LIST) { P.pixelList = list; P.adaptiveMoments = moments; }       // (the hand-off's and the cold pool's slots: unused here)
    const size_t smemBytes = sizeof(WaveSmemHeader) + (size_t)P.smemPairs * sizeof(NodePair) + (size_t)WAVE_MAX_SMEM_SPHERES * sizeof(DevSphere);
    return with_camera_kernel(form, P, [&](auto F, auto S, auto X, auto T) -> cudaError_t {
        const auto kernel = P.chunks > 1 ? wave_kernel<F, S, X, T, true>() : wave_kernel<F, S, X, T, false>();
        unsigned int grid = 0;
        cudaError_t e = persistent_grid(kernel, smemBytes, (J.total + 31u) / 32u, numSMs, grid);      // (whole pixels: a chunk of a pixel cannot run beside the chunk before it)
        if (e != cudaSuccess) return e;
        grid = fit_persistent_grid(P.gridFit, grid, WAVE_THREADS, J.total);
        if ((e = cudaMemsetAsync(P.workCounter, 0, sizeof(unsigned int), stream)) != cudaSuccess) return e;
        if ((e = cudaEventRecord(evA, stream)) != cudaSuccess) return e;
        if constexpr (F == FORM_LIST) RT_LAUNCH(grid, WAVE_THREADS, smemBytes, stream, kernel, P, J.total);
        else RT_LAUNCH(grid, WAVE_THREADS, smemBytes, stream, kernel, P, J.total, J.tilesX, J.ownedRows);
        if ((e = cudaGetLastError()) != cudaSuccess) return e;
        return cudaEventRecord(evB, stream);
    });
}

} // namespace rtd
