// rt_kernel_pool.cuh — kernel variant 2: persistent-thread WAVEFRONT path tracer with per-warp path pools.
//
// Why: in variant 1 a lane owns one path, so during BVH traversal the warp waits for its longest ray — on the earlier
// GPU only a few of 32 lanes were active in the node loop on the mesh scene.  Here every warp owns a pool of M paths
// (M = 1..3 x 32) that lives in shared memory, and alternates two phases, each of which keeps the lanes full:
//
//   SHADE phase   the paths that came back from tracing are SORTED by what their hit needs (miss / opaque / glass)
//                 with ballot+popcount compaction into an index list, then shaded 32 at a time — each batch runs one
//                 material branch.  Finished pixels are written out; their slots are refilled from the global pixel
//                 queue (ballot compaction of free slots, ONE atomicAdd per warp per refill); camera rays for new
//                 samples are generated in compacted batches.
//   TRACE phase   the warp's M rays are consumed through a warp-local queue: a lane that finishes its ray flips its slot's
//                 state and immediately takes the next ray (ballot-ranked pop from a warp-uniform counter, no atomics); the
//                 slot's hit record is written whenever a test improves the result, so the lane keeps only the closest distance,
//                 the hit kind and the model-local ray in registers, and re-reads the world ray from the slot when it changes
//                 models.  Every lane is a small state machine (inner node / leaf primitive / next model); each
//                 iteration one warp reduction counts the lanes per state and the warp executes the step kind most
//                 lanes wait for (two inner-node visits per census).  When the queue is empty and at most `tailLanes`
//                 lanes still trace, the phase ends and those rays stay in flight, in their lanes, across the next
//                 shade phase (slot state PS_FLIGHT) — long rays never hold the warp back.
//
// A pool slot is a PIXEL: its NumRaysPerPixel samples run one after the other on the slot, threading the pixel's
// single rng state and summing in order (HL:552,563-579) — the reference's per-pixel arithmetic order is untouched,
// and traversal visits the reference's nodes and triangles in the reference's order (HL:243-283), so the output is
// bit-identical to the oracle's and the box / triangle test counts are too.
//
// NodePair / TriGeom records are fetched with 128-bit loads from the repacked aligned streams; small Spheres buffers are
// staged in shared memory.  The first `smemPairs` pair records of every tree CAN be staged into shared memory once per CTA
// by TMA bulk copies (cp.async.bulk + mbarrier) — implemented, parity-tested, and off by default because it measured
// neutral-to-negative (L1 already holds the hot tree tops; DESIGN.md §5).  Large Spheres buffers go through the padded-box
// accelerator as "model -1" of the same state machine (EXT instantiation).
#pragma once
#include "rt_kernel_wave.cuh"

namespace rtd {

#ifndef RT_INNER_REPEAT
#define RT_INNER_REPEAT 2      // 2 visits per census beat 1 on the mesh scenes, 3 was no better
#endif
#ifndef RT_POOL_WARPS
#define RT_POOL_WARPS 24      // one CTA of 24 warps per SM (80 registers): on the H100 faster than 20 warps (95 registers) and 16 (126) on the mesh scenes, DESIGN §5
#endif
// Compile-time switches (each is bit-exact on the SIMT interpreter build; the winners of the round-2 A/B runs are on by default, rt_devmath.cuh,
// the rest stays available for A/B runs):
//   RT_STACK_TOP_REG   the top entry of the traversal stack lives in two registers: a pop hands it over at once and issues
//                      the local-memory load of the entry below, which is only needed at the next pop / push — the pop's
//                      load latency (a large share of the stall samples on the 1M-triangle scene) overlaps
//                      the fetch and box tests of the popped node instead of preceding them
//   RT_CACHE_RAYINV    1 / world ray direction (model skipping) computed once per ray instead of at every model step
//   RT_LEAF_REPEAT=n   n leaf primitives per census (like RT_INNER_REPEAT for inner nodes)
//   (RT_PREFETCH_CUR: below)
//   RT_PREFETCH_NEXT_PAIR   L1 prefetch of the record after the one being fetched (meant for "pairOrder" = 1, where that is child A's)
//   RT_SMEM_STACK=N    (N a power of two) the top N entries of every lane's traversal stack live in shared memory — a ring, entry-major
//                      across the warp (entry i = 32 lanes x one int2), so a push or pop is one conflict-free 8-byte access instead of a
//                      local-memory access that touches up to 32 different lines (divergent stack depths); deeper entries spill to the
//                      local array, oldest first.  Costs N * 6 KB of shared memory per CTA (taken from L1).
// RING = entries of the shared-memory ring of a kernel instantiation: RT_SMEM_STACK, except for the 96-slot pools, whose 223 KB of path
// state leave no room for it (they keep the whole stack in local memory).
#if defined(RT_SMEM_STACK) && !defined(RT_STACK_TOP_REG)
static_assert((RT_SMEM_STACK & (RT_SMEM_STACK - 1)) == 0 && RT_SMEM_STACK >= 2, "RT_SMEM_STACK must be a power of two");
#ifdef RT_POOL_COLD_GLOBAL
template <int M> struct PoolRing { static constexpr int N = RT_SMEM_STACK; };
#else
template <int M> struct PoolRing { static constexpr int N = M >= 96 ? 0 : RT_SMEM_STACK; };
#endif
#else
template <int M> struct PoolRing { static constexpr int N = 0; };
#endif
#if defined(RT_SMEM_STACK) && !defined(RT_STACK_TOP_REG)
#define RT_RING_DEFAULT RT_SMEM_STACK
#else
#define RT_RING_DEFAULT 0
#endif
#if defined(RT_STACK_TOP_REG)
#define RT_PUSH(x) do { if (stackCount > 0) stack[stackCount - 1] = stackTop; stackTop = (x); stackCount++; } while (0)
#define RT_POP(dst) do { (dst) = stackTop; --stackCount; if (stackCount > 0) stackTop = stack[stackCount - 1]; } while (0)
#else
// entries [stackSpilled, stackCount) are in the ring at index (i & (RING - 1)); entries [0, stackSpilled) in the local array.
// A ring entry is one int2 (start, count) per lane: entry i of the warp is 32 x 8 bytes, one conflict-free 64-bit access per push / pop.
// `ringLane` (this lane's word of entry 0) is computed once per kernel, so an access is that base plus (i & (RING - 1)) * 256 bytes.
// (RT_PROF 28 / 29 of the profile build count spills of the ring's oldest entry and pops that reload an entry from the local array;
// 30 the reloads of the inner step's branchless pop among them.)
#define RT_RING(i) ringLane[((i) & (RING - 1)) * 32]
#define RT_PUSH(x) do { if constexpr (RING > 0) { \
                            if (stackCount - stackSpilled == RING) { const int2 sp_ = RT_RING(stackSpilled); stack[stackSpilled++] = node_ref(sp_); RT_PROF(28, 1); } \
                            const NodeRef px_ = (x); RT_RING(stackCount) = make_int2(px_.start, px_.count); stackCount++; } \
                        else { stack[stackCount++] = (x); } } while (0)
#define RT_POP(dst) do { if constexpr (RING > 0) { --stackCount; if (stackCount < stackSpilled) { (dst) = stack[--stackSpilled]; RT_PROF(29, 1); } \
                             else { (dst) = node_ref(RT_RING(stackCount)); } } \
                         else { (dst) = stack[--stackCount]; } } while (0)
#endif
#define RT_STACK_RESET() stackSpilled = 0
#ifndef RT_LEAF_REPEAT
#define RT_LEAF_REPEAT 1
#endif
//   RT_VOTE_WI / RT_VOTE_WL / RT_VOTE_WN   weights of the vote: the warp runs the step kind with the largest lanes x weight.  A leaf step
//                      (one triangle) costs about a third of an inner step (two node visits) and returns its lanes to the inner
//                      population sooner; counted on the SIMT interpreter build (step counts are exact there, the instruction cost per
//                      step kind is an estimate from the SASS line profile: census 20, inner 150, leaf 55, next 90), weights 1 / 3 / 2
//                      cut the inner steps of the 200k-triangle soup by 22 % (they run with 20 lanes instead of 15.6) and the estimated
//                      instruction count by 17 %; likewise on the knot scenes and on 24 instanced models; default 1 / 3 / 2 (rt_devmath.cuh).
#ifndef RT_VOTE_WI
#define RT_VOTE_WI 1
#endif
#ifndef RT_VOTE_WL
#define RT_VOTE_WL 1
#endif
#ifndef RT_VOTE_WN
#define RT_VOTE_WN 1
#endif
// Schedule profiler of the SIMT interpreter build (tools/simt_schedule_profile.py; never defined in the product build): the
// scheduling knobs become run-time values and the kernel counts census iterations, the lanes per step kind, phases and batches.
#if defined(RT_SIMT_PROFILE) && defined(RT_SIMT_EMU)
#undef RT_VOTE_WI
#undef RT_VOTE_WL
#undef RT_VOTE_WN
#undef RT_INNER_REPEAT
#undef RT_LEAF_REPEAT
#define RT_VOTE_WI simt::knob[0]
#define RT_VOTE_WL simt::knob[1]
#define RT_VOTE_WN simt::knob[2]
#define RT_INNER_REPEAT simt::knob[3]
#define RT_LEAF_REPEAT_RUNTIME simt::knob[4]
#define RT_PROF(i, v) simt::prof_add(i, (unsigned long long)(v))
#else
#define RT_PROF(i, v) do { } while (0)
#endif
//   RT_PREFETCH_CUR    the moment a lane learns which node it visits next (descent, pop, start of a model) it asks L1 for that node's
//                      record (or the leaf's first triangle): the census, the vote and the other step kinds of the following
//                      iterations run while the line travels, instead of the load being issued at the top of the step that needs it
#if defined(RT_PREFETCH_CUR) && !defined(RT_SIMT_EMU)
#define RT_PF_CUR() do { const void* pfAddr = cur.count > 0 ? (EXT && P.sphBvh && model < 0 ? (const void*)(P.sphLeaves + cur.start) : (const void*)(P.triGeom + cur.start)) \
                                                             : (EXT && P.sphBvh && model < 0 ? (const void*)(P.sphPairs + cur.start) : (const void*)(P.pairs + (cur.start & 0x3fffffff))); \
                         asm volatile("prefetch.global.L1 [%0];" :: "l"(pfAddr)); } while (0)
#else
#define RT_PF_CUR() do { } while (0)
#endif
// RT_POOL_CLOCKS (variant build only, tools/build_variants.py "clocks", read by tools/pool_clocks.py): a cycle account of the kernel.
// Lane 0 of every warp adds, per step kind, the clock64() cycles since the previous mark, the number of such steps and the lanes (or
// slots) they served into 32-bit counters in shared memory (96 bytes per warp after the stack rings); when the warp ends it adds them
// to g_poolClocks.  The marks cost a few instructions per step: on the default workload the build runs 16-21 % slower (DESIGN §5).
#if defined(RT_POOL_CLOCKS) && !defined(RT_SIMT_EMU)
enum : int { CK_CENSUS = 0, CK_INNER, CK_LEAF, CK_NEXT, CK_SHADE, CK_REFILL, CK_CAMERA, CK_QUEUE, CK_KINDS };
constexpr int POOL_CLOCK_BYTES = 3 * CK_KINDS * 4;                  // per warp: [cycles, steps, lanes] x kind
__device__ unsigned long long g_poolClocks[3 * CK_KINDS];
#define RT_CK_INIT() unsigned* ckAcc = reinterpret_cast<unsigned*>(poolBase + (size_t)POOL_WARPS * POOL_BYTES + (size_t)POOL_THREADS * RING * 8) \
                                       + warp * (3 * CK_KINDS); \
                     if (lane < 3u * CK_KINDS) ckAcc[lane] = 0u; __syncwarp(); long long ckT = clock64()
#define RT_CK(kind, lanes) do { const long long t_ = clock64(); \
                                if (lane == 0) { ckAcc[3 * (kind)] += (unsigned)(t_ - ckT); ckAcc[3 * (kind) + 1]++; ckAcc[3 * (kind) + 2] += (unsigned)(lanes); } \
                                ckT = t_; } while (0)
#define RT_CK_FLUSH() do { __syncwarp(); if (lane < 3u * CK_KINDS) atomicAdd(g_poolClocks + lane, (unsigned long long)ckAcc[lane]); } while (0)
#else
constexpr int POOL_CLOCK_BYTES = 0;
#define RT_CK_INIT() do { } while (0)
#define RT_CK(kind, lanes) do { } while (0)
#define RT_CK_FLUSH() do { } while (0)
#endif
constexpr int POOL_WARPS = RT_POOL_WARPS;      // warps per CTA (one persistent CTA per SM)
constexpr int POOL_THREADS = POOL_WARPS * 32;
constexpr int POOL_WORDS = 24;                 // 32-bit words of state per path slot

// slot state (low 4 bits of the info word)
enum : unsigned { PS_EMPTY = 0, PS_GEN = 1, PS_RAY = 2, PS_HIT_MISS = 3, PS_HIT_OPAQUE = 4, PS_HIT_GLASS = 5, PS_DONE = 6,
                  PS_FLIGHT = 7 /* a lane is tracing this slot's ray (possibly across phases) */ };


// word index of each field inside a pool (field-major: word f of slot e is pool[f * M + e], conflict-free for lane = e).
// RT_POOL_COLD_GLOBAL: the first POOL_HOT_WORDS fields — what the trace phase touches: info, ray, hit record — stay in shared memory;
// the others (pixel, RNG state, transmittance, light, running sum: read and written once per segment, in the shade phase) live in a
// per-warp block of global memory (L2-resident, ~80 bytes per segment against ~10 KB of node records), which hands 66 KB of
// shared memory per CTA back to L1.
#ifdef RT_POOL_COLD_GLOBAL
enum : int { F_INFO = 0, F_POS, F_DIR = F_POS + 3, F_HDST = F_DIR + 3, F_HPRIM, F_HU, F_HV, F_HDET, F_HMODEL,
             F_XY, F_RNG, F_TRN, F_LGT = F_TRN + 3, F_SUM = F_LGT + 3 };
constexpr int POOL_HOT_WORDS = F_XY;
static_assert(F_SUM + 3 == POOL_WORDS && POOL_HOT_WORDS == 13, "pool layout");
#else
enum : int { F_XY = 0, F_RNG, F_INFO, F_POS, F_DIR = F_POS + 3, F_TRN = F_DIR + 3, F_LGT = F_TRN + 3, F_SUM = F_LGT + 3,
             F_HDST = F_SUM + 3, F_HPRIM, F_HU, F_HV, F_HDET, F_HMODEL };
constexpr int POOL_HOT_WORDS = POOL_WORDS;
static_assert(F_HMODEL == POOL_WORDS - 1, "pool layout");
#endif
constexpr int POOL_COLD_WORDS = POOL_WORDS - POOL_HOT_WORDS;

RT_DI NodeRef node_ref(int2 v) { NodeRef r; r.start = v.x; r.count = v.y; return r; }

RT_DI unsigned info_pack(unsigned sample, unsigned bounce, unsigned state) { return (sample << 12) | (bounce << 4) | state; }
RT_DI unsigned info_state(unsigned i) { return i & 15u; }
RT_DI unsigned info_bounce(unsigned i) { return (i >> 4) & 255u; }
RT_DI unsigned info_sample(unsigned i) { return i >> 12; }

template <int M> struct PoolView
{
    float* w;                                   // POOL_HOT_WORDS * M words of shared memory
    float* g;                                   // POOL_COLD_WORDS * M words of global memory (RT_POOL_COLD_GLOBAL)
    unsigned char* order;                       // M slot indices
    // (`field` is a constant at every call site: after inlining each access is a plain shared or a plain global one)
    RT_DI float* at(int field, int e) const { return field < POOL_HOT_WORDS ? w + field * M + e : g + (field - POOL_HOT_WORDS) * M + e; }
    RT_DI float& f(int field, int e) const { return *at(field, e); }
    RT_DI unsigned& u(int field, int e) const { return *reinterpret_cast<unsigned*>(at(field, e)); }
    RT_DI int& i(int field, int e) const { return *reinterpret_cast<int*>(at(field, e)); }
    RT_DI f3 get3(int field, int e) const { return make_f3(f(field, e), f(field + 1, e), f(field + 2, e)); }
    RT_DI void set3(int field, int e, f3 v) const { f(field, e) = v.x; f(field + 1, e) = v.y; f(field + 2, e) = v.z; }
    // the hit record of slot e (the running result of the ray traced on it): a triangle of a model ...
    RT_DI void set_hit(int e, float dst, int prim, float u, float v, float det, int model) const
    { f(F_HDST, e) = dst; i(F_HPRIM, e) = prim; f(F_HU, e) = u; f(F_HV, e) = v; f(F_HDET, e) = det; i(F_HMODEL, e) = model; }
    // ... or sphere s of the Spheres buffer (u, v and model keep their values: the shade phase does not read them for spheres)
    RT_DI void set_sphere_hit(int e, float dst, int s, bool inside) const
    { f(F_HDST, e) = dst; i(F_HPRIM, e) = -(s + 1); f(F_HDET, e) = inside ? -1.0f : 1.0f; }
};

// Build in `order` the list of slots whose state is in [lo, hi], grouped by state (ascending); returns the count.
template <int M> RT_DI int CompactByState(const PoolView<M>& pool, unsigned lane, unsigned lo, unsigned hi)
{
    const unsigned ltMask = (1u << lane) - 1u;
    int base = 0;
    for (unsigned st = lo; st <= hi; st++)
    {
#pragma unroll
        for (int c = 0; c < M / 32; c++)
        {
            const int e = c * 32 + (int)lane;
            const bool has = info_state(pool.u(F_INFO, e)) == st;
            const unsigned m = __ballot_sync(0xffffffffu, has);
            if (has) pool.order[base + __popc(m & ltMask)] = (unsigned char)e;
            base += __popc(m);
        }
    }
    __syncwarp();
    return base;
}

// Ray queue of the trace phase, grouped by the octant of the ray direction (sign bits): rays that pop together tend to
// order the children of a node the same way and touch the same nodes.  Active-path sorting; the order in which rays are
// traced does not enter any result.
template <int M> RT_DI int CompactRaysByOctant(const PoolView<M>& pool, unsigned lane)
{
    const unsigned ltMask = (1u << lane) - 1u;
    unsigned key[M / 32];
#pragma unroll
    for (int c = 0; c < M / 32; c++)
    {
        const int e = c * 32 + (int)lane;
        const bool isRay = info_state(pool.u(F_INFO, e)) == PS_RAY;
        const unsigned oct = (pool.u(F_DIR, e) >> 31) | ((pool.u(F_DIR + 1, e) >> 31) << 1) | ((pool.u(F_DIR + 2, e) >> 31) << 2);
        key[c] = isRay ? oct : 8u;
    }
    int base = 0;
    for (unsigned o = 0; o < 8u; o++)
    {
#pragma unroll
        for (int c = 0; c < M / 32; c++)
        {
            const bool has = key[c] == o;
            const unsigned m = __ballot_sync(0xffffffffu, has);
            if (has) pool.order[base + __popc(m & ltMask)] = (unsigned char)(c * 32 + (int)lane);
            base += __popc(m);
        }
    }
    __syncwarp();
    return base;
}

// The kernel body.  TLAS = the many-model instantiation (k_raytrace_pool_tlas): at the start of a ray's model loop one walk of the
// TLAS marks the models the ray can reach (TlasCollect, rt_device.cuh); the T_NEXT step then jumps from marked model to marked model,
// in buffer order, re-testing each against the running result.  The kernels measured in round 1 are the TLAS = false instantiations.
// FRAMES = the batch instantiations of rtDispatchFrames: a slot keeps its pixel for frames Frame .. Frame + P.frames - 1.  The sample
// field of the info word counts the samples of all of them (frame = sample / NumRaysPerPixel); when a frame's samples end the slot
// writes and accumulates that frame, reseeds and starts the next one instead of freeing itself.
// LIST = the list-driven instantiations of rtDispatchAdaptive: the refill takes job < totalJobs -> list[job] ((y << 16) | x), and the
// pixel's write also updates its moments.
template <bool STATS, bool EXT, bool TLAS, int M, bool FRAMES = false, bool LIST = false>
RT_DI void pool_body(const DevParams& P, const unsigned int totalJobs, const unsigned int tilesX, const unsigned int ownedRows,
                     const unsigned int* list = nullptr, float4* moments = nullptr)
{
    static_assert(!(LIST && FRAMES), "a pixel list runs one frame");
    RT_DYNAMIC_SMEM(smemRaw);
    WaveSmemHeader* hdr = reinterpret_cast<WaveSmemHeader*>(smemRaw);
    float4* smemPairs = reinterpret_cast<float4*>(smemRaw + sizeof(WaveSmemHeader));
    DevSphere* smemSpheres = reinterpret_cast<DevSphere*>(smemRaw + sizeof(WaveSmemHeader) + (size_t)P.smemPairs * sizeof(NodePair));
    const int nSmemSpheres = P.sphereCount < WAVE_MAX_SMEM_SPHERES ? P.sphereCount : WAVE_MAX_SMEM_SPHERES;
    unsigned char* poolBase = reinterpret_cast<unsigned char*>(smemSpheres + nSmemSpheres);
    constexpr int POOL_BYTES = POOL_HOT_WORDS * M * 4 + M;      // M is a multiple of 32, so every pool stays 16-byte aligned

    const unsigned lane = threadIdx.x & 31u;
    const unsigned warp = threadIdx.x >> 5;
    const unsigned ltMask = (1u << lane) - 1u;
    PoolView<M> pool;
    pool.w = reinterpret_cast<float*>(poolBase + (size_t)warp * POOL_BYTES);
    pool.order = reinterpret_cast<unsigned char*>(pool.w + POOL_HOT_WORDS * M);
    pool.g = POOL_COLD_WORDS ? P.poolCold + ((size_t)blockIdx.x * POOL_WARPS + warp) * (size_t)(POOL_COLD_WORDS * M) : nullptr;
    constexpr int RING = PoolRing<M>::N;
    // this warp's RING x 32 int2 entries; ringLane = this lane's word of entry 0
    int2* ringLane = reinterpret_cast<int2*>(poolBase + (size_t)POOL_WARPS * POOL_BYTES) + (size_t)warp * (RING * 32) + lane;
    int stackSpilled = 0;
    (void)ringLane; (void)stackSpilled;

    // ---- stage the tree tops (TMA bulk copy) and the spheres; initialise the pool -------------------------------------
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
        uint32_t off = 0;
        while (off < bytes)
        {
            const uint32_t n = (bytes - off) < 32768u ? (bytes - off) : 32768u;
            tma_bulk_g2s(smem_u32(smemPairs) + off, reinterpret_cast<const unsigned char*>(P.pairs) + off, n, mbar);
            off += n;
        }
    }
    for (int i = threadIdx.x; i < nSmemSpheres; i += POOL_THREADS) smemSpheres[i] = P.spheres[i];
#pragma unroll
    for (int c = 0; c < M / 32; c++) pool.u(F_INFO, c * 32 + (int)lane) = info_pack(0, 0, PS_EMPTY);
    if (P.smemPairs > 0) { while (!mbar_try_wait(mbar, 0)) { } }
    __syncthreads();
    RT_CK_INIT();

    Counters cnt; cnt.rays = cnt.box = cnt.tri = cnt.sph = cnt.sbox = 0;
    // STATS: the counters when this lane fetched the ray it traces (which may stay in flight across shade phases); the difference
    // goes to the ray's pixel (the slot's F_XY) when the ray finishes
    Counters rayStart = cnt;
    bool exhausted = false;                     // warp-uniform: the global pixel queue is empty
    // Fair share: when the image is small for the machine (multi-GPU tiles, small images) a warp fills at most its share of the
    // pixels, so that every SM gets work and — a pixel's samples being one sequential chain — all pixels start in the first round
    // instead of the first CTAs swallowing the queue.  With more pixels than slots (the usual case) the cap is the pool size.
    const unsigned int fairShare = (totalJobs + gridDim.x * POOL_WARPS - 1u) / (gridDim.x * POOL_WARPS);
    const int slotCap = fairShare < (unsigned int)M ? (int)(fairShare ? fairShare : 1u) : M;

    // per-lane ray state of the trace phase.  It lives across phases: a lane whose ray is still in flight when the phase
    // ends keeps it (slot state PS_FLIGHT) and continues in the next trace phase, so long rays never hold the warp back.
    enum { T_IDLE = 0, T_INNER = 1, T_LEAF = 2, T_NEXT = 3 };
    int mode = T_IDLE;
    int myEntry = -1;                                                // slot this lane is tracing
    f3 lpos = splat3(0.0f), ldir = splat3(0.0f), linv = splat3(0.0f);
    // The ray's running result lives in its slot's hit words (F_HDST .. F_HMODEL): an improving hit writes them at once (rare,
    // predicated stores), so a ray that ends only flips its slot's state.  The registers keep what the tests compare
    // against: bestDst (= result.dst; every model starts from it, HL:359, so a model's winner always becomes the result), the
    // hit kind, and for the sphere accelerator's first-index tie rule the buffer index of its best sphere.  The world ray is
    // re-read from F_POS / F_DIR in the T_NEXT step, the only one that needs it.
    float bestDst = inf32(); int bestTri = -1; unsigned hitKind = PS_HIT_MISS;
    int model = 0; bool cull = true;
    NodeRef cur; cur.start = 0; cur.count = 0;
    int leafK = 0;
    NodeRef stack[WAVE_STACK];
    int stackCount = 0;
#ifdef RT_STACK_TOP_REG
    NodeRef stackTop; stackTop.start = 0; stackTop.count = 0;
#endif
#ifdef RT_CACHE_RAYINV
    f3 rayInvW = splat3(0.0f);
#endif
    unsigned int tlasMask[TLAS ? RT_TLAS_WORDS : 1];                 // models this lane's ray can reach (valid from its first model step)
    const bool useTlas = TLAS && !STATS && P.modelSkip && P.tlas;

    for (;;)
    {
        // ================================================= SHADE phase =================================================
        // (1) shade the slots that came back from tracing, sorted by hit kind
        {
            const int n = CompactByState<M>(pool, lane, PS_HIT_MISS, PS_HIT_GLASS);
            if (lane == 0) { RT_PROF(14, 1); RT_PROF(15, (n + 31) / 32); RT_PROF(16, n); }
            for (int i0 = 0; i0 < n; i0 += 32)
            {
                const int i = i0 + (int)lane;
                if (i < n)
                {
                    const int e = pool.order[i];
                    const unsigned info = pool.u(F_INFO, e);
                    PathState ray;
                    ray.pos = pool.get3(F_POS, e); ray.dir = pool.get3(F_DIR, e);
                    ray.transmittance = pool.get3(F_TRN, e); ray.totalLight = pool.get3(F_LGT, e);
                    uint32_t rngState = pool.u(F_RNG, e);

                    // rebuild the hit (HL:319-320 / HL:208-209,365-369) from the compact record
                    Hit hit;
                    hit.dst = pool.f(F_HDST, e); hit.isBackface = false; hit.material = nullptr;
                    hit.normal = splat3(0.0f); hit.pos = splat3(0.0f);
                    if (info_state(info) != PS_HIT_MISS)
                    {
                        const int prim = pool.i(F_HPRIM, e);
                        hit.pos = ray.pos + ray.dir * hit.dst;
                        if (prim < 0)
                        {
                            const int s = -prim - 1;
                            const bool inside = pool.f(F_HDET, e) < 0.0f;
                            f3 centre;
                            if (s < WAVE_MAX_SMEM_SPHERES) { const DevSphere sp = smemSpheres[s]; centre = make_f3(sp.cx, sp.cy, sp.cz); }
                            else centre = make_f3(P.spheres[s].cx, P.spheres[s].cy, P.spheres[s].cz);
                            hit.isBackface = inside;
                            hit.normal = normalize3(hit.pos - centre) * (inside ? -1.0f : 1.0f);
                            hit.material = &P.Spheres[s].material;
                        }
                        else
                        {
                            const int model = pool.i(F_HMODEL, e);
                            const float det = pool.f(F_HDET, e);
                            const float4* nq = reinterpret_cast<const float4*>(P.triNormals + prim);
                            const float4 n0 = ldg_tri(nq), n1 = ldg_tri(nq + 1), n2 = ldg_tri(nq + 2);
                            const f3 n = TriangleSmoothNormal(make_f3(n0.x, n0.y, n0.z), make_f3(n0.w, n1.x, n1.y), make_f3(n1.z, n1.w, n2.x),
                                                              pool.f(F_HU, e), pool.f(F_HV, e), det);
                            const float4* mr = reinterpret_cast<const float4*>(P.models + model) + 3;
                            const float4 r0 = __ldg(mr), r1 = __ldg(mr + 1), r2 = __ldg(mr + 2);
                            const float l2w[12] = {r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, r1.z, r1.w, r2.x, r2.y, r2.z, r2.w};
                            hit.isBackface = det < 0.0f;
                            hit.normal = normalize3(mul_rm(l2w, n, 0.0f));
                            hit.material = &P.ModelInfo[model].material;
                        }
                    }
                    const bool cont = ShadeSegment(P, hit, ray, rngState);
                    unsigned sample = info_sample(info), bounce = info_bounce(info) + 1u;
                    unsigned state = PS_RAY;
                    pool.u(F_RNG, e) = rngState;
                    if (!cont || (int)bounce > P.MaxBounceCount)
                    {
                        const f3 sum = pool.get3(F_SUM, e) + ray.totalLight;              // HL:578
                        sample++;
                        if (FRAMES ? sample % (unsigned)P.NumRaysPerPixel == 0u : (int)sample >= P.NumRaysPerPixel)
                        {
                            // pixel finished (RC:18-23)
                            const unsigned xy = pool.u(F_XY, e);
                            const size_t o = (size_t)(xy >> 16) * P.W + (xy & 0xffffu);
                            const f3 pixelCol = sum / __int2float_rn(P.NumRaysPerPixel);
                            WritePixel<EXT, LIST>(P, o, pixelCol.x, pixelCol.y, pixelCol.z, moments);
                            state = PS_EMPTY;
                            if (FRAMES && sample < (unsigned)P.NumRaysPerPixel * (unsigned)P.frames)
                            {
                                // the pixel's next frame on the same slot
                                pool.u(F_RNG, e) = FrameSeed(SetupPixel(P, xy & 0xffffu, xy >> 16).rngState, sample / (unsigned)P.NumRaysPerPixel);
                                pool.set3(F_SUM, e, splat3(0.0f));
                                state = PS_GEN;
                            }
                        }
                        else { pool.set3(F_SUM, e, sum); state = PS_GEN; }
                        bounce = 0;
                    }
                    else
                    {
                        pool.set3(F_POS, e, ray.pos); pool.set3(F_DIR, e, ray.dir);
                        pool.set3(F_TRN, e, ray.transmittance); pool.set3(F_LGT, e, ray.totalLight);
                    }
                    pool.u(F_INFO, e) = info_pack(sample, bounce, state);
                }
            }
            __syncwarp();
            RT_CK(CK_SHADE, n);
        }

        // (2) refill free slots from the global pixel queue (ballot compaction, one atomic per warp per pass)
        while (!exhausted)
        {
            bool anyEmpty = false;
#pragma unroll
            for (int c = 0; c < M / 32; c++)
            {
                const int e = c * 32 + (int)lane;
                const bool need = info_state(pool.u(F_INFO, e)) == PS_EMPTY && e < slotCap;
                const unsigned needMask = __ballot_sync(0xffffffffu, need);
                if (needMask == 0u || exhausted) continue;
                unsigned base = 0;
                const int leader = __ffs(needMask) - 1;
                if ((int)lane == leader) base = atomicAdd(P.workCounter, (unsigned)__popc(needMask));
                base = __shfl_sync(0xffffffffu, base, leader);
                if (need)
                {
                    const unsigned job = base + (unsigned)__popc(needMask & ltMask);
                    if (LIST && job < totalJobs)
                    {
                        const unsigned xy = list[job];
                        pool.u(F_XY, e) = xy;
                        pool.u(F_RNG, e) = SetupPixel(P, xy & 0xffffu, xy >> 16).rngState;
                        pool.set3(F_SUM, e, splat3(0.0f));
                        pool.u(F_INFO, e) = info_pack(0, 0, PS_GEN);
                    }
                    else if (!LIST && job < totalJobs)
                    {
                        const unsigned tile = job >> 5, l = job & 31u;
                        const unsigned x = (tile % tilesX) * 8u + (l & 7u);
                        const unsigned r = (tile / tilesX) * 4u + (l >> 3);
                        if (x < P.limX && r < ownedRows)
                        {
                            const unsigned y = ((r / (unsigned)P.bandRows) * (unsigned)P.tileWorld + (unsigned)P.tileRank) * (unsigned)P.bandRows
                                             + (r % (unsigned)P.bandRows);
                            pool.u(F_XY, e) = (y << 16) | x;
                            pool.u(F_RNG, e) = SetupPixel(P, x, y).rngState;
                            pool.set3(F_SUM, e, splat3(0.0f));
                            pool.u(F_INFO, e) = info_pack(0, 0, PS_GEN);
                        }
                    }
                }
                if (base + (unsigned)__popc(needMask) >= totalJobs) exhausted = true;        // warp-uniform
                else if (__ballot_sync(0xffffffffu, info_state(pool.u(F_INFO, e)) == PS_EMPTY && e < slotCap)) anyEmpty = true;   // padding jobs: try again
            }
            if (!anyEmpty) break;
        }
        if (exhausted)
        {
#pragma unroll
            for (int c = 0; c < M / 32; c++)
            {
                const int e = c * 32 + (int)lane;
                if (info_state(pool.u(F_INFO, e)) == PS_EMPTY) pool.u(F_INFO, e) = info_pack(0, 0, PS_DONE);
            }
        }
        __syncwarp();
        RT_CK(CK_REFILL, 0);

        // (3) camera rays for the slots that start a sample (HL:567-576), in compacted batches
        {
            const int n = CompactByState<M>(pool, lane, PS_GEN, PS_GEN);
            if (lane == 0) { RT_PROF(17, (n + 31) / 32); RT_PROF(18, n); }
            for (int i0 = 0; i0 < n; i0 += 32)
            {
                const int i = i0 + (int)lane;
                if (i < n)
                {
                    const int e = pool.order[i];
                    const unsigned xy = pool.u(F_XY, e);
                    const PixelSetup px = SetupPixel(P, xy & 0xffffu, xy >> 16);
                    uint32_t rngState = pool.u(F_RNG, e);
                    PathState ray;
                    GenerateCameraRay(P, px, rngState, ray);
                    pool.u(F_RNG, e) = rngState;
                    pool.set3(F_POS, e, ray.pos); pool.set3(F_DIR, e, ray.dir);
                    pool.set3(F_TRN, e, ray.transmittance); pool.set3(F_LGT, e, ray.totalLight);
                    pool.u(F_INFO, e) = info_pack(info_sample(pool.u(F_INFO, e)), 0, PS_RAY);
                }
            }
            __syncwarp();
            RT_CK(CK_CAMERA, n);
        }

        // ================================================= TRACE phase =================================================
        const int nRays = P.sortRays ? CompactRaysByOctant<M>(pool, lane) : CompactByState<M>(pool, lane, PS_RAY, PS_RAY);
        RT_CK(CK_QUEUE, nRays);
        if (nRays == 0 && __ballot_sync(0xffffffffu, mode != T_IDLE) == 0u) break;   // every slot is DONE: this warp is finished
        int next = 0;                                                // warp-uniform queue head
        bool finishedAny = false;                                    // warp-uniform: some ray completed in this phase

        for (;;)
        {
            // ---- census: how many lanes wait in each mode (one warp reduction on byte-packed counters) ----
            const unsigned census = __reduce_add_sync(0xffffffffu, 1u << (8 * mode));
            const int nIdle = (int)(census & 255u), nInner = (int)((census >> 8) & 255u), nLeaf = (int)((census >> 16) & 255u), nNext = (int)(census >> 24);
            if (lane == 0) { RT_PROF(0, 1); RT_PROF(1, nIdle); RT_PROF(2, nInner); RT_PROF(3, nLeaf); RT_PROF(4, nNext); }

            // ---- fetch: idle lanes take the next rays of the warp queue in the T_NEXT step below (ballot rank, no atomics) ----
            const bool fetch = nIdle != 0 && next < nRays;
            if (nIdle == 32 && !fetch) break;
            // queue drained and only a few long rays left: go shade what has finished, they continue next phase
            if (next >= nRays && (32 - nIdle) <= P.tailLanes && finishedAny) break;

            // ---- vote: run the step kind most lanes are waiting for (ties: finish/advance first, then inner nodes) ----
            // Lanes are independent state machines (inner node / leaf triangle / next model); executing every kind each
            // iteration would run each at a fraction of the warp.  One kind per iteration keeps the executed block dense,
            // the others catch up when their kind becomes the majority.  The per-ray visiting order is unchanged.
            // (RT_VOTE_W*: cost-weighted vote, see the macro block at the top; all weights 1 = the plain majority)
            RT_CK(CK_CENSUS, 32 - nIdle);         // (census and vote of this iteration)
            const int scoreInner = nInner * RT_VOTE_WI, scoreLeaf = nLeaf * RT_VOTE_WL, scoreNext = nNext * RT_VOTE_WN;
            if (fetch || (scoreNext >= scoreInner && scoreNext >= scoreLeaf))
            {
                if (lane == 0) { RT_PROF(5, 1); RT_PROF(6, nNext); }
                // ---- advance to the next model / finish the ray, and start the next rays of the queue ----
                // A lane whose ray ends, and at the start of a phase every idle lane, takes the next ray of the queue in this step
                // and advances it to its first model, instead of going idle for a census, a fetch and another T_NEXT step.  A new
                // ray that reaches no model ends in its turn, hence the loop: it stops at the first pass that leaves no lane idle
                // or finds the queue empty (warp-uniform).
                bool adv = mode == T_NEXT;
                for (;;)
                {
                    if (adv)
                    {
                        // (a model's winner, HL:362-370, and the sphere phase's are in the slot's hit words already)
                        const f3 rayPos = pool.get3(F_POS, myEntry), rayDir = pool.get3(F_DIR, myEntry);
                        model++;
                        // skip the models this ray cannot reach before its current best hit (not in the instrumented build, which
                        // walks every model like the reference so that the test counts stay identical)
                        if (!STATS && P.modelSkip && model >= 0)
                        {
#ifdef RT_CACHE_RAYINV
                            const f3 rayInv = rayInvW;
#else
                            const f3 rayInv = rcp3(rayDir);
#endif
                            if (useTlas)
                            {
                                if (model == 0) TlasCollect(P, rayPos, rayInv, bestDst, tlasMask);
                                for (;;)
                                {
                                    model = TlasNext(tlasMask, model, P.modelCount);
                                    if (model >= P.modelCount || !ModelOutOfReach(reinterpret_cast<const float4*>(P.models + model), rayPos, rayInv, bestDst)) break;
                                    model++;
                                }
                            }
                            else
                            while (model < P.modelCount && ModelOutOfReach(reinterpret_cast<const float4*>(P.models + model), rayPos, rayInv, bestDst)) model++;
                        }
                    }
                    const bool fin = adv && model >= P.modelCount;
                    if (fin)
                    {
                        const unsigned info = pool.u(F_INFO, myEntry);
                        pool.u(F_INFO, myEntry) = (info & ~15u) | hitKind;
                        if (STATS)
                        {
                            const unsigned xy = pool.u(F_XY, myEntry);
                            AddPixelStats(P, (size_t)(xy >> 16) * P.W + (xy & 0xffffu), cnt, rayStart);
                        }
                        mode = T_IDLE; myEntry = -1;
                    }
                    if (__ballot_sync(0xffffffffu, fin) != 0u) finishedAny = true;
                    const bool need = mode == T_IDLE;
                    const unsigned needMask = __ballot_sync(0xffffffffu, need);
                    if (needMask == 0u || next >= nRays) break;
                    const int idx = next + __popc(needMask & ltMask);
                    next += __popc(needMask);
                    adv = need && idx < nRays;
                    if (adv)
                    {
                        // start the ray of queue entry idx; the next pass advances it to its first model
                        myEntry = pool.order[idx];
                        pool.u(F_INFO, myEntry) = (pool.u(F_INFO, myEntry) & ~15u) | PS_FLIGHT;
                        if (STATS) rayStart = cnt;
                        cnt.rays++;
#ifdef RT_CACHE_RAYINV
                        rayInvW = rcp3(pool.get3(F_DIR, myEntry));
#endif
                        bestDst = inf32(); hitKind = PS_HIT_MISS;
                        pool.set_hit(myEntry, inf32(), 0, 0.0f, 0.0f, 0.0f, 0);
                        // spheres first (extension; where the reference's commented call sits, HL:341)
                        // A large Spheres buffer is searched through its accelerator by the same state machine as the meshes
                        // ("model -1": inner nodes = padded sphere boxes, leaves = spheres), see the T_NEXT / T_INNER / T_LEAF blocks.
                        if (!(EXT && P.sphBvh) && P.sphereCount > 0)
                        {
                            const f3 rayPos = pool.get3(F_POS, myEntry), rayDir = pool.get3(F_DIR, myEntry);
                            for (int s = 0; s < P.sphereCount; s++)
                            {
                                float cx, cy, cz, r2; int flag;
                                if (s < WAVE_MAX_SMEM_SPHERES) { const DevSphere sp = smemSpheres[s]; cx = sp.cx; cy = sp.cy; cz = sp.cz; r2 = sp.r2; flag = sp.pad0; }
                                else { const float4 s0 = __ldg(reinterpret_cast<const float4*>(P.spheres + s)); cx = s0.x; cy = s0.y; cz = s0.z;
                                       r2 = __ldg(&P.spheres[s].r2); flag = __ldg(&P.spheres[s].pad0); }
                                float dst; bool inside;
                                if (STATS) cnt.sph++;
                                if (RaySphereCore(rayPos, rayDir, make_f3(cx, cy, cz), r2, dst, inside) && dst < bestDst)
                                {
                                    bestDst = dst; hitKind = flag == RT_MATERIAL_GLASS ? PS_HIT_GLASS : PS_HIT_OPAQUE;
                                    pool.set_sphere_hit(myEntry, dst, s, inside);
                                }
                            }
                        }
                        model = (EXT && P.sphBvh) ? -2 : -1; mode = T_NEXT;
                    }
                }
                // enter the model (or the sphere phase) the advance stopped at: lanes that stay on their ray and lanes that
                // started a new one together
                if (mode == T_NEXT)
                {
                    const f3 rayPos = pool.get3(F_POS, myEntry), rayDir = pool.get3(F_DIR, myEntry);
                    if (EXT && P.sphBvh && model == -1)
                    {
                        // sphere phase: world-space ray against the accelerator of the Spheres buffer (semantics of TraverseSpheres).
                        // It comes first, so bestDst is still inf (no small-buffer sphere loop runs with an accelerator).
                        lpos = rayPos; ldir = rayDir; linv = rcp3(rayDir);
                        bestTri = 0x7fffffff;
                        cur.start = P.sphRootStart; cur.count = P.sphRootCount; leafK = 0; stackCount = 0; RT_STACK_RESET();
                        mode = cur.count > 0 ? T_LEAF : T_INNER; RT_PF_CUR();
                    }
                    else
                    {
                        const float4* mr = reinterpret_cast<const float4*>(P.models + model);
                        const float4 r0 = __ldg(mr), r1 = __ldg(mr + 1), r2 = __ldg(mr + 2);
                        const float w2l[12] = {r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, r1.z, r1.w, r2.x, r2.y, r2.z, r2.w};
                        const int4 meta = __ldg(reinterpret_cast<const int4*>(mr + 6));
                        lpos = mul_rm(w2l, rayPos, 1.0f);
                        ldir = mul_rm(w2l, rayDir, 0.0f);
                        linv = rcp3(ldir);
                        cull = meta.z != 0;                          // bestDst: result.dst is the ray length shared across models (HL:359)
                        cur.start = meta.x; cur.count = meta.y; leafK = 0; stackCount = 0; RT_STACK_RESET();
                        mode = cur.count > 0 ? T_LEAF : T_INNER; RT_PF_CUR();
                    }
                }
                RT_CK(CK_NEXT, nNext);
            }
            else if (scoreInner >= scoreLeaf)
            {
                if (lane == 0) { RT_PROF(7, 1); RT_PROF(8, nInner); }
                // ---- inner nodes: HL:262-282 ----  (RT_INNER_REPEAT visits per census: most lanes stay in this mode after a
                // visit, and the census / vote / loop control of an iteration costs about a third of a visit)
#pragma unroll 1
                for (int rep = 0; rep < RT_INNER_REPEAT; rep++)
                if (mode == T_INNER)
                {
                    const bool sph = EXT && P.sphBvh && model < 0;
                    float4 q0, q1, q2, q3;
                    if (sph)
                    {
                        const float4* p = reinterpret_cast<const float4*>(P.sphPairs + cur.start);
                        ldg_record64(p, q0, q1, q2, q3);
                        if (STATS) cnt.sbox += 2;
                    }
                    else
                    {
                        LoadPair<EXT>(P, smemPairs, cur.start, q0, q1, q2, q3);
                        RT_PROF(13, 1);
#if defined(RT_PREFETCH_NEXT_PAIR) && !defined(RT_SIMT_EMU)
                        // with "pairOrder" = 1 (pre-order records) the record of an inner child A is the next one: ask for it while this one is
                        // still in flight, so that a descent into A finds it in L1 (a wasted 64-byte prefetch when the ray goes to B or up)
                        asm volatile("prefetch.global.L1 [%0];" :: "l"(P.pairs + cur.start + 1));
#endif
                        if (STATS) cnt.box += 2;
                    }
                    const float dstA = RayBoundingBoxDst(lpos, linv, make_f3(q0.x, q0.y, q0.z), make_f3(q0.w, q1.x, q1.y));
                    const float dstB = RayBoundingBoxDst(lpos, linv, make_f3(q2.x, q2.y, q2.z), make_f3(q2.w, q3.x, q3.y));
                    NodeRef a, b;
                    a.start = __float_as_int(q1.z); a.count = __float_as_int(q1.w);
                    b.start = __float_as_int(q3.z); b.count = __float_as_int(q3.w);
                    const bool isNearestA = dstA <= dstB;
                    const float dstNear = isNearestA ? dstA : dstB;
                    const float dstFar = isNearestA ? dstB : dstA;
                    const NodeRef nearRef = isNearestA ? a : b;
                    const NodeRef farRef = isNearestA ? b : a;
                    // meshes: the reference's push-time test dst < best (HL:280-281).  Sphere boxes: conservative slack, ties kept
                    // (x*1 - 0 is x exactly, so the mesh comparison is unchanged; inf stays inf and never passes)
                    const float cs = sph ? 0.99999619f : 1.0f, cb = sph ? 1e-6f : 0.0f;
#if defined(RT_PUSH_PREDICATED) && !defined(RT_STACK_TOP_REG)
                    if constexpr (RING > 0)
                    {
                        // the push runs with few of 32 lanes: only the spill of a full ring stays a branch,
                        // the ring store is predicated
                        const bool push = (dstFar * cs - cb) < bestDst && stackCount < WAVE_STACK;
                        if (push && stackCount - stackSpilled == RING) { const int2 sp_ = RT_RING(stackSpilled); stack[stackSpilled++] = node_ref(sp_); RT_PROF(28, 1); }
                        if (push) RT_RING(stackCount) = make_int2(farRef.start, farRef.count);
                        stackCount += push ? 1 : 0;
                        if (push) { RT_PROF(11, 1); RT_PROF(32 + (stackCount < 31 ? stackCount : 31), 1); }
                    }
                    else
#endif
                    if ((dstFar * cs - cb) < bestDst && stackCount < WAVE_STACK) { RT_PUSH(farRef); RT_PROF(11, 1); RT_PROF(32 + (stackCount < 31 ? stackCount : 31), 1); }   // (prefetching the far record here was slower)
#if defined(RT_BRANCHLESS_POP) && !defined(RT_STACK_TOP_REG)
                    if constexpr (RING > 0)
                    {
                    // The pop below runs with few of 32 lanes: few lanes miss both children in the same step.
                    // With the stack top in shared memory every lane can afford to READ the top (a conflict-free 8-byte access) and
                    // select: descend into the near child or take the top.  When the near child is out of reach so is the far one
                    // (dstFar >= dstNear), so the stack was not pushed in this step and its top is exactly what a pop returns.
                    {
                        const bool goNear = (dstNear * cs - cb) < bestDst;
                        const bool ringHas = stackCount > stackSpilled;
                        NodeRef top = node_ref(RT_RING(stackCount - 1));
                        if (!goNear && !ringHas && stackCount > 0) { top = stack[stackSpilled - 1]; --stackSpilled; RT_PROF(29, 1); RT_PROF(30, 1); }      // rare: the ring ran empty above spilled entries
                        const bool pop = !goNear && stackCount > 0;
                        cur = goNear ? nearRef : top;
                        stackCount -= pop ? 1 : 0;
                        leafK = 0;
                        mode = (goNear || pop) ? (cur.count > 0 ? T_LEAF : T_INNER) : T_NEXT;
                        RT_PF_CUR();
                    }
                    }
                    else
#endif
                    {
                    if ((dstNear * cs - cb) < bestDst) { cur = nearRef; leafK = 0; mode = cur.count > 0 ? T_LEAF : T_INNER; RT_PF_CUR(); }
                    else if (stackCount > 0) { RT_POP(cur); leafK = 0; mode = cur.count > 0 ? T_LEAF : T_INNER; RT_PF_CUR(); }
                    else mode = T_NEXT;
                    }
                }
                RT_CK(CK_INNER, nInner);
            }
            else
            {
                if (lane == 0) { RT_PROF(9, 1); RT_PROF(10, nLeaf); }
                // ---- one leaf triangle: HL:248-260 ----
#ifdef RT_LEAF_REPEAT_RUNTIME
                for (int rep = 0; rep < RT_LEAF_REPEAT_RUNTIME; rep++)
#elif RT_LEAF_REPEAT > 1
#pragma unroll 1
                for (int rep = 0; rep < RT_LEAF_REPEAT; rep++)
#endif
                if (EXT && P.sphBvh && mode == T_LEAF && model < 0)
                {
                    // one sphere of the accelerator's leaf (reference test, first-index rule on equal dst)
                    const float4* q = reinterpret_cast<const float4*>(P.sphLeaves + cur.start + leafK);
                    const float4 s0 = __ldg(q), s1 = __ldg(q + 1);
                    float dst; bool inside;
                    if (STATS) cnt.sph++;
                    if (RaySphereCore(lpos, ldir, make_f3(s0.x, s0.y, s0.z), s1.x, dst, inside))
                    {
                        const int orig = __float_as_int(s1.z);
                        if (dst < bestDst || (dst == bestDst && orig < bestTri))
                        {
                            bestDst = dst; bestTri = orig;
                            hitKind = __float_as_int(s1.y) == RT_MATERIAL_GLASS ? PS_HIT_GLASS : PS_HIT_OPAQUE;
                            pool.set_sphere_hit(myEntry, dst, orig, inside);
                        }
                    }
                    leafK++;
                    if (leafK >= cur.count)
                    {
                        if (stackCount > 0) { RT_POP(cur); leafK = 0; mode = cur.count > 0 ? T_LEAF : T_INNER; RT_PF_CUR(); }
                        else mode = T_NEXT;
                    }
                }
                else if (mode == T_LEAF)
                {
                    const float4* g = reinterpret_cast<const float4*>(P.triGeom + cur.start + leafK);
                    float4 g0, g1, g2;
                    ldg_trigeom(g, g0, g1, g2);
                    float dst, u, v, det;
                    const bool didHit = RayTriangleCore(lpos, ldir, make_f3(g0.x, g0.y, g0.z), make_f3(g0.w, g1.x, g1.y), make_f3(g1.z, g1.w, g2.x),
                                                        make_f3(g2.y, g2.z, g2.w), cull, dst, u, v, det);
                    if (STATS) cnt.tri++;
                    if (didHit && dst < bestDst)
                    {
                        bestDst = dst; hitKind = cull ? PS_HIT_OPAQUE : PS_HIT_GLASS;   // cull == (flag != GLASS)
                        pool.set_hit(myEntry, dst, cur.start + leafK, u, v, det, model);
                    }
                    leafK++;
                    if (leafK >= cur.count)
                    {
                        if (stackCount > 0) { RT_POP(cur); leafK = 0; mode = cur.count > 0 ? T_LEAF : T_INNER; RT_PF_CUR(); }
                        else mode = T_NEXT;
                    }
                }
                RT_CK(CK_LEAF, nLeaf);
            }
        }
        __syncwarp();
    }
    RT_CK_FLUSH();

    // ---- counters ---------------------------------------------------------------------------------------------------------------
    const unsigned int r = __reduce_add_sync(0xffffffffu, cnt.rays);
    if (lane == 0) atomicAdd(P.counters + 0, (unsigned long long)r);
    if (STATS)
    {
        const unsigned int b = __reduce_add_sync(0xffffffffu, cnt.box), t = __reduce_add_sync(0xffffffffu, cnt.tri), s = __reduce_add_sync(0xffffffffu, cnt.sph), sb = __reduce_add_sync(0xffffffffu, cnt.sbox);
        if (lane == 0) { atomicAdd(P.counters + 1, (unsigned long long)b); atomicAdd(P.counters + 2, (unsigned long long)t); atomicAdd(P.counters + 3, (unsigned long long)s); atomicAdd(P.counters + 4, (unsigned long long)sb); }
    }
}

template <bool STATS, bool EXT, int M>
__global__ void __launch_bounds__(POOL_THREADS, 1) k_raytrace_pool(const __grid_constant__ DevParams P, const unsigned int totalJobs,
                                                                  const unsigned int tilesX, const unsigned int ownedRows)
{
    pool_body<STATS, EXT, false, M>(P, totalJobs, tilesX, ownedRows);
}

// many-model scenes: every extension + the TLAS (never instrumented: the counting build walks every model like the reference)
template <int M>
__global__ void __launch_bounds__(POOL_THREADS, 1) k_raytrace_pool_tlas(const __grid_constant__ DevParams P, const unsigned int totalJobs,
                                                                       const unsigned int tilesX, const unsigned int ownedRows)
{
    pool_body<false, true, true, M>(P, totalJobs, tilesX, ownedRows);
}

// rtDispatchFrames: P.frames frames of every pixel in one launch (kernels of their own, so that the kernels above keep their code)
template <bool STATS, bool EXT, int M>
__global__ void __launch_bounds__(POOL_THREADS, 1) k_raytrace_pool_frames(const __grid_constant__ DevParams P, const unsigned int totalJobs,
                                                                         const unsigned int tilesX, const unsigned int ownedRows)
{
    pool_body<STATS, EXT, false, M, true>(P, totalJobs, tilesX, ownedRows);
}

template <int M>
__global__ void __launch_bounds__(POOL_THREADS, 1) k_raytrace_pool_tlas_frames(const __grid_constant__ DevParams P, const unsigned int totalJobs,
                                                                              const unsigned int tilesX, const unsigned int ownedRows)
{
    pool_body<false, true, true, M, true>(P, totalJobs, tilesX, ownedRows);
}

// rtDispatchAdaptive: the selection's pixel list (totalJobs = its length), one frame per pixel (kernels of their own, so that the
// kernels above keep their code)
template <bool STATS, bool EXT, int M>
__global__ void __launch_bounds__(POOL_THREADS, 1) k_raytrace_pool_list(const __grid_constant__ DevParams P, const unsigned int totalJobs,
                                                                       const unsigned int* __restrict__ list, float4* __restrict__ moments)
{
    pool_body<STATS, EXT, false, M, false, true>(P, totalJobs, 0u, 0u, list, moments);
}

template <int M>
__global__ void __launch_bounds__(POOL_THREADS, 1) k_raytrace_pool_tlas_list(const __grid_constant__ DevParams P, const unsigned int totalJobs,
                                                                            const unsigned int* __restrict__ list, float4* __restrict__ moments)
{
    pool_body<false, true, true, M, false, true>(P, totalJobs, 0u, 0u, list, moments);
}

template <int M> inline size_t pool_smem_bytes(const DevParams& P)
{
    const int nS = P.sphereCount < WAVE_MAX_SMEM_SPHERES ? P.sphereCount : WAVE_MAX_SMEM_SPHERES;
    return sizeof(WaveSmemHeader) + (size_t)P.smemPairs * sizeof(NodePair) + (size_t)nS * sizeof(DevSphere) + (size_t)POOL_WARPS * (POOL_HOT_WORDS * M * 4 + M) + (size_t)POOL_THREADS * PoolRing<M>::N * 8
         + (size_t)POOL_WARPS * POOL_CLOCK_BYTES;
}

// Kernel 2's table: the __global__ of form F, <STATS, EXT, TLAS> and pool size M
template <CameraForm F, bool S, bool X, bool T, int M>
inline auto pool_kernel()
{
    if constexpr (F == FORM_LIST && T) return k_raytrace_pool_tlas_list<M>;
    else if constexpr (F == FORM_LIST) return k_raytrace_pool_list<S, X, M>;
    else if constexpr (F == FORM_FRAMES && T) return k_raytrace_pool_tlas_frames<M>;
    else if constexpr (F == FORM_FRAMES) return k_raytrace_pool_frames<S, X, M>;
    else if constexpr (T) return k_raytrace_pool_tlas<M>;
    else return k_raytrace_pool<S, X, M>;
}

// `f` with the pool size M (slots per warp) as a std::integral_constant; M = 0 is automatic: 64.  (96 slots so that every pixel of a
// small tile is resident at once lost on small tiles: the 96-slot pools have no room for the stack ring.)
template <class F>
inline cudaError_t with_pool_slots(int M, F f)
{
    if (M == 0 || M == 64) return f(std::integral_constant<int, 64>());
    if (M == 32) return f(std::integral_constant<int, 32>());
    if (M == 96) return f(std::integral_constant<int, 96>());
    return cudaErrorInvalidValue;
}

inline cudaError_t pool_configure()
{
    for (const int M : {32, 64, 96})
    {
        const cudaError_t e = with_pool_slots(M, [](auto m) {
            return for_each_camera_kernel([](auto F, auto S, auto X, auto T) {
                return cudaFuncSetAttribute(pool_kernel<F, S, X, T, decltype(m)::value>(), cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
            });
        });
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

// shared-memory bytes the pools leave for the tree-top cache (in NodePair records)
inline int pool_max_smem_pairs(int M, int sphereCount)
{
    const int nS = sphereCount < WAVE_MAX_SMEM_SPHERES ? sphereCount : WAVE_MAX_SMEM_SPHERES;
    const long long left = 227LL * 1024 - (long long)sizeof(WaveSmemHeader) - (long long)nS * (long long)sizeof(DevSphere)
                         - (long long)POOL_WARPS * (POOL_HOT_WORDS * M * 4 + M) - (long long)POOL_THREADS * (M >= 96 && !POOL_COLD_WORDS ? 0 : RT_RING_DEFAULT) * 8
                         - (long long)POOL_WARPS * POOL_CLOCK_BYTES - 1024;
    return left <= 0 ? 0 : (int)(left / (long long)sizeof(NodePair));
}

// Kernel 2 over one dispatch in `form` with pools of M slots; FORM_LIST: over the `count` pixels of `list`, whose moments its writes update
inline cudaError_t pool_launch(CameraForm form, const DevParams& P, int M, int numSMs, unsigned int count, const unsigned int* list,
                               float4* moments, cudaStream_t stream, cudaEvent_t evA, cudaEvent_t evB)
{
    CameraJobs J;
    if (!camera_jobs(form, P, count, J)) return cudaErrorInvalidValue;
    return with_pool_slots(M, [&](auto m) -> cudaError_t {
        const size_t smemBytes = pool_smem_bytes<m>(P);
        if (smemBytes > 227 * 1024) return cudaErrorInvalidConfiguration;
        unsigned int grid = (unsigned int)numSMs;                                   // one persistent CTA per SM
        const unsigned int ctasNeeded = (J.total + POOL_WARPS - 1) / POOL_WARPS;   // at least one pixel per warp: small images spread over the SMs (fair share, pool_body)
        if (grid > ctasNeeded) grid = ctasNeeded ? ctasNeeded : 1;
        grid = fit_persistent_grid(P.gridFit, grid, POOL_WARPS * m, J.total);
        return with_camera_kernel(form, P, [&](auto F, auto S, auto X, auto T) -> cudaError_t {
            const auto kernel = pool_kernel<F, S, X, T, decltype(m)::value>();
            cudaError_t e;
            if ((e = cudaMemsetAsync(P.workCounter, 0, sizeof(unsigned int), stream)) != cudaSuccess) return e;
            if ((e = cudaEventRecord(evA, stream)) != cudaSuccess) return e;
            if constexpr (F == FORM_LIST) RT_LAUNCH(grid, POOL_THREADS, smemBytes, stream, kernel, P, J.total, list, moments);
            else RT_LAUNCH(grid, POOL_THREADS, smemBytes, stream, kernel, P, J.total, J.tilesX, J.ownedRows);
            if ((e = cudaGetLastError()) != cudaSuccess) return e;
            return cudaEventRecord(evB, stream);
        });
    });
}

} // namespace rtd
