// rt_device.cuh — device functions of the path-tracing hot path, shared by every kernel variant.
//
// What is computed follows the reference shader (paths relative to the reference repo:
//   HL = Assets/Scripts/Tracer/RayCommon.hlsl, RC = Assets/Scripts/Tracer/RayCompute.compute);
// how it is organised (parameter block, material pointers instead of 88-byte copies, deferred
// normal evaluation, repacked node/triangle streams, ...) is this implementation's own.
#pragma once
#include "rt_devmath.cuh"
#include "../../include/rt_types.h"

namespace rtd {

// ---- cache policy of the triangle stream (compiled out by default) ------------------------------------------------------------
// Leaf triangles (48-byte TriGeom records, the normals of a winner) are touched once per test and rarely again soon, while the
// node-pair records of the upper tree are re-read by every ray: L1 capacity was the lever in round 1 (no shared-memory tree
// tops, 64-slot pools).  RT_TRI_LOAD_POLICY = 1 loads triangle data with L1::no_allocate, 2 with L1::evict_first, so that they do
// not displace node records; 0 (default) = plain read-only loads.  Same values either way.
#ifndef RT_TRI_LOAD_POLICY
#define RT_TRI_LOAD_POLICY 0
#endif
RT_DI float4 ldg_tri(const float4* p)
{
#if RT_TRI_LOAD_POLICY == 0 || defined(RT_SIMT_EMU)
    return __ldg(p);
#else
    float4 v;
#if RT_TRI_LOAD_POLICY == 1
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
#else
    asm volatile("ld.global.nc.L1::evict_first.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
#endif
    return v;
#endif
}

// ---- 64-byte record loads -------------------------------------------------------------------------------------------------------
// A node-pair record is read as four 128-bit loads (LDG.E.128, the widest global load sm_90 has), all issued before any is used.
RT_DI void ldg_record64(const float4* p, float4& q0, float4& q1, float4& q2, float4& q3)      // p: 64-byte aligned, read-only data
{
    q0 = __ldg(p); q1 = __ldg(p + 1); q2 = __ldg(p + 2); q3 = __ldg(p + 3);
}

// ---- repacked device-side scene records (built at upload time by rt_repack.cu) ---------------------------

// Two sibling BVH nodes in one 64-byte, 64-byte-aligned record (children are allocated adjacently by the
// reference builder, BVH.cs:161-162).  Records are numbered breadth-first per mesh so that the top of
// every tree is one contiguous range (staged in shared memory by a TMA bulk copy).
//   start: leaf  -> first triangle, global index into triGeom (triOffset already added)
//          inner -> global index of the pair record holding its two children
//   count: > 0 <=> leaf (HL:246)
struct __align__(64) NodePair
{
    float aMinX, aMinY, aMinZ, aMaxX, aMaxY, aMaxZ; int aStart, aCount;
    float bMinX, bMinY, bMinZ, bMaxX, bMaxY, bMaxZ; int bStart, bCount;
};

// Triangle geometry as the intersection test consumes it: vertex A, the two edges and the face vector
// cross(AB, AC) — each the single IEEE operation sequence of HL:190-192, evaluated once at upload
// instead of once per test (same bits).  48 bytes = 3 × float4.
// RT_TRI_PAD64 (compiled out by default): the record padded to 64 bytes, 64-byte aligned, so that a record never straddles a
// 128-byte line (a 48-byte one does in three of eight positions); costs a third more triangle bytes in L2 / HBM.
#ifdef RT_TRI_PAD64
struct __align__(64) TriGeom
{
    float ax, ay, az, abx;
    float aby, abz, acx, acy;
    float acz, nx, ny, nz;
    float pad[4];
};
#else
struct __align__(16) TriGeom
{
    float ax, ay, az, abx;
    float aby, abz, acx, acy;
    float acz, nx, ny, nz;
};
#endif
constexpr int TRI_GEOM_F4 = (int)(sizeof(TriGeom) / 16);     // float4 stride from one record to the next

// the three float4 of a TriGeom record (g points at the record)
RT_DI void ldg_trigeom(const float4* g, float4& g0, float4& g1, float4& g2)
{
    g0 = ldg_tri(g); g1 = ldg_tri(g + 1); g2 = ldg_tri(g + 2);
}

// Vertex normals, fetched only for the winning triangle of a traversal.  48 bytes = 3 × float4.
struct __align__(16) TriNormals
{
    float nax, nay, naz, nbx;
    float nby, nbz, ncx, ncy;
    float ncz, pad0, pad1, pad2;
};

// Per-model record: rows 0..2 of both matrices (all four columns kept, see mul_point/mul_dir), the root
// of its BVH, where its material lives, and a padded world-space box of the whole model.  144 bytes.
struct __align__(16) DevModel
{
    float w2l[12];      // row-major rows 0..2 of worldToLocalMatrix
    float l2w[12];      // row-major rows 0..2 of localToWorldMatrix
    int   rootStart;    // root node's start (pair index or first triangle), same encoding as NodePair
    int   rootCount;    // root node's triangleCount
    int   cullBackface; // material.flag != GLASS (HL:355)
    int   matIndex;     // index into ModelInfo (material is read from the 224-byte record)
    // Padded world-space bounds of the model (image of its root box under the inverse of worldToLocal; the padding is described at
    // buildModels, rt_repack.cuh).  A ray that misses this box, or enters it beyond the closest hit so far, cannot be changed by this model:
    // the non-instrumented kernels skip the model without transforming the ray (the reference's per-model loop, HL:347-371,
    // would traverse it and find nothing).  Placed through the inverse of worldToLocal (rt_repack.cuh); +-inf when that is singular.
    float wmin[3], wmaxx;
    float wmaxy, wmaxz; int pad[2];
};
static_assert(sizeof(DevModel) == 144, "DevModel layout");

// Counters of the SIMT interpreter's profile build (tools/simt_*_profile.py; never defined in the product build):
// [25] per-model box tests  [26] TLAS box tests  [27] TLAS walks
#if defined(RT_SIMT_PROFILE) && defined(RT_SIMT_EMU)
#define RT_DEV_PROF(i, v) simt::prof_add(i, (unsigned long long)(v))
#else
#define RT_DEV_PROF(i, v) do { } while (0)
#endif

// true when nothing inside the padded world-space box [bmin, bmax] can change the current result: the ray misses the box or
// enters it beyond bestDst (with a relative 2^-18 and an absolute 1e-6 of slack on the entry distance).  Used on a model's own
// box and on the TLAS boxes that enclose the boxes of several models.
RT_DI bool WorldBoxOutOfReach(f3 bmin, f3 bmax, f3 rayPos, f3 rayInv, float bestDst)
{
    const f3 tMin = (bmin - rayPos) * rayInv;
    const f3 tMax = (bmax - rayPos) * rayInv;
    const float tNear = fmaxf(fmaxf(fminf(tMin.x, tMax.x), fminf(tMin.y, tMax.y)), fminf(tMin.z, tMax.z));
    const float tFar  = fminf(fminf(fmaxf(tMin.x, tMax.x), fmaxf(tMin.y, tMax.y)), fmaxf(tMin.z, tMax.z));
    const bool hit = tFar >= tNear && tFar > 0.0f;
    return !hit || (tNear * 0.99999619f - 1e-6f) > bestDst;
}

// true when model record `mr` cannot change the current result (its padded world box, DevModel::wmin .. wmaxz)
RT_DI bool ModelOutOfReach(const float4* __restrict__ mr, f3 rayPos, f3 rayInv, float bestDst)
{
    RT_DEV_PROF(25, 1);
    const float4 b0 = __ldg(mr + 7), b1 = __ldg(mr + 8);
    return WorldBoxOutOfReach(make_f3(b0.x, b0.y, b0.z), make_f3(b0.w, b1.x, b1.y), rayPos, rayInv, bestDst);
}

// Sphere with r*r precomputed (the exact product of HL:299).  32 bytes.
struct __align__(16) DevSphere
{
    float cx, cy, cz, radius;
    float r2; int pad0, pad1, pad2;
};

// ---- kernel parameter block (uniform names as in HL:5-21, RC:7-8) ---------------------------------------------

constexpr int RT_MAX_PEERS = 7;
constexpr int RT_MAX_BVH_DEPTH = 63;                     // levels of inner nodes a Nodes buffer may have: every traversal stack holds 64 entries (rtDispatch rejects deeper trees)

struct DevParams
{
    int   MaxBounceCount, NumRaysPerPixel, Frame, renderSeed;
    int   UseSky, modelCount, sphereCount, accumulate;
    float DefocusStrength, DivergeStrength, SunFocus, SunIntensity;
    float ViewParams[3]; float pad0;
    float SunColour[3];  float pad1;
    float dirToSun[3];   float pad2;
    float cam[16];                          // CamLocalToWorldMatrix, column-major
    unsigned int W, H;                      // Resolution
    unsigned int limX, limY;                // pixels covered by the dispatched 8x8 groups
    int   tileRank, tileWorld, bandRows, countStats;

    // reference-layout buffers (what the host uploaded)
    const RtNode*     Nodes;
    const RtTriangle* Triangles;
    const RtModel*    ModelInfo;
    const RtSphere*   Spheres;
    // repacked buffers
    const NodePair*   pairs;
    const TriGeom*    triGeom;
    const TriNormals* triNormals;
    const DevModel*   models;
    const DevSphere*  spheres;
    // sphere accelerator (only when the Spheres buffer is large): pair records over padded sphere boxes + the spheres in
    // leaf order (pad1 = index in the Spheres buffer)
    const NodePair*   sphPairs;
    const DevSphere*  sphLeaves;
    int   sphBvh, sphRootStart, sphRootCount;
    int   zeroDefocus;                      // host: DefocusStrength == 0 and adding +-0 to the camera origin cannot change a bit of it (RT_SKIP_ZERO_DEFOCUS builds)
    int   smemPairs;                        // number of leading pair records staged in shared memory
    int   tailLanes;                        // pooled kernel: leave the trace phase when this few lanes are still tracing
    int   sortRays;                         // pooled kernel: group the ray queue by direction octant
    int   gridFit;                          // host only: size the persistent grid so that every lane gets a whole number of pixels

    float4* FrameRender;
    float4* AccumulatedRender;
    // fused tile exchange: the same images on the other GPUs of the job (CUDA-IPC mapped peer memory over NVLink);
    // a finished pixel is stored straight into every peer's images by the kernel that produced it
    float4* peerFrame[RT_MAX_PEERS];
    float4* peerAccum[RT_MAX_PEERS];
    int   nPeers;
    int   modelSkip;                        // skip models whose padded world box the ray cannot reach (exact; default on)
    int   frames;                           // rtDispatchFrames: frames Frame .. Frame + frames - 1 of every pixel in one launch (only the FRAMES kernels read it)
    int   forceExt;                         // testing: run the <EXT = true> instantiation although no extension is active
    unsigned long long* counters;           // [0] rays [1] boxTests [2] triTests [3] sphereTests [4] sphere-accelerator box tests
    unsigned int* workCounter;              // persistent kernel: next job
    // TLAS over the models' padded world boxes (many-model scenes; only the <TLAS> kernels read these — appended so that the
    // parameter offsets of everything above stay where they were)
    const NodePair* tlasPairs;              // inner records: two child boxes each; count > 0 <=> leaf, start -> tlasLeaves
    const int*      tlasLeaves;             // model indices in leaf order
    int   tlas, tlasRootStart, tlasRootCount, pad8;
    // kernel 1 on small tiles: a pixel's samples in `chunks` consecutive jobs (1 = whole pixels); the RNG state and the running sum travel
    // from one chunk to the next through `handoff`: four 64-bit words per pixel job, each {tag, value} with tag = chunkSerial << 8 | chunks
    // completed, so that every word validates itself (aligned 8-byte stores are single-copy atomic: no fence, no flag)
    // rtDispatchAdaptive's kernel-1 list instantiations (never chunked) take their pixel list in the same slot, and the moments in
    // poolCold's (kernel 2 only): the slots keep the parameter layout, and wave_body's signature, of every existing kernel
    int   chunks, chunkSerial;
    union { unsigned long long* handoff; const unsigned int* pixelList; };
    // "countStats" launches: the W*H per-pixel counters ([y][x], RtPixelStats).  Only the instrumented code reads it (kept at the
    // offset of a retired pointer so that the parameter layout of every kernel stays where it was)
    RtPixelStats* pixelStats;
    union { float* poolCold; float4* adaptiveMoments; };   // kernel 2 built with RT_POOL_COLD_GLOBAL: the per-warp blocks of the slot fields kept out of shared memory
};

struct Counters { unsigned int rays, box, tri, sph, sbox; };

// What a camera-kernel launch renders: one frame of the region (rtDispatch), P.frames frames of it (rtDispatchFrames) or the pixels of a
// list (rtDispatchAdaptive).  Every kernel family has kernels of its own for each form.
enum CameraForm { FORM_PLAIN, FORM_FRAMES, FORM_LIST };

// Instrumented launches: add one pixel's share of the counters (`now` - `before`, all of it by the lane that traced it) into its
// PixelStats record.  Relaxed atomics: several lanes may add to one pixel in the same launch (sample chunks, the pooled kernel's
// rays of one pixel traced by different lanes); the sums are order-independent and wrap modulo 2^32.
RT_DI void AddPixelStats(const DevParams& P, size_t o, const Counters& now, const Counters& before)
{
    unsigned int* r = reinterpret_cast<unsigned int*>(P.pixelStats + o);
    atomicAdd(r + 0, now.rays - before.rays);
    atomicAdd(r + 1, now.box - before.box);
    atomicAdd(r + 2, now.tri - before.tri);
    atomicAdd(r + 3, now.sph - before.sph);
    atomicAdd(r + 4, now.sbox - before.sbox);
}

// RC:18-23: write the pixel of this frame and accumulate; with peers, also store both values into every peer GPU's copy
// (the all-gather of finished tiles fused into the producing kernel: 32 bytes per pixel per peer over NVLink).
// EXT = the launch has peers (or another extension) — the common single-GPU instantiation carries no trace of them.
// ADAPTIVE = the list-driven kernels of rtDispatchAdaptive: the accumulating write also adds the frame's luminance to the pixel's
// moments (s1 + l, s2 + l*l, n + 1) in `moments` (AdaptiveMoments; the call is refused without accumulation).
template <bool EXT, bool ADAPTIVE = false>
__device__ __forceinline__ void WritePixel(const DevParams& P, size_t o, float r, float g, float b, float4* moments = nullptr)
{
    if constexpr (ADAPTIVE)
    {
        const float l = (0.2126f * r + 0.7152f * g) + 0.0722f * b;
        float4 m = moments[o];
        m.x += l; m.y += l * l; m.z += 1.0f;
        moments[o] = m;
    }
    const float4 f = make_float4(r, g, b, 1.0f);
    float4 a = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
#if defined(RT_STREAM_IMAGES) && !defined(RT_SIMT_EMU)
    // the two render targets are touched once per pixel per frame (48 bytes) and never again by this launch: streaming loads / stores
    // (evict-first) keep them from displacing node and triangle records in L2 (4096 x 4096: 2 x 268 MB against 50 MB of L2)
    __stcs(&P.FrameRender[o], f);
    if (P.accumulate)
    {
        a = __ldcs(&P.AccumulatedRender[o]);
        a.x += r; a.y += g; a.z += b; a.w += 1.0f;
        __stcs(&P.AccumulatedRender[o], a);
    }
#else
    P.FrameRender[o] = f;
    if (P.accumulate)
    {
        a = P.AccumulatedRender[o];
        a.x += r; a.y += g; a.z += b; a.w += 1.0f;
        P.AccumulatedRender[o] = a;
    }
#endif
    if (EXT)
    {
        for (int k = 0; k < P.nPeers; k++)
        {
            P.peerFrame[k][o] = f;
            if (P.accumulate) P.peerAccum[k][o] = a;
        }
    }
}

// ---- RNG (HL:127-164) ---------------------------------------------------------------------------------------------

RT_DI uint32_t NextRandom(uint32_t& state)
{
    state = state * 747796405u + 2891336453u;
    uint32_t result = ((state >> ((state >> 28) + 4u)) ^ state) * 277803737u;
    result = (result >> 22) ^ result;
    return result;
}
// HL:137 divides by the float literal 4294967295.0 == 2^32 in FP32: an exact scaling
RT_DI float RandomValue(uint32_t& state) { return __uint2float_rn(NextRandom(state)) * 2.3283064365386963e-10f; }

RT_DI float RandomValueNormalDistribution(uint32_t& state)
{
    const float theta = 6.2831852f * RandomValue(state);             // 2 * 3.1415926 (HL:144)
    const float rho = sqrtf(-2.0f * log_rt(RandomValue(state)));
    return rho * cos_rt(theta);
}
RT_DI f3 RandomDirection(uint32_t& state)
{
    const float x = RandomValueNormalDistribution(state);
    const float y = RandomValueNormalDistribution(state);
    const float z = RandomValueNormalDistribution(state);
    return normalize3(make_f3(x, y, z));
}
// (not inlined: two call sites per camera sample; keeping one copy shrinks the kernels' instruction footprint)
RT_DNI f2 RandomPointInCircle(uint32_t& state)
{
    const float angle = (RandomValue(state) * 2.0f) * 3.1415f;       // PI = 3.1415 (HL:2,161)
    float s, c; sincos_rt(angle, s, c);
    const float rad = sqrtf(RandomValue(state));
    return make_f2(c * rad, s * rad);
}

// ---- environment (HL:167-183) -----------------------------------------------------------------------------------

// (not inlined: two pow() bodies that only sky scenes execute, on miss)
RT_DNI f3 GetEnvironmentLight(const DevParams& P, f3 dir)
{
    if (P.UseSky == 0) return splat3(0.0f);
    const f3 GroundColour = make_f3(0.35f, 0.3f, 0.35f);
    const f3 SkyColourHorizon = make_f3(1.0f, 1.0f, 1.0f);
    const f3 SkyColourZenith = make_f3(0.08f, 0.37f, 0.73f);
    const float skyGradientT = pow_rt(smoothstep1(0.0f, 0.4f, dir.y), 0.35f);
    const float groundToSkyT = smoothstep1(-0.01f, 0.0f, dir.y);
    const f3 skyGradient = lerp3(SkyColourHorizon, SkyColourZenith, skyGradientT);
    const float s = 1000.0f / P.SunFocus;
    const float sun = pow_rt(fmaxf(0.0f, dot3(dir, load3(P.dirToSun))), s) * P.SunIntensity;
    return lerp3(GroundColour, skyGradient, groundToSkyT) + (sun * load3(P.SunColour)) * (groundToSkyT >= 1.0f ? 1.0f : 0.0f);
}

// ---- matrix · vector, all four products kept and summed left to right (HL:351-352,367,547,556) ------------

RT_DI f3 mul_cm(const float* m, f3 v, float w)      // column-major 4x4, rows 0..2
{
    return make_f3(((m[0] * v.x + m[4] * v.y) + m[8]  * v.z) + m[12] * w,
                   ((m[1] * v.x + m[5] * v.y) + m[9]  * v.z) + m[13] * w,
                   ((m[2] * v.x + m[6] * v.y) + m[10] * v.z) + m[14] * w);
}
RT_DI f3 mul_rm(const float* r, f3 v, float w)      // row-major rows 0..2 (DevModel)
{
    return make_f3(((r[0] * v.x + r[1] * v.y) + r[2]  * v.z) + r[3]  * w,
                   ((r[4] * v.x + r[5] * v.y) + r[6]  * v.z) + r[7]  * w,
                   ((r[8] * v.x + r[9] * v.y) + r[10] * v.z) + r[11] * w);
}

// ---- primitive tests ---------------------------------------------------------------------------------------------------

// HL:219-231
RT_DI float RayBoundingBoxDst(f3 pos, f3 invDir, f3 boxMin, f3 boxMax)
{
    const f3 tMin = (boxMin - pos) * invDir;
    const f3 tMax = (boxMax - pos) * invDir;
    const float tNear = fmaxf(fmaxf(fminf(tMin.x, tMax.x), fminf(tMin.y, tMax.y)), fminf(tMin.z, tMax.z));
    const float tFar  = fminf(fminf(fmaxf(tMin.x, tMax.x), fmaxf(tMin.y, tMax.y)), fmaxf(tMin.z, tMax.z));
    const bool hit = tFar >= tNear && tFar > 0.0f;
    return hit ? (tNear > 0.0f ? tNear : 0.0f) : inf32();
}

// HL:188-207 without the normal (evaluated later for the winner only): returns didHit, writes dst,u,v,det
RT_DI bool RayTriangleCore(f3 pos, f3 dir, f3 A, f3 edgeAB, f3 edgeAC, f3 triFaceVector, bool cullBackface,
                           float& dst, float& u, float& v, float& determinant)
{
    const f3 vertRayOffset = pos - A;
    const f3 rayOffsetPerp = cross3(vertRayOffset, dir);
    determinant = -dot3(dir, triFaceVector);
    const float invDet = 1.0f / determinant;
    dst = dot3(vertRayOffset, triFaceVector) * invDet;
    u = dot3(edgeAC, rayOffsetPerp) * invDet;
    v = -dot3(edgeAB, rayOffsetPerp) * invDet;
    const float w = (1.0f - u) - v;
    const bool keep = cullBackface ? determinant >= 1E-8f : fabsf(determinant) >= 1E-8f;
    return keep && dst > 0.0f && u >= 0.0f && v >= 0.0f && w >= 0.0f;
}
// HL:208-209
RT_DI f3 TriangleSmoothNormal(f3 nA, f3 nB, f3 nC, float u, float v, float determinant)
{
    const float w = (1.0f - u) - v;
    const f3 smoothNormal = normalize3((nA * w + nB * u) + nC * v);
    return smoothNormal * sign1(determinant);
}

// HL:289-320 (sphere extension): returns didHit; dst / isInside valid on hit.
// Same values as the reference's expressions; the two divisions are only evaluated when their result is used:
//   dstFar >= 0  <=>  (-b + s) >= 0  whenever 2a > 0 (an IEEE quotient has the sign of its numerator, and -0 >= 0 holds
//   for both), so a sphere behind the ray is rejected without dividing; dstFar itself is needed only from inside.
RT_DI bool RaySphereCore(f3 rayPos, f3 rayDir, f3 centre, float r2, float& dst, bool& isInside)
{
    const f3 offsetRayOrigin = rayPos - centre;
    const float a = dot3(rayDir, rayDir);
    const float b = 2.0f * dot3(offsetRayOrigin, rayDir);
    const float c = dot3(offsetRayOrigin, offsetRayOrigin) - r2;
    const float discriminant = b * b - (4.0f * a) * c;
    if (discriminant >= 0.0f)
    {
#ifdef RT_SPHERE_SKIP_SQRT
        // Experimental (off by default; slower on the Cornell box): a sphere the ray is moving away from (b > 0) is hit only if
        // sqrt(disc) >= b.  With bb = fl(b*b) in b^2 (1 +- 2^-24):  disc < bb (1 - 2^-21)  =>  disc < b^2 (1 - 2^-22)  =>
        // sqrt_rn(disc) < b  =>  -b + s < 0  =>  the reference's dstFar < 0  =>  no hit.  Saves the sqrt; never changes an answer.
        {
            const float den0 = 2.0f * a;
            if (b > 0.0f && den0 > 0.0f && den0 < inf32() && discriminant < (b * b) * 0.99999952f) return false;
        }
#endif
        const float s = sqrtf(discriminant);
        const float den = 2.0f * a;
        const float numFar = -b + s;
        // dstFar >= 0  <=>  numFar >= 0 for a positive denominator (an IEEE quotient has the sign of its numerator, -0 >= 0
        // holds for both, inf/inf cannot occur for a finite den): spheres behind the ray are rejected without dividing
#ifndef RT_SPHERE_INLINE_DIV     // keeping the two rare divisions behind a call was faster on config 2
        const bool farOk = (den > 0.0f && den < inf32()) ? (numFar >= 0.0f) : (div_cold(numFar, den) >= 0.0f);
        if (farOk)
        {
            const float dstNear = fmaxf(0.0f, (-b - s) / den);
            isInside = dstNear == 0.0f;
            dst = dstNear;
            if (isInside) dst = div_cold(numFar, den);      // only from inside a sphere (glass interiors)
            return true;
        }
#else
        const bool farOk = (den > 0.0f && den < inf32()) ? (numFar >= 0.0f) : ((numFar / den) >= 0.0f);
        if (farOk)
        {
            const float dstNear = fmaxf(0.0f, (-b - s) / den);
            isInside = dstNear == 0.0f;
            dst = isInside ? (numFar / den) : dstNear;
            return true;
        }
#endif
    }
    return false;
}

// Closest sphere of a LARGE Spheres buffer through a BVH over padded sphere boxes, with the reference's semantics: the
// result is the sphere a front-to-back linear scan with strict `<` would keep (HL:341 extended to a buffer) — the smallest
// dst, and among equal dst the smallest buffer index.  Every sphere that is tested is tested with RaySphereCore, so dst is
// the reference's value; the tree only decides which spheres can be skipped, and it is conservative:
//   * boxes are padded (rt_repack.cuh) by more than the reference's own rounding error can move a computed hit point, so
//     a computed hit point always lies inside its sphere's box;
//   * a box is skipped only if its entry distance, reduced by a relative 2^-18 and an absolute 1e-6, still exceeds the best
//     dst so far (strictly), so equal-distance candidates with a smaller index are never lost.
// The walk keeps RT_SPHERE_STACK entries; the host limits the tree's depth to fit (sphereSahDepth, rt_repack.cuh), so the guard on
// the push below never drops an entry.
constexpr int RT_SPHERE_STACK = 48;

RT_DNI void TraverseSpheres(const DevParams& P, f3 rayPos, f3 rayDir, float& bestDst, int& bestIndex, bool& bestInside, int& bestFlag,
                           Counters& cnt, bool countStats)
{
    const f3 invDir = rcp3(rayDir);
    int2 stack[RT_SPHERE_STACK];
    int stackCount = 0;
    int2 cur = make_int2(P.sphRootStart, P.sphRootCount);
    for (;;)
    {
        if (cur.y > 0)
        {
            for (int i = 0; i < cur.y; i++)
            {
                const float4* q = reinterpret_cast<const float4*>(P.sphLeaves + cur.x + i);
                const float4 s0 = __ldg(q);
                const float4 s1 = __ldg(q + 1);
                float dst; bool inside;
                if (countStats) cnt.sph++;
                if (RaySphereCore(rayPos, rayDir, make_f3(s0.x, s0.y, s0.z), s1.x, dst, inside))
                {
                    const int orig = __float_as_int(s1.z);
                    if (dst < bestDst || (dst == bestDst && orig < bestIndex))
                    {
                        bestDst = dst; bestIndex = orig; bestInside = inside; bestFlag = __float_as_int(s1.y);
                    }
                }
            }
            if (stackCount == 0) return;
            cur = stack[--stackCount];
        }
        else
        {
            const float4* p = reinterpret_cast<const float4*>(P.sphPairs + cur.x);
            const float4 q0 = __ldg(p), q1 = __ldg(p + 1), q2 = __ldg(p + 2), q3 = __ldg(p + 3);
            const float dA = RayBoundingBoxDst(rayPos, invDir, make_f3(q0.x, q0.y, q0.z), make_f3(q0.w, q1.x, q1.y));
            const float dB = RayBoundingBoxDst(rayPos, invDir, make_f3(q2.x, q2.y, q2.z), make_f3(q2.w, q3.x, q3.y));
            if (countStats) cnt.sbox += 2;
            const bool nearA = dA <= dB;
            const float dNear = nearA ? dA : dB, dFar = nearA ? dB : dA;
            const int2 a = make_int2(__float_as_int(q1.z), __float_as_int(q1.w)), b = make_int2(__float_as_int(q3.z), __float_as_int(q3.w));
            const int2 nearRef = nearA ? a : b, farRef = nearA ? b : a;
            if (dFar < inf32() && (dFar * 0.99999619f - 1e-6f) <= bestDst && stackCount < RT_SPHERE_STACK) stack[stackCount++] = farRef;
            if (dNear < inf32() && (dNear * 0.99999619f - 1e-6f) <= bestDst) cur = nearRef;
            else { if (stackCount == 0) return; cur = stack[--stackCount]; }
        }
    }
}

// ---- TLAS over the models (SURVEY 8f #3; many-model scenes) ------------------------------------------------------------------
// The reference walks every Model for every ray segment, in buffer order, with one running result (HL:347-371).  Exactness pins
// the ORDER in which models are processed (a model's traversal is culled against the result of the models before it), so the
// TLAS does not reorder anything: one walk per ray segment marks, in a bit mask, the models whose padded world box the ray can
// reach before its current best hit; the model loop then visits the marked models in ascending buffer index and repeats the
// per-model test (ModelOutOfReach) against the result as it stands by then.  A model is therefore skipped only if its own box
// test — or the same test on a TLAS box that encloses its box — fails, and either means its traversal could not have changed
// the result (DESIGN.md section 5, "Models a ray cannot reach are skipped").  Whatever the walk cannot decide (stack full)
// it marks, so the mask is always a superset of what the linear test would keep at the same bestDst.
constexpr int RT_TLAS_MAX_MODELS = 4096;                 // mask words per lane = 128 (local memory, touched only up to modelCount / 32)
constexpr int RT_TLAS_WORDS = RT_TLAS_MAX_MODELS / 32;
constexpr int RT_TLAS_STACK = 24;                        // median-split tree over <= 4096 models: depth <= 12

RT_DNI void TlasCollect(const DevParams& P, f3 rayPos, f3 rayInv, float bestDst, unsigned int* __restrict__ mask)
{
    const int words = (P.modelCount + 31) >> 5;
    for (int w = 0; w < words; w++) mask[w] = 0u;
    int2 stack[RT_TLAS_STACK];
    int stackCount = 0;
    int2 cur = make_int2(P.tlasRootStart, P.tlasRootCount);
    RT_DEV_PROF(27, 1);
    for (;;)
    {
        if (cur.y > 0)
        {
            for (int k = 0; k < cur.y; k++) { const int m = __ldg(P.tlasLeaves + cur.x + k); mask[m >> 5] |= 1u << (m & 31); }
            if (stackCount == 0) return;
            cur = stack[--stackCount];
        }
        else
        {
            const float4* p = reinterpret_cast<const float4*>(P.tlasPairs + cur.x);
            const float4 q0 = __ldg(p), q1 = __ldg(p + 1), q2 = __ldg(p + 2), q3 = __ldg(p + 3);
            RT_DEV_PROF(26, 2);
            const bool skipA = WorldBoxOutOfReach(make_f3(q0.x, q0.y, q0.z), make_f3(q0.w, q1.x, q1.y), rayPos, rayInv, bestDst);
            const bool skipB = WorldBoxOutOfReach(make_f3(q2.x, q2.y, q2.z), make_f3(q2.w, q3.x, q3.y), rayPos, rayInv, bestDst);
            const int2 a = make_int2(__float_as_int(q1.z), __float_as_int(q1.w)), b = make_int2(__float_as_int(q3.z), __float_as_int(q3.w));
            if (!skipA && !skipB)
            {
                if (stackCount == RT_TLAS_STACK) { for (int w = 0; w < words; w++) mask[w] = 0xffffffffu; return; }   // cannot happen with the host's tree; stay conservative
                stack[stackCount++] = b; cur = a;
            }
            else if (!skipA) cur = a;
            else if (!skipB) cur = b;
            else { if (stackCount == 0) return; cur = stack[--stackCount]; }
        }
    }
}

// smallest marked model index >= from, or modelCount
RT_DI int TlasNext(const unsigned int* __restrict__ mask, int from, int modelCount)
{
    const int words = (modelCount + 31) >> 5;
    int w = from >> 5;
    if (from >= modelCount || w >= words) return modelCount;
    unsigned int bits = mask[w] & (0xffffffffu << (from & 31));
    while (bits == 0u) { if (++w >= words) return modelCount; bits = mask[w]; }
    const int m = (w << 5) + __ffs((int)bits) - 1;
    return m < modelCount ? m : modelCount;
}

// ---- hit record -----------------------------------------------------------------------------------------------------------

struct Hit
{
    float dst;                 // +inf = miss
    bool  isBackface;
    f3    normal;
    f3    pos;
    const RtMaterial* material;
};

// ---- shading (HL:383-466, 497-538) -----------------------------------------------------------------------------------

RT_DI float CalculateReflectance(f3 inDir, f3 normal, float iorA, float iorB)
{
    const float refractRatio = iorA / iorB;
    const float cosAngleIn = -dot3(inDir, normal);
    const float sinSqrAngleOfRefraction = (refractRatio * refractRatio) * (1.0f - cosAngleIn * cosAngleIn);
    if (sinSqrAngleOfRefraction >= 1.0f) return 1.0f;
    const float cosAngleOfRefraction = sqrtf(1.0f - sinSqrAngleOfRefraction);
    const float denominatorPerpendicular = iorA * cosAngleIn + iorB * cosAngleOfRefraction;
    const float denominatorParallel = iorA * cosAngleIn + iorB * cosAngleOfRefraction;   // as in the reference (HL:392)
    if (fminf(denominatorPerpendicular, denominatorParallel) < 1E-8f) return 1.0f;
    float rPerpendicular = (iorA * cosAngleIn - iorB * cosAngleOfRefraction) / denominatorPerpendicular;
    rPerpendicular *= rPerpendicular;
    float rParallel = (iorB * cosAngleIn - iorA * cosAngleOfRefraction) / denominatorParallel;
    rParallel *= rParallel;
    return (rPerpendicular + rParallel) / 2.0f;
}
RT_DI f3 Refract(f3 inDir, f3 normal, float iorA, float iorB)
{
    const float refractRatio = iorA / iorB;
    const float cosAngleIn = -dot3(inDir, normal);
    const float sinSqrAngleOfRefraction = (refractRatio * refractRatio) * (1.0f - cosAngleIn * cosAngleIn);
    if (sinSqrAngleOfRefraction > 1.0f) return splat3(0.0f);
    return refractRatio * inDir + (refractRatio * cosAngleIn - sqrtf(1.0f - sinSqrAngleOfRefraction)) * normal;
}
RT_DI f3 Reflect(f3 inDir, f3 normal) { return inDir - (2.0f * dot3(inDir, normal)) * normal; }

RT_DI f3 GetMaterialColour(const RtMaterial* mat, f3 pos, f3 normal, bool isSpecularBounce)
{
    f3 col = make_f3(mat->diffuseCol[0], mat->diffuseCol[1], mat->diffuseCol[2]);
    if (mat->flag == RT_MATERIAL_CHECKERED)
    {
        f2 checkerPoint = make_f2(pos.x, pos.z);
        if (fabsf(normal.x) > fabsf(normal.y)) checkerPoint = make_f2(pos.z, pos.y);
        if (fabsf(normal.z) > fmaxf(fabsf(normal.x), fabsf(normal.y))) checkerPoint = make_f2(pos.x, pos.y);
        checkerPoint.x = checkerPoint.x * 1.5f; checkerPoint.y = checkerPoint.y * 1.5f;
        const float fx = floorf(checkerPoint.x), fy = floorf(checkerPoint.y);
        const float cx = fx - 2.0f * floorf(fx / 2.0f);
        const float cy = fy - 2.0f * floorf(fy / 2.0f);
        if (!(cx == cy)) col = make_f3(mat->emissionCol[0], mat->emissionCol[1], mat->emissionCol[2]);
    }
    return lerp3(col, make_f3(mat->specularCol[0], mat->specularCol[1], mat->specularCol[2]), isSpecularBounce ? 1.0f : 0.0f);
}

// exp of three components (not inlined: glass back-face hits only)
RT_DNI f3 exp3_rt(f3 a) { return make_f3(exp_rt(a.x), exp_rt(a.y), exp_rt(a.z)); }

struct PathState
{
    f3 pos, dir, transmittance, totalLight;
};

#ifdef RT_GLASS_OUT_OF_LINE
// Compiled out by default (slower on the Cornell box and the mesh scenes): the glass branch of ShadeSegment (HL:499-518) as one out-of-line function.  Three of 32
// lanes take it on config 2; inlined it is ~150 instructions of the per-iteration footprint, and instruction fetch is a fifth of the
// stall cycles of that issue-bound kernel.  Same operations in the same order.
RT_DNI void ShadeGlass(const RtMaterial* material, float hitDst, bool isBackface, f3 normal, f3 hitPos, f3 diffuseDir, float v7, PathState& ray)
{
    if (isBackface)
    {
        const f3 absorb = ((-hitDst) * make_f3(material->absorption[0], material->absorption[1], material->absorption[2])) * material->absorptionStrength;
        ray.transmittance = ray.transmittance * exp3_rt(absorb);
    }
    const float iorCurrent = isBackface ? material->ior : 1.0f;
    const float iorNext = isBackface ? 1.0f : material->ior;
    f3 reflectDir = Reflect(ray.dir, normal);
    f3 refractDir = Refract(ray.dir, normal, iorCurrent, iorNext);
    const float reflectWeight = CalculateReflectance(ray.dir, normal, iorCurrent, iorNext);
    reflectDir = normalize3(lerp3(diffuseDir, reflectDir, material->specularProbability));
    refractDir = normalize3(lerp3(-diffuseDir, refractDir, material->smoothness));
    const bool followReflection = v7 <= reflectWeight;
    ray.dir = followReflection ? reflectDir : refractDir;
    ray.pos = hitPos + (0.001f * normal) * sign1(dot3(normal, ray.dir));
}
#endif

// One iteration of the bounce loop after the intersection (HL:488-538).
// Returns true when the path continues with another segment.
//
// Both material branches consume seven draws before the roulette draw, in a different order (Appendix A of SURVEY.md):
//   glass     : RandomDirection (draws 1-6), reflect-vs-refract test (draw 7)
//   otherwise : specular test (draw 1), RandomDirection (draws 2-7)
// The seven values are drawn once and the Box-Muller / normalize work of RandomDirection — the most expensive part of
// shading — is evaluated once on the selected six, instead of once per divergent branch.  Same values, same order.
RT_DI bool ShadeSegment(const DevParams& P, const Hit& hit, PathState& ray, uint32_t& rngState)
{
    const float epsilon = 0.001f;
    if (!(hit.dst < inf32()))
    {
        if (P.UseSky) ray.totalLight = ray.totalLight + ray.transmittance * GetEnvironmentLight(P, ray.dir);
        return false;
    }
    const RtMaterial* material = hit.material;
    const bool isGlass = material->flag == RT_MATERIAL_GLASS;

    const float v1 = RandomValue(rngState), v2 = RandomValue(rngState), v3 = RandomValue(rngState), v4 = RandomValue(rngState);
    const float v5 = RandomValue(rngState), v6 = RandomValue(rngState), v7 = RandomValue(rngState);
    // RandomDirection (HL:141-157): component k uses (theta draw, rho draw) = consecutive pairs
    const float tx = isGlass ? v1 : v2, rx = isGlass ? v2 : v3;
    const float ty = isGlass ? v3 : v4, ry = isGlass ? v4 : v5;
    const float tz = isGlass ? v5 : v6, rz = isGlass ? v6 : v7;
    // three independent log / sqrt / cos chains (the unrolled form beat a rolled loop, ILP > instruction footprint)
    float nx = 0.0f, ny = 0.0f, nz = 0.0f;
#ifdef RT_RANDDIR_LOOP
#pragma unroll 1
#else
#pragma unroll
#endif
    for (int k = 0; k < 3; k++)
    {
        const float t = k == 0 ? tx : (k == 1 ? ty : tz);
        const float r = k == 0 ? rx : (k == 1 ? ry : rz);
        const float val = sqrtf(-2.0f * log_rt(r)) * cos_rt(6.2831852f * t);
        if (k == 0) nx = val; else if (k == 1) ny = val; else nz = val;
    }
    const f3 randomDirection = normalize3(make_f3(nx, ny, nz));
    const f3 diffuseDir = normalize3(hit.normal + randomDirection);

    if (isGlass)
    {
#ifdef RT_GLASS_OUT_OF_LINE
        ShadeGlass(material, hit.dst, hit.isBackface, hit.normal, hit.pos, diffuseDir, v7, ray);
#else
        if (hit.isBackface)
        {
            const f3 absorb = ((-hit.dst) * make_f3(material->absorption[0], material->absorption[1], material->absorption[2])) * material->absorptionStrength;
            ray.transmittance = ray.transmittance * exp3_rt(absorb);
        }
        const float iorCurrent = hit.isBackface ? material->ior : 1.0f;
        const float iorNext = hit.isBackface ? 1.0f : material->ior;
        f3 reflectDir = Reflect(ray.dir, hit.normal);
        f3 refractDir = Refract(ray.dir, hit.normal, iorCurrent, iorNext);
        const float reflectWeight = CalculateReflectance(ray.dir, hit.normal, iorCurrent, iorNext);

        reflectDir = normalize3(lerp3(diffuseDir, reflectDir, material->specularProbability));
        refractDir = normalize3(lerp3(-diffuseDir, refractDir, material->smoothness));

        const bool followReflection = v7 <= reflectWeight;
        ray.dir = followReflection ? reflectDir : refractDir;
        ray.pos = hit.pos + (epsilon * hit.normal) * sign1(dot3(hit.normal, ray.dir));
#endif
    }
    else
    {
        const bool isSpecularBounce = material->specularProbability >= v1;
        ray.pos = hit.pos + (hit.normal * epsilon);
        const f3 specularDir = reflect3(ray.dir, hit.normal);
        ray.dir = normalize3(lerp3(diffuseDir, specularDir, material->smoothness * (isSpecularBounce ? 1.0f : 0.0f)));

        const f3 emittedLight = make_f3(material->emissionCol[0], material->emissionCol[1], material->emissionCol[2]) * material->emissionStrength;
        ray.totalLight = ray.totalLight + emittedLight * ray.transmittance;
        ray.transmittance = ray.transmittance * GetMaterialColour(material, hit.pos, hit.normal, isSpecularBounce);
    }
    const float p = fmaxf(ray.transmittance.x, fmaxf(ray.transmittance.y, ray.transmittance.z));
    if (RandomValue(rngState) >= p) return false;
    ray.transmittance = ray.transmittance * (1.0f / p);
    return true;
}

// ---- display (Display.shader:42-47 + sRGB back buffer) -------------------------------------------------------------------
RT_DI unsigned int DisplayEncode(float v)
{
    // NaN -> 0; clamp; IEC 61966-2-1 transfer function with the pinned pow; round to nearest
    if (!(v > 0.0f)) return 0u;
    if (v > 1.0f) v = 1.0f;
    const float e = v <= 0.0031308f ? 12.92f * v : 1.055f * pow_rt(v, 0.41666666f) - 0.055f;
    return __float2uint_rz(fminf(fmaxf(e, 0.0f), 1.0f) * 255.0f + 0.5f);
}

// ---- camera (HL:545-576) --------------------------------------------------------------------------------------------------

struct PixelSetup
{
    f3 camOrigin, focusPoint, camRight, camUp;
    uint32_t rngState;
};

// Per-pixel constants and the RNG seed for thread id (x, y)  (RC:15, HL:547-558)
RT_DI PixelSetup SetupPixel(const DevParams& P, unsigned int idx, unsigned int idy)
{
    PixelSetup s;
    const float uvx = __uint2float_rn(idx) / (__uint2float_rn(P.W) - 1.0f);
    const float uvy = __uint2float_rn(idy) / (__uint2float_rn(P.H) - 1.0f);
    s.camOrigin = mul_cm(P.cam, make_f3(0.0f, 0.0f, 0.0f), 1.0f);
    const uint32_t pixelCoordX = __float2uint_rz(uvx * __uint2float_rn(P.W));
    const uint32_t pixelCoordY = __float2uint_rz(uvy * __uint2float_rn(P.H));
    const uint32_t pixelIndex = pixelCoordY * P.W + pixelCoordX;
    s.rngState = pixelIndex + (uint32_t)P.Frame * 719393u + (uint32_t)P.renderSeed;
    const f3 focusPointLocal = make_f3(uvx - 0.5f, uvy - 0.5f, 1.0f) * load3(P.ViewParams);
    s.focusPoint = mul_cm(P.cam, focusPointLocal, 1.0f);
    s.camRight = make_f3(P.cam[0], P.cam[1], P.cam[2]);
    s.camUp = make_f3(P.cam[4], P.cam[5], P.cam[6]);
    return s;
}

// Seed of frame Frame + k of the pixel whose frame-Frame seed is `seed` (HL:552: the frame enters as Frame * 719393, modulo 2^32)
RT_DI uint32_t FrameSeed(uint32_t seed, unsigned int k) { return seed + k * 719393u; }

// One camera sample (HL:567-576): consumes four draws, returns the path's initial state
RT_DI void GenerateCameraRay(const DevParams& P, const PixelSetup& s, uint32_t& rngState, PathState& ray)
{
    const float numPixelsX = __uint2float_rn(P.W);
#ifdef RT_SKIP_ZERO_DEFOCUS
    // Compiled out by default (it was slower): with DefocusStrength == 0 — every shipped scene but one — the defocus jitter is
    // (finite * +-0) / W = +-0 and origin + camRight * +-0 + camUp * +-0 is the origin bit for bit as long as no origin component is
    // itself a zero (whose sign could flip) and the camera axes are finite; the host checks that once per dispatch.  The two random
    // numbers are still drawn (the stream must advance), only the sine, cosine, square root and two IEEE divisions are not evaluated.
    f3 rayOrigin;
    if (P.zeroDefocus) { NextRandom(rngState); NextRandom(rngState); rayOrigin = s.camOrigin; }
    else
    {
        const f2 c0 = RandomPointInCircle(rngState);
        const f2 defocusJitter = make_f2((c0.x * P.DefocusStrength) / numPixelsX, (c0.y * P.DefocusStrength) / numPixelsX);
        rayOrigin = (s.camOrigin + s.camRight * defocusJitter.x) + s.camUp * defocusJitter.y;
    }
#else
    const f2 c0 = RandomPointInCircle(rngState);
    const f2 defocusJitter = make_f2((c0.x * P.DefocusStrength) / numPixelsX, (c0.y * P.DefocusStrength) / numPixelsX);
    const f3 rayOrigin = (s.camOrigin + s.camRight * defocusJitter.x) + s.camUp * defocusJitter.y;
#endif
    const f2 c1 = RandomPointInCircle(rngState);
    const f2 jitter = make_f2((c1.x * P.DivergeStrength) / numPixelsX, (c1.y * P.DivergeStrength) / numPixelsX);
    const f3 jitteredFocusPoint = (s.focusPoint + s.camRight * jitter.x) + s.camUp * jitter.y;
    ray.pos = rayOrigin;
    ray.dir = normalize3(jitteredFocusPoint - rayOrigin);
    ray.transmittance = splat3(1.0f);
    ray.totalLight = splat3(0.0f);
}

} // namespace rtd
