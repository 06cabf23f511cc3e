/* rt_oracle.cpp — TEST INFRASTRUCTURE.  CPU restatement ("oracle") of the reference's path-tracing
 * hot path: Assets/Scripts/Tracer/RayCompute.compute:10-32 and Assets/Scripts/Tracer/RayCommon.hlsl:1-582
 * of SebLague/Ray-Tracing, transcribed function by function, line by line (each function cites the
 * lines it follows; identifiers are the reference's).
 *
 * PARITY UNPINNED against the real reference: the reference ships no tests, golden images or
 * known-answer vectors (SURVEY.md §4, §8c) and neither its HLSL nor its C# can run in this image
 * (no Unity / dxc / dotnet / mono).  What pins this oracle instead: the integer RNG known-answer
 * vectors hand-derived from RayCommon.hlsl:127-137 (tests/golden/pcg_kat.json), analytic checks
 * (sphere hit distances, furnace test), BVH-vs-brute-force equality, and the arithmetic contract
 * in rt_oracle_math.h.
 *
 * Who may use this file: tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl
 * reference legs — as the checker and as the reported CPU baseline.  The product
 * (ray_tracing_b200/csrc, librt_b200.so) never includes, links or calls anything in oracle/.
 *
 * It exports the same C-ABI as include/rt_b200.h (so the same host call sequence drives either
 * implementation) plus or* helpers for tests.  Plain C-style C++; std::thread over rows.
 */
#include "../include/rt_b200.h"
#include "rt_oracle_math.h"   // HL = Assets/Scripts/Tracer/RayCommon.hlsl of the reference in the comments below

#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

using namespace orc;

namespace {

/* ======================================================================================================
 *  The shader.  One instance = one thread's view of the HLSL global scope (uniforms + buffers).
 * ====================================================================================================== */
struct Shader
{
    // --- Settings and constants ---                                           RayCommon.hlsl:1-31
    static constexpr float PI = 3.1415f;                                     // :2  (sic)

    // Raytracing Settings                                                      :4-8
    int MaxBounceCount = 0;
    int NumRaysPerPixel = 0;
    int Frame = 0;
    int renderSeed = 0;

    // Camera settings                                                          :10-14
    float DefocusStrength = 0;
    float DivergeStrength = 0;
    float3 ViewParams = {0, 0, 0};
    float4x4 CamLocalToWorldMatrix = {{1,0,0,0, 0,1,0,0, 0,0,1,0, 0,0,0,1}};

    // Sky settings                                                             :16-21
    int UseSky = 0;
    float3 SunColour = {0, 0, 0};
    float SunFocus = 0;      // HLSL initialisers (:19-20) are ignored for cbuffer globals; host always sets them
    float SunIntensity = 0;
    float3 dirToSun = {0, 0, 0};

    // Constants                                                                :28-31
    static constexpr int MATERIAL_CHECKERED = 1;
    static constexpr int MATERIAL_GLASS = 2;

    // RayCompute.compute:7-8
    uint Resolution[2] = {0, 0};
    bool accumulate = false;

    // --- Buffers ---                                                          :115-121
    const RtModel* ModelInfo = nullptr;
    const RtTriangle* Triangles = nullptr;
    const RtNode* Nodes = nullptr;
    int modelCount = 0;
    // extension (SURVEY.md §8a row S): Sphere structured buffer
    const RtSphere* Spheres = nullptr;
    int sphereCount = 0;

    // work counters (the reference's `stats`, :254,271, plus rays = CalculateRayCollision calls)
    unsigned long long nTri = 0, nBox = 0, nRays = 0, nSphere = 0;

    // ---- Structures ----                                                     :33-113
    struct Ray
    {
        float3 pos;
        float3 dir;
        float3 invDir;
        float3 transmittance;
        int bounceCount;
    };

    struct TriangleHitInfo
    {
        bool didHit;
        bool isBackface;
        float dst;
        float3 hitPoint;
        float3 normal;
    };

    struct ModelHitInfo
    {
        bool didHit;
        bool isBackface;
        float3 normal;
        float3 pos;
        float dst;
        RtMaterial material;
    };

    struct LightResponse
    {
        float3 reflectDir;
        float3 refractDir;
        float reflectWeight;
        float refractWeight;
    };

    // ---- RNG Functions ----                                                  :123-164
    static uint NextRandom(uint& state)                                      // :127-133
    {
        state = state * 747796405u + 2891336453u;
        uint result = ((state >> ((state >> 28) + 4)) ^ state) * 277803737u;
        result = (result >> 22) ^ result;
        return result;
    }

    static float RandomValue(uint& state)                                    // :135-138
    {
        // the literal 4294967295.0 is a float: it rounds to 2^32
        return (float)NextRandom(state) / 4294967296.0f;
    }

    static float RandomValueNormalDistribution(uint& state)                  // :141-147
    {
        float theta = (2.0f * 3.1415926f) * RandomValue(state);
        float rho = orc::sqrt(-2.0f * orc::log(RandomValue(state)));
        return rho * orc::cos(theta);
    }

    static float3 RandomDirection(uint& state)                               // :150-157
    {
        float x = RandomValueNormalDistribution(state);
        float y = RandomValueNormalDistribution(state);
        float z = RandomValueNormalDistribution(state);
        return normalize(mk3(x, y, z));
    }

    static float2 RandomPointInCircle(uint& rngState)                        // :159-164
    {
        float angle = RandomValue(rngState) * 2.0f * PI;
        float2 pointOnCircle = mk2(orc::cos(angle), orc::sin(angle));
        return pointOnCircle * orc::sqrt(RandomValue(rngState));
    }

    float3 GetEnvironmentLight(float3 dir) const                             // :167-183
    {
        if (UseSky == 0) return mk3(0.0f);
        const float3 GroundColour = mk3(0.35f, 0.3f, 0.35f);
        const float3 SkyColourHorizon = mk3(1.0f, 1.0f, 1.0f);
        const float3 SkyColourZenith = mk3(0.08f, 0.37f, 0.73f);

        float skyGradientT = orc::pow(smoothstep(0.0f, 0.4f, dir.y), 0.35f);
        float groundToSkyT = smoothstep(-0.01f, 0.0f, dir.y);
        float3 skyGradient = lerp(SkyColourHorizon, SkyColourZenith, skyGradientT);
        float s = 1000.0f * 1.0f / SunFocus;
        float sun = orc::pow(orc::max(0.0f, dot(dir, dirToSun)), s) * SunIntensity;
        // (HL:180)
        float3 composite = lerp(GroundColour, skyGradient, groundToSkyT) + sun * SunColour * (groundToSkyT >= 1.0f ? 1.0f : 0.0f);
        return composite;
    }

    // (HL:185)
    static TriangleHitInfo RayTriangle(const Ray& ray, const RtTriangle& tri, bool cullBackface)   // :188-215
    {
        float3 posA = mk3(tri.posA), posB = mk3(tri.posB), posC = mk3(tri.posC);
        float3 edgeAB = posB - posA;
        float3 edgeAC = posC - posA;
        float3 triFaceVector = cross(edgeAB, edgeAC);
        float3 vertRayOffset = ray.pos - posA;
        float3 rayOffsetPerp = cross(vertRayOffset, ray.dir);
        float determinant = -dot(ray.dir, triFaceVector);
        float invDet = 1.0f / determinant;

        // (HL:198)
        float dst = dot(vertRayOffset, triFaceVector) * invDet;
        float u = dot(edgeAC, rayOffsetPerp) * invDet;
        float v = -dot(edgeAB, rayOffsetPerp) * invDet;
        float w = 1.0f - u - v;

        // (HL:204)
        TriangleHitInfo hitInfo;
        bool keep = cullBackface ? determinant >= 1E-8f : orc::abs(determinant) >= 1E-8f;
        hitInfo.didHit = keep && dst > 0.0f && u >= 0.0f && v >= 0.0f && w >= 0.0f;
        float3 smoothNormal = normalize(mk3(tri.normA) * w + mk3(tri.normB) * u + mk3(tri.normC) * v);
        hitInfo.normal = smoothNormal * sign(determinant);
        hitInfo.isBackface = determinant < 0.0f;
        hitInfo.hitPoint = ray.pos + ray.dir * dst;
        hitInfo.dst = dst;
        return hitInfo;
    }

    static float RayBoundingBoxDst(const Ray& ray, float3 boxMin, float3 boxMax)     // :219-231
    {
        float3 tMin = (boxMin - ray.pos) * ray.invDir;
        float3 tMax = (boxMax - ray.pos) * ray.invDir;
        float3 t1 = orc::min(tMin, tMax);
        float3 t2 = orc::max(tMin, tMax);
        float tNear = orc::max(orc::max(t1.x, t1.y), t1.z);
        float tFar = orc::min(orc::min(t2.x, t2.y), t2.z);

        bool hit = tFar >= tNear && tFar > 0.0f;
        float dst = hit ? tNear > 0.0f ? tNear : 0.0f : rt_inf();
        return dst;
    }

    TriangleHitInfo RayTriangleBVH(Ray& ray, float rayLength, int nodeOffset, int triOffset, bool cullBackface)   // :234-287
    {
        TriangleHitInfo result;
        result.didHit = false; result.isBackface = false;          // (uninitialised in the HLSL; never read unless dst improved)
        result.hitPoint = mk3(0.0f); result.normal = mk3(0.0f);
        result.dst = rayLength;

        // the reference declares int stack[32] (:239) but its builder's MaxDepth = 32 (BVH.cs:91) can
        // need 33 entries; 64 here — identical whenever the reference does not overflow.
        int stack[64];
        int stackCount = 0;
        stack[stackCount++] = nodeOffset + 0;

        while (stackCount > 0)
        {
            const RtNode& node = Nodes[stack[--stackCount]];
            bool isLeaf = node.triangleCount > 0;

            if (isLeaf)
            {
                for (int i = 0; i < node.triangleCount; i++)
                {
                    const RtTriangle& tri = Triangles[triOffset + node.startIndex + i];
                    TriangleHitInfo triHitInfo = RayTriangle(ray, tri, cullBackface);
                    nTri++; // count triangle intersection tests                       :254

                    if (triHitInfo.didHit && triHitInfo.dst < result.dst)
                    {
                        result = triHitInfo;
                    }
                }
            }
            else
            {
                int childIndexA = nodeOffset + node.startIndex + 0;
                int childIndexB = nodeOffset + node.startIndex + 1;
                const RtNode& childA = Nodes[childIndexA];
                const RtNode& childB = Nodes[childIndexB];

                float dstA = RayBoundingBoxDst(ray, mk3(childA.boundsMin), mk3(childA.boundsMax));
                float dstB = RayBoundingBoxDst(ray, mk3(childB.boundsMin), mk3(childB.boundsMax));
                nBox += 2; // count bounding box intersection tests                   :271

                // (HL:273)
                bool isNearestA = dstA <= dstB;
                float dstNear = isNearestA ? dstA : dstB;
                float dstFar = isNearestA ? dstB : dstA;
                int childIndexNear = isNearestA ? childIndexA : childIndexB;
                int childIndexFar = isNearestA ? childIndexB : childIndexA;

                if (dstFar < result.dst) stack[stackCount++] = childIndexFar;
                if (dstNear < result.dst) stack[stackCount++] = childIndexNear;
            }
        }

        return result;
    }

    // :289-332, with the hard-coded debug material (:321-327) replaced by the sphere's own (extension)
    static ModelHitInfo RaySphere(float3 rayPos, float3 rayDir, float3 sphereCentre, float sphereRadius)
    {
        ModelHitInfo hitInfo;
        memset(&hitInfo, 0, sizeof(hitInfo));
        hitInfo.dst = rt_inf();

        float3 offsetRayOrigin = rayPos - sphereCentre;
        float a = dot(rayDir, rayDir);
        float b = 2.0f * dot(offsetRayOrigin, rayDir);
        float c = dot(offsetRayOrigin, offsetRayOrigin) - sphereRadius * sphereRadius;
        float discriminant = b * b - 4.0f * a * c;

        if (discriminant >= 0.0f)
        {
            float s = orc::sqrt(discriminant);
            float dstNear = orc::max(0.0f, (-b - s) / (2.0f * a));
            float dstFar = (-b + s) / (2.0f * a);

            if (dstFar >= 0.0f)
            {
                hitInfo.didHit = true;
                bool isInside = dstNear == 0.0f;
                hitInfo.isBackface = isInside;
                hitInfo.dst = isInside ? dstFar : dstNear;

                hitInfo.pos = rayPos + rayDir * hitInfo.dst;
                hitInfo.normal = normalize(hitInfo.pos - sphereCentre) * (isInside ? -1.0f : 1.0f);
            }
        }

        return hitInfo;
    }

    ModelHitInfo CalculateRayCollision(const Ray& worldRay, bool forceDontCullBack)      // :335-374
    {
        ModelHitInfo result;
        memset(&result, 0, sizeof(result));
        result.dst = rt_inf();
        nRays++;

        // Sphere extension: analytic spheres are tested in world space before the model loop, where the
        // reference's commented-out call sits (:341); first index wins ties (strict <).
        for (int i = 0; i < sphereCount; i++)
        {
            const RtSphere& sphere = Spheres[i];
            ModelHitInfo s = RaySphere(worldRay.pos, worldRay.dir, mk3(sphere.centre), sphere.radius);
            nSphere++;
            if (s.didHit && s.dst < result.dst)
            {
                result = s;
                result.material = sphere.material;
            }
        }

        Ray localRay;
        localRay.transmittance = mk3(0.0f);
        localRay.bounceCount = 0;

        for (int i = 0; i < modelCount; i++)
        {
            const RtModel& model = ModelInfo[i];
            float4x4 worldToLocalMatrix, localToWorldMatrix;
            memcpy(worldToLocalMatrix.m, model.worldToLocal, 64);
            memcpy(localToWorldMatrix.m, model.localToWorld, 64);
            // (HL:350)
            localRay.pos = mul_xyz(worldToLocalMatrix, mk4(worldRay.pos, 1.0f));
            localRay.dir = mul_xyz(worldToLocalMatrix, mk4(worldRay.dir, 0.0f));
            localRay.invDir = 1.0f / localRay.dir;

            bool cullBackface = model.material.flag != MATERIAL_GLASS;
            if (forceDontCullBack) cullBackface = false;
            // (HL:358)
            TriangleHitInfo hit = RayTriangleBVH(localRay, result.dst, model.nodeOffset, model.triOffset, cullBackface);

            // (HL:361)
            if (hit.dst < result.dst)
            {
                result.didHit = true;
                result.isBackface = hit.isBackface;
                result.dst = hit.dst;
                result.normal = normalize(mul_xyz(localToWorldMatrix, mk4(hit.normal, 0.0f)));
                result.pos = worldRay.pos + worldRay.dir * hit.dst;
                result.material = model.material;
            }
        }

        return result;
    }

    static float2 mod2(float2 x, float y)                                      // :376-379
    {
        return mk2(x.x - y * orc::floor(x.x / y), x.y - y * orc::floor(x.y / y));
    }

    static float CalculateReflectance(float3 inDir, float3 normal, float iorA, float iorB)   // :383-405
    {
        float refractRatio = iorA / iorB;
        float cosAngleIn = -dot(inDir, normal);
        float sinSqrAngleOfRefraction = refractRatio * refractRatio * (1.0f - cosAngleIn * cosAngleIn);
        if (sinSqrAngleOfRefraction >= 1.0f) return 1.0f; // Ray is fully reflected, no refraction occurs

        float cosAngleOfRefraction = orc::sqrt(1.0f - sinSqrAngleOfRefraction);
        float denominatorPerpendicular = iorA * cosAngleIn + iorB * cosAngleOfRefraction;
        float denominatorParallel = iorA * cosAngleIn + iorB * cosAngleOfRefraction;    // (sic, :392)

        if (orc::min(denominatorPerpendicular, denominatorParallel) < 1E-8f) return 1.0f;

        // (HL:396)
        float rPerpendicular = (iorA * cosAngleIn - iorB * cosAngleOfRefraction) / denominatorPerpendicular;
        rPerpendicular *= rPerpendicular;
        // (HL:399)
        float rParallel = (iorB * cosAngleIn - iorA * cosAngleOfRefraction) / denominatorParallel;
        rParallel *= rParallel;

        // (HL:403)
        return (rPerpendicular + rParallel) / 2.0f;
    }

    static float3 Refract(float3 inDir, float3 normal, float iorA, float iorB)        // :408-417
    {
        float refractRatio = iorA / iorB;
        float cosAngleIn = -dot(inDir, normal);
        float sinSqrAngleOfRefraction = refractRatio * refractRatio * (1.0f - cosAngleIn * cosAngleIn);
        if (sinSqrAngleOfRefraction > 1.0f) return mk3(0.0f); // Ray is fully reflected, no refraction occurs

        float3 refractDir = refractRatio * inDir + (refractRatio * cosAngleIn - orc::sqrt(1.0f - sinSqrAngleOfRefraction)) * normal;
        return refractDir;
    }

    static float3 Reflect(float3 inDir, float3 normal)                              // :419-422
    {
        return inDir - 2.0f * dot(inDir, normal) * normal;
    }

    static LightResponse CalculateReflectionAndRefraction(float3 inDir, float3 normal, float iorA, float iorB)   // :424-437
    {
        LightResponse result;

        // (HL:428)
        result.reflectDir = Reflect(inDir, normal);
        result.refractDir = Refract(inDir, normal, iorA, iorB);

        // (HL:432)
        result.reflectWeight = CalculateReflectance(inDir, normal, iorA, iorB);
        result.refractWeight = 1.0f - result.reflectWeight;

        return result;
    }

    static Ray CreateRay(float3 origin, float3 dir, float3 transmittance, int bounceIndex)   // :439-448
    {
        Ray ray;
        ray.pos = origin;
        ray.dir = dir;
        ray.invDir = 1.0f / dir;
        ray.transmittance = transmittance;
        ray.bounceCount = bounceIndex;
        return ray;
    }

    static float3 GetMaterialColour(const RtMaterial& mat, float3 pos, float3 normal, bool isSpecularBounce)   // :450-466
    {
        float3 col = mk3(mat.diffuseCol);

        if (mat.flag == MATERIAL_CHECKERED)
        {
            float2 checkerPoint = mk2(pos.x, pos.z);
            if (orc::abs(normal.x) > orc::abs(normal.y)) checkerPoint = mk2(pos.z, pos.y);
            if (orc::abs(normal.z) > orc::max(orc::abs(normal.x), orc::abs(normal.y))) checkerPoint = mk2(pos.x, pos.y);

            checkerPoint = checkerPoint * 1.5f;
            float2 c = mod2(mk2(orc::floor(checkerPoint.x), orc::floor(checkerPoint.y)), 2.0f);
            col = c.x == c.y ? col : mk3(mat.emissionCol);
        }

        return lerp(col, mk3(mat.specularCol), isSpecularBounce ? 1.0f : 0.0f);
    }

    static constexpr float epsilon = 0.001f;                                    // :468

    float3 Trace(Ray initialRay, uint& rngState)                             // :479-542
    {
        float3 totalLight = mk3(0.0f);
        Ray ray = initialRay;

        // (HL:484)
        for (int i = ray.bounceCount; i <= MaxBounceCount; i++)
        {
            ModelHitInfo hit = CalculateRayCollision(ray, false);
            if (!hit.didHit)
            {
                if (UseSky)
                {
                    totalLight += ray.transmittance * GetEnvironmentLight(ray.dir);
                }
                break;
            }

            const RtMaterial& material = hit.material;

            if (material.flag == MATERIAL_GLASS) // Glass-like material
            {
                // (HL:501)
                if (hit.isBackface) ray.transmittance *= orc::exp(-hit.dst * mk3(material.absorption) * material.absorptionStrength);

                float iorCurrent = hit.isBackface ? material.ior : 1.0f;
                float iorNext = hit.isBackface ? 1.0f : material.ior;
                LightResponse lr = CalculateReflectionAndRefraction(ray.dir, hit.normal, iorCurrent, iorNext);

                // (HL:508)
                float3 diffuseDir = normalize(hit.normal + RandomDirection(rngState));
                // (HL:510)
                lr.reflectDir = normalize(lerp(diffuseDir, lr.reflectDir, material.specularProbability));
                lr.refractDir = normalize(lerp(-diffuseDir, lr.refractDir, material.smoothness));

                // (HL:514)
                bool followReflection = RandomValue(rngState) <= lr.reflectWeight;
                ray.dir = followReflection ? lr.reflectDir : lr.refractDir;
                ray.pos = hit.pos + epsilon * hit.normal * sign(dot(hit.normal, ray.dir));
            }
            else
            {
                bool isSpecularBounce = material.specularProbability >= RandomValue(rngState);

                // (HL:523)
                ray.pos = hit.pos + (hit.normal * epsilon);
                float3 diffuseDir = normalize(hit.normal + RandomDirection(rngState));
                float3 specularDir = reflect(ray.dir, hit.normal);
                ray.dir = normalize(lerp(diffuseDir, specularDir, material.smoothness * (isSpecularBounce ? 1.0f : 0.0f)));

                // (HL:529)
                float3 emittedLight = mk3(material.emissionCol) * material.emissionStrength;
                totalLight += emittedLight * ray.transmittance;
                ray.transmittance *= GetMaterialColour(material, hit.pos, hit.normal, isSpecularBounce);
            }

            // (HL:535)
            float p = orc::max(ray.transmittance.x, orc::max(ray.transmittance.y, ray.transmittance.z));
            if (RandomValue(rngState) >= p) break;
            ray.transmittance *= 1.0f / p; // scale by inverse probability so result averages out over many iterations
        }

        return totalLight;
    }

    float3 RayTrace(float2 uv, const uint numPixels[2])                      // :545-582
    {
        float3 camOrigin = mul_xyz(CamLocalToWorldMatrix, mk4(mk3(0.0f, 0.0f, 0.0f), 1.0f));

        // (HL:549)
        uint pixelCoordX = orc::f2uint_rz(uv.x * (float)numPixels[0]);
        uint pixelCoordY = orc::f2uint_rz(uv.y * (float)numPixels[1]);
        uint pixelIndex = pixelCoordY * numPixels[0] + pixelCoordX;
        uint rngState = pixelIndex + (uint)Frame * 719393u + (uint)renderSeed;

        // (HL:554)
        float3 focusPointLocal = mk3(uv.x - 0.5f, uv.y - 0.5f, 1.0f) * ViewParams;
        float3 focusPoint = mul_xyz(CamLocalToWorldMatrix, mk4(focusPointLocal, 1.0f));
        float3 camRight = mk3(M(CamLocalToWorldMatrix,0,0), M(CamLocalToWorldMatrix,1,0), M(CamLocalToWorldMatrix,2,0));
        float3 camUp = mk3(M(CamLocalToWorldMatrix,0,1), M(CamLocalToWorldMatrix,1,1), M(CamLocalToWorldMatrix,2,1));

        // (HL:560)
        float3 totalIncomingLight = mk3(0.0f);

        for (int rayIndex = 0; rayIndex < NumRaysPerPixel; rayIndex++)
        {
            // (HL:565)
            float2 defocusJitter = RandomPointInCircle(rngState) * DefocusStrength / (float)numPixels[0];
            float3 rayOrigin = camOrigin + camRight * defocusJitter.x + camUp * defocusJitter.y;

            float2 jitter = RandomPointInCircle(rngState) * DivergeStrength / (float)numPixels[0];
            float3 jitteredFocusPoint = focusPoint + camRight * jitter.x + camUp * jitter.y;
            float3 rayDir = normalize(jitteredFocusPoint - rayOrigin);

            Ray ray = CreateRay(rayOrigin, rayDir, mk3(1.0f), 0);

            totalIncomingLight += Trace(ray, rngState);
        }

        return totalIncomingLight / (float)NumRaysPerPixel;
    }

    // kernel RayTrace, RayCompute.compute:10-24 (one invocation = one thread id)
    void Kernel_RayTrace(uint idx, uint idy, float* FrameRender, float* AccumulatedRender)
    {
        if (idx >= Resolution[0] || idy >= Resolution[1]) return;

        float2 uv = mk2((float)idx / ((float)Resolution[0] - 1.0f), (float)idy / ((float)Resolution[1] - 1.0f));
        float3 pixelCol = RayTrace(uv, Resolution);

        size_t o = ((size_t)idy * Resolution[0] + idx) * 4;
        FrameRender[o + 0] = pixelCol.x; FrameRender[o + 1] = pixelCol.y; FrameRender[o + 2] = pixelCol.z; FrameRender[o + 3] = 1.0f;

        if (accumulate)
        {
            AccumulatedRender[o + 0] += pixelCol.x; AccumulatedRender[o + 1] += pixelCol.y;
            AccumulatedRender[o + 2] += pixelCol.z; AccumulatedRender[o + 3] += 1.0f;
        }
    }
};

} // namespace

/* ======================================================================================================
 *  C-ABI (same surface as include/rt_b200.h) — host-side state, no arithmetic of the path below here.
 * ====================================================================================================== */
struct RtContext
{
    Shader sh;                        // uniforms live here; buffers point into the vectors below
    std::vector<RtTriangle> triangles;
    std::vector<RtNode> nodes;
    std::vector<RtModel> models;
    std::vector<RtSphere> spheres;
    std::vector<float> frame, accum;
    int width = 0, height = 0;
    int tileRank = 0, tileWorld = 1, bandRows = 1;
    int threads = 0;
    RtStats stats = {};
    std::string err;
};

static std::string g_createErr;

static int fail(RtContext* c, int code, const std::string& msg) { if (c) c->err = msg; else g_createErr = msg; return code; }

// The traversal stack below is int stack[64] (the reference's is 32, RayCommon.hlsl:239); a Nodes buffer whose inner nodes nest deeper
// than 63 levels would overflow it.  Same limit and same error as the product's rtDispatch (rt_repack.cuh planScene).
static bool bvhTooDeepOrBroken(const RtContext* c, std::string& why)
{
    const long long nn = (long long)c->nodes.size();
    for (int i = 0; i < c->sh.modelCount && i < (int)c->models.size(); i++)
    {
        const int off = c->models[i].nodeOffset;
        if (off < 0 || off >= nn) { why = "model nodeOffset out of range"; return true; }
        std::vector<std::pair<long long, int>> todo(1, std::make_pair((long long)off, 1));
        size_t visited = 0;
        while (!todo.empty())
        {
            const std::pair<long long, int> cur = todo.back(); todo.pop_back();
            const RtNode& nd = c->nodes[(size_t)cur.first];
            if (nd.triangleCount > 0) continue;
            if (cur.second > 63) { why = "BVH too deep: more than 63 levels of inner nodes (the traversal stacks hold 64 entries; the reference's builder stops at 32)"; return true; }
            if (++visited > c->nodes.size()) { why = "BVH has a cycle"; return true; }
            const long long a = (long long)off + nd.startIndex;
            if (a < 0 || a + 1 >= nn) { why = "BVH child index out of range"; return true; }
            todo.push_back(std::make_pair(a, cur.second + 1)); todo.push_back(std::make_pair(a + 1, cur.second + 1));
        }
    }
    return false;
}

extern "C" {

int rtGetVersion(void) { return RT_B200_VERSION; }

int rtCreate(RtContext** out, int /*device*/)
{
    if (!out) return fail(nullptr, RT_E_INVALID, "rtCreate: out is NULL");
    *out = new RtContext();
    const char* e = getenv("RT_ORACLE_THREADS");
    (*out)->threads = e ? atoi(e) : (int)std::thread::hardware_concurrency();
    if ((*out)->threads < 1) (*out)->threads = 1;
    return RT_OK;
}

int rtDestroy(RtContext* ctx) { delete ctx; return RT_OK; }

const char* rtLastError(const RtContext* ctx) { return ctx ? ctx->err.c_str() : g_createErr.c_str(); }

int rtSetBuffer(RtContext* c, const char* name, const void* data, int count, int stride)
{
    if (!c || !name || count < 0 || (count > 0 && !data)) return fail(c, RT_E_INVALID, "rtSetBuffer: bad argument");
    std::string n(name);
#define SETBUF(NAME, VEC, T) if (n == NAME) { if (stride != (int)sizeof(T)) return fail(c, RT_E_INVALID, std::string("rtSetBuffer: stride mismatch for ") + NAME); \
        c->VEC.resize(count); if (count) memcpy(c->VEC.data(), data, (size_t)count * sizeof(T)); return RT_OK; }
    SETBUF("Triangles", triangles, RtTriangle)
    SETBUF("Nodes", nodes, RtNode)
    SETBUF("ModelInfo", models, RtModel)
    SETBUF("Spheres", spheres, RtSphere)
#undef SETBUF
    return fail(c, RT_E_UNKNOWN_NAME, std::string("rtSetBuffer: unknown buffer ") + name);
}

int rtSetInt(RtContext* c, const char* name, int v)
{
    if (!c || !name) return fail(c, RT_E_INVALID, "rtSetInt: bad argument");
    std::string n(name);
    if (n == "Frame") c->sh.Frame = v;
    else if (n == "UseSky") c->sh.UseSky = v;
    else if (n == "MaxBounceCount") c->sh.MaxBounceCount = v;
    else if (n == "NumRaysPerPixel") c->sh.NumRaysPerPixel = v;
    else if (n == "renderSeed") c->sh.renderSeed = v;
    else if (n == "modelCount") c->sh.modelCount = v;
    else if (n == "triangleCount" || n == "visMode") { /* declared but unused by the shader (:24,120) */ }
    else return fail(c, RT_E_UNKNOWN_NAME, std::string("rtSetInt: unknown uniform ") + name);
    return RT_OK;
}

int rtSetInts(RtContext* c, const char* name, const int* v, int n)
{
    if (!c || !name || !v) return fail(c, RT_E_INVALID, "rtSetInts: bad argument");
    if (std::string(name) == "Resolution")
    {
        if (n != 2) return fail(c, RT_E_INVALID, "rtSetInts: Resolution takes 2 values");
        c->sh.Resolution[0] = (uint)v[0]; c->sh.Resolution[1] = (uint)v[1];
        return RT_OK;
    }
    return fail(c, RT_E_UNKNOWN_NAME, std::string("rtSetInts: unknown uniform ") + name);
}

int rtSetFloat(RtContext* c, const char* name, float v)
{
    if (!c || !name) return fail(c, RT_E_INVALID, "rtSetFloat: bad argument");
    std::string n(name);
    if (n == "DefocusStrength") c->sh.DefocusStrength = v;
    else if (n == "DivergeStrength") c->sh.DivergeStrength = v;
    else if (n == "SunFocus") c->sh.SunFocus = v;
    else if (n == "SunIntensity") c->sh.SunIntensity = v;
    else if (n == "debugVisScale") { }
    else return fail(c, RT_E_UNKNOWN_NAME, std::string("rtSetFloat: unknown uniform ") + name);
    return RT_OK;
}

int rtSetVector(RtContext* c, const char* name, const float v[4])
{
    if (!c || !name || !v) return fail(c, RT_E_INVALID, "rtSetVector: bad argument");
    std::string n(name);
    if (n == "ViewParams") c->sh.ViewParams = mk3(v);
    else if (n == "SunColour") c->sh.SunColour = mk3(v);
    else if (n == "dirToSun") c->sh.dirToSun = mk3(v);
    else if (n == "debugParams") { }
    else return fail(c, RT_E_UNKNOWN_NAME, std::string("rtSetVector: unknown uniform ") + name);
    return RT_OK;
}

int rtSetMatrix(RtContext* c, const char* name, const float v[16])
{
    if (!c || !name || !v) return fail(c, RT_E_INVALID, "rtSetMatrix: bad argument");
    if (std::string(name) == "CamLocalToWorldMatrix") { memcpy(c->sh.CamLocalToWorldMatrix.m, v, 64); return RT_OK; }
    return fail(c, RT_E_UNKNOWN_NAME, std::string("rtSetMatrix: unknown uniform ") + name);
}

int rtSetBool(RtContext* c, const char* name, int v)
{
    if (!c || !name) return fail(c, RT_E_INVALID, "rtSetBool: bad argument");
    if (std::string(name) == "accumulate") { c->sh.accumulate = v != 0; return RT_OK; }
    return fail(c, RT_E_UNKNOWN_NAME, std::string("rtSetBool: unknown uniform ") + name);
}

int rtResize(RtContext* c, int w, int h)
{
    if (!c || w <= 0 || h <= 0) return fail(c, RT_E_INVALID, "rtResize: bad size");
    if (w != c->width || h != c->height)
    {
        c->width = w; c->height = h;
        c->frame.assign((size_t)w * h * 4, 0.0f);
        c->accum.assign((size_t)w * h * 4, 0.0f);
    }
    c->sh.Resolution[0] = (uint)w; c->sh.Resolution[1] = (uint)h;
    return RT_OK;
}

int rtSetTile(RtContext* c, int rank, int world, int bandRows)
{
    if (!c || world < 1 || rank < 0 || rank >= world || bandRows < 1) return fail(c, RT_E_INVALID, "rtSetTile: bad argument");
    c->tileRank = rank; c->tileWorld = world; c->bandRows = bandRows;
    return RT_OK;
}

static void bind_buffers(RtContext* c, Shader& s)
{
    s.Triangles = c->triangles.data(); s.Nodes = c->nodes.data(); s.ModelInfo = c->models.data();
    s.Spheres = c->spheres.data();
    s.sphereCount = (int)c->spheres.size();     // the Spheres buffer length is its count (extension)
}

int rtDispatch(RtContext* c, int kernelIndex, int gx, int gy, int gz)
{
    if (!c || gx < 0 || gy < 0 || gz < 0) return fail(c, RT_E_INVALID, "rtDispatch: bad argument");
    if (c->width == 0) return fail(c, RT_E_STATE, "rtDispatch: rtResize has not been called");
    uint W = c->sh.Resolution[0], H = c->sh.Resolution[1];
    if ((int)W != c->width || (int)H != c->height) return fail(c, RT_E_STATE, "rtDispatch: Resolution does not match the textures");
    uint limX = (uint)gx * 8u < W ? (uint)gx * 8u : W, limY = (uint)gy * 8u < H ? (uint)gy * 8u : H;
    if (gz == 0) limX = limY = 0;

    if (kernelIndex == RT_KERNEL_RESET_ACCUMULATED)                    // RayCompute.compute:26-32
    {
        for (uint y = 0; y < limY; y++)
            memset(&c->accum[((size_t)y * W) * 4], 0, (size_t)limX * 16);
        return RT_OK;
    }
    if (kernelIndex != RT_KERNEL_RAYTRACE) return fail(c, RT_E_INVALID, "rtDispatch: kernelIndex must be 0 or 1");
    if (c->sh.modelCount > (int)c->models.size()) return fail(c, RT_E_STATE, "rtDispatch: modelCount exceeds ModelInfo length");
    { std::string why; if (bvhTooDeepOrBroken(c, why)) return fail(c, RT_E_STATE, "rtDispatch: " + why); }

    auto t0 = std::chrono::steady_clock::now();
    std::atomic<uint> nextRow(0);
    int nt = c->threads;
    std::vector<Shader> shaders(nt, c->sh);
    std::vector<std::thread> pool;
    for (int t = 0; t < nt; t++)
    {
        pool.emplace_back([&, t]() {
            Shader& s = shaders[t];
            bind_buffers(c, s);
            for (;;)
            {
                uint y = nextRow.fetch_add(1);
                if (y >= limY) break;
                if ((int)((y / (uint)c->bandRows) % (uint)c->tileWorld) != c->tileRank) continue;
                for (uint x = 0; x < limX; x++) s.Kernel_RayTrace(x, y, c->frame.data(), c->accum.data());
            }
        });
    }
    for (auto& th : pool) th.join();
    for (auto& s : shaders) { c->stats.rays += s.nRays; c->stats.boxTests += s.nBox; c->stats.triTests += s.nTri; c->stats.sphereTests += s.nSphere; }
    c->stats.dispatches++;
    c->stats.kernelMs += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    return RT_OK;
}

int rtReadback(RtContext* c, const char* tex, float* dst, size_t bytes)
{
    if (!c || !tex || !dst) return fail(c, RT_E_INVALID, "rtReadback: bad argument");
    std::string n(tex);
    const std::vector<float>* src = n == "FrameRender" ? &c->frame : n == "AccumulatedRender" ? &c->accum : nullptr;
    if (!src) return fail(c, RT_E_UNKNOWN_NAME, std::string("rtReadback: unknown texture ") + tex);
    if (bytes != src->size() * 4) return fail(c, RT_E_INVALID, "rtReadback: bytes must be W*H*16");
    memcpy(dst, src->data(), bytes);
    return RT_OK;
}

// Display.shader:42-47 (col = tex / Frame) + sRGB 8-bit back buffer
static unsigned DisplayEncode(float v)
{
    if (!(v > 0.0f)) return 0u;
    if (v > 1.0f) v = 1.0f;
    const float e = v <= 0.0031308f ? 12.92f * v : 1.055f * orc::pow(v, 0.41666666f) - 0.055f;
    return orc::f2uint_rz(orc::min(orc::max(e, 0.0f), 1.0f) * 255.0f + 0.5f);
}

int rtDisplay(RtContext* c, int useAccumulated, int Frame, uint8_t* dst, size_t bytes)
{
    if (!c || !dst) return fail(c, RT_E_INVALID, "rtDisplay: bad argument");
    const std::vector<float>& tex = useAccumulated ? c->accum : c->frame;
    if (tex.empty()) return fail(c, RT_E_STATE, "rtDisplay: rtResize has not been called");
    if (bytes != tex.size()) return fail(c, RT_E_INVALID, "rtDisplay: bytes must equal W*H*4");
    const float frame = (float)Frame;
    for (size_t i = 0; i < tex.size(); i++) dst[i] = (uint8_t)DisplayEncode(tex[i] / frame);
    return RT_OK;
}

int rtSynchronize(RtContext* c) { return c ? RT_OK : RT_E_INVALID; }
int rtReadbackAsync(RtContext* c, const char* tex, float* dst, size_t bytes) { return rtReadback(c, tex, dst, bytes); }      // the CPU has nothing to overlap
int rtDisplayAsync(RtContext* c, int useAccumulated, int Frame, uint8_t* dst, size_t bytes) { return rtDisplay(c, useAccumulated, Frame, dst, bytes); }
int rtReadbackWait(RtContext* c) { return c ? RT_OK : RT_E_INVALID; }
// multi-GPU entry points of the ABI: the oracle is one CPU "device"
int rtCreateMulti(RtContext** out, const int* devices, int nDevices)
{
    if (nDevices != 1) return fail(nullptr, RT_E_STATE, "oracle: one device only");
    return rtCreate(out, devices ? devices[0] : 0);
}
int rtGetUniqueId(void*, size_t) { return fail(nullptr, RT_E_STATE, "oracle: no NCCL"); }
int rtCommInit(RtContext* c, const void*, size_t, int, int) { return fail(c, RT_E_STATE, "oracle: no NCCL"); }
int rtCommDestroy(RtContext* c) { return fail(c, RT_E_STATE, "oracle: no NCCL"); }
int rtExchangeTiles(RtContext* c) { return fail(c, RT_E_STATE, "oracle: no device tile staging"); }
int rtSetStream(RtContext* c, void*) { return c ? RT_OK : RT_E_INVALID; }
int rtPackTile(RtContext* c) { return fail(c, RT_E_STATE, "oracle: no device tile staging"); }
int rtUnpackTiles(RtContext* c) { return fail(c, RT_E_STATE, "oracle: no device tile staging"); }
int rtGetDevicePointer(RtContext* c, const char*, void**, size_t*) { return fail(c, RT_E_STATE, "oracle: no device memory"); }

int rtGetIpcHandles(RtContext* c, void*, size_t) { return fail(c, RT_E_STATE, "oracle: no device memory"); }
int rtSetPeers(RtContext* c, int, const void*, size_t) { return fail(c, RT_E_STATE, "oracle: no device memory"); }

int rtSetOption(RtContext* c, const char* name, int value)
{
    if (!c || !name) return fail(c, RT_E_INVALID, "rtSetOption: bad argument");
    std::string n(name);
    if (n == "threads") { c->threads = value < 1 ? 1 : value; return RT_OK; }
    if (n == "kernel" || n == "countStats" || n == "smemNodes" || n == "poolSlots" || n == "tailLanes" || n == "sortRays" || n == "extInstantiation" || n == "modelSkip") return RT_OK;   // accepted, meaningless on the CPU
    return fail(c, RT_E_UNKNOWN_NAME, std::string("rtSetOption: unknown option ") + name);
}

int rtGetStats(RtContext* c, RtStats* out) { if (!c || !out) return RT_E_INVALID; *out = c->stats; return RT_OK; }
int rtResetStats(RtContext* c) { if (!c) return RT_E_INVALID; c->stats = RtStats(); return RT_OK; }

/* ---- oracle-only helpers for tests -------------------------------------------------------------------- */

/* Trace only the listed pixels (xy = n pairs of global pixel coordinates) with the context's current
 * uniforms and buffers; out = n float4 (the FrameRender value of each pixel).  Exact, because pixels are
 * independent and seeded from their global index (RayCommon.hlsl:550-552).  Multi-threaded. */
int orRenderPixels(RtContext* c, const int* xy, int n, float* out)
{
    if (!c || !xy || !out || n < 0) return fail(c, RT_E_INVALID, "orRenderPixels: bad argument");
    if (c->sh.modelCount > (int)c->models.size()) return fail(c, RT_E_STATE, "orRenderPixels: modelCount exceeds ModelInfo length");
    { std::string why; if (bvhTooDeepOrBroken(c, why)) return fail(c, RT_E_STATE, "orRenderPixels: " + why); }
    auto t0 = std::chrono::steady_clock::now();
    std::atomic<int> next(0);
    int nt = c->threads;
    std::vector<Shader> shaders(nt, c->sh);
    std::vector<std::thread> pool;
    for (int t = 0; t < nt; t++)
    {
        pool.emplace_back([&, t]() {
            Shader& s = shaders[t];
            bind_buffers(c, s);
            const uint* R = s.Resolution;
            for (;;)
            {
                int i0 = next.fetch_add(16);
                if (i0 >= n) break;
                for (int i = i0; i < n && i < i0 + 16; i++)
                {
                    uint x = (uint)xy[2 * i], y = (uint)xy[2 * i + 1];
                    float2 uv = mk2((float)x / ((float)R[0] - 1.0f), (float)y / ((float)R[1] - 1.0f));   // RayCompute.compute:15
                    float3 col = s.RayTrace(uv, R);
                    out[4 * i + 0] = col.x; out[4 * i + 1] = col.y; out[4 * i + 2] = col.z; out[4 * i + 3] = 1.0f;
                }
            }
        });
    }
    for (auto& th : pool) th.join();
    for (auto& s : shaders) { c->stats.rays += s.nRays; c->stats.boxTests += s.nBox; c->stats.triTests += s.nTri; c->stats.sphereTests += s.nSphere; }
    c->stats.kernelMs += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    return RT_OK;
}

/* PCG known-answer access: advances *state once, returns NextRandom's result; *value = RandomValue. */
unsigned orNextRandom(unsigned* state, float* value)
{
    uint s = *state;
    uint r = Shader::NextRandom(s);
    *state = s;
    if (value) *value = (float)r / 4294967296.0f;
    return r;
}

/* Pinned transcendental routines, for accuracy tests: fn 0 log, 1 exp, 2 sin, 3 cos, 4 pow(x, y[i]). */
void orMath(int fn, const float* x, const float* y, float* out, int n)
{
    for (int i = 0; i < n; i++)
    {
        switch (fn)
        {
        case 0: out[i] = orc::log(x[i]); break;
        case 1: out[i] = orc::exp(x[i]); break;
        case 2: out[i] = orc::sin(x[i]); break;
        case 3: out[i] = orc::cos(x[i]); break;
        case 4: out[i] = orc::pow(x[i], y[i]); break;
        default: out[i] = 0.0f;
        }
    }
}

/* Single-primitive probes for analytic tests. */
float orRayBoundingBoxDst(const float pos[3], const float dir[3], const float bmin[3], const float bmax[3])
{
    Shader::Ray r; r.pos = mk3(pos); r.dir = mk3(dir); r.invDir = 1.0f / r.dir;
    return Shader::RayBoundingBoxDst(r, mk3(bmin), mk3(bmax));
}
int orRayTriangle(const float pos[3], const float dir[3], const RtTriangle* tri, int cull, float* dst, float normal[3])
{
    Shader::Ray r; r.pos = mk3(pos); r.dir = mk3(dir); r.invDir = 1.0f / r.dir;
    Shader::TriangleHitInfo h = Shader::RayTriangle(r, *tri, cull != 0);
    *dst = h.dst; normal[0] = h.normal.x; normal[1] = h.normal.y; normal[2] = h.normal.z;
    return (h.didHit ? 1 : 0) | (h.isBackface ? 2 : 0);
}
int orRaySphere(const float pos[3], const float dir[3], const float centre[3], float radius, float* dst, float normal[3])
{
    Shader::ModelHitInfo h = Shader::RaySphere(mk3(pos), mk3(dir), mk3(centre), radius);
    *dst = h.dst; normal[0] = h.normal.x; normal[1] = h.normal.y; normal[2] = h.normal.z;
    return (h.didHit ? 1 : 0) | (h.isBackface ? 2 : 0);
}

} // extern "C"

/* Batched primitive evaluation, the oracle's side of the device probe (tests/gpu_probe/rt_probe.cu, rtpRun): same function codes,
 * same records, same index mode and digest.  Every value comes from an orc:: or Shader:: function of this file. */
namespace probe {

static unsigned long long mix64(unsigned long long z)
{
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
    return z ^ (z >> 31);
}
static unsigned long long digest_term(unsigned long long i, uint w, bool isFloat)
{
    if (isFloat && (w & 0x7fffffffu) > 0x7f800000u) w = 0x7fc00000u;
    return mix64((i << 32) ^ w);                              // i < 2^32 within one call: injective in (i, w)
}
static float3 F3(const uint* a) { return mk3(u2f(a[0]), u2f(a[1]), u2f(a[2])); }
static void put3(uint* r, float3 v) { r[0] = f2u(v.x); r[1] = f2u(v.y); r[2] = f2u(v.z); }

static int arity(int fn, int& nin, int& nout)
{
    switch (fn)
    {
    case 0: case 1: case 2: case 3: case 6: case 9: case 10: nin = 1; nout = 1; return 1;     // log exp sin cos saturate f2uint_rz DisplayEncode
    case 4: case 11: case 12: case 13: nin = 1; nout = 2; return 1;                          // sin+cos, NextRandom, RandomValue, normal draw
    case 5: case 7: case 8: nin = 2; nout = 1; return 1;                                     // pow min max
    case 14: nin = 1; nout = 4; return 1;                                                    // RandomDirection
    case 15: nin = 1; nout = 3; return 1;                                                    // RandomPointInCircle
    case 20: nin = 12; nout = 1; return 1;                                                   // RayBoundingBoxDst
    case 21: nin = 25; nout = 5; return 1;                                                   // RayTriangle
    case 22: nin = 10; nout = 2; return 1;                                                   // RaySphere
    case 23: case 24: nin = 8; nout = fn == 23 ? 1 : 3; return 1;                            // CalculateReflectance, Refract
    case 25: nin = 6; nout = 3; return 1;                                                    // Reflect
    case 26: nin = 17; nout = 3; return 1;                                                   // GetMaterialColour
    case 27: nin = 11; nout = 3; return 1;                                                   // GetEnvironmentLight
    default: return 0;
    }
}

static void eval(int fn, const uint* a, uint* r)
{
    switch (fn)
    {
    case 0: r[0] = f2u(orc::log(u2f(a[0]))); break;
    case 1: r[0] = f2u(orc::exp(u2f(a[0]))); break;
    case 2: r[0] = f2u(orc::sin(u2f(a[0]))); break;
    case 3: r[0] = f2u(orc::cos(u2f(a[0]))); break;
    case 4: r[0] = f2u(orc::sin(u2f(a[0]))); r[1] = f2u(orc::cos(u2f(a[0]))); break;
    case 5: r[0] = f2u(orc::pow(u2f(a[0]), u2f(a[1]))); break;
    case 6: r[0] = f2u(orc::saturate(u2f(a[0]))); break;
    case 7: r[0] = f2u(orc::min(u2f(a[0]), u2f(a[1]))); break;
    case 8: r[0] = f2u(orc::max(u2f(a[0]), u2f(a[1]))); break;
    case 9: r[0] = orc::f2uint_rz(u2f(a[0])); break;
    case 10: r[0] = DisplayEncode(u2f(a[0])); break;
    case 11: { uint s = a[0]; r[0] = Shader::NextRandom(s); r[1] = s; break; }
    case 12: { uint s = a[0]; r[0] = f2u(Shader::RandomValue(s)); r[1] = s; break; }
    case 13: { uint s = a[0]; r[0] = f2u(Shader::RandomValueNormalDistribution(s)); r[1] = s; break; }
    case 14: { uint s = a[0]; put3(r, Shader::RandomDirection(s)); r[3] = s; break; }
    case 15: { uint s = a[0]; const float2 p = Shader::RandomPointInCircle(s); r[0] = f2u(p.x); r[1] = f2u(p.y); r[2] = s; break; }
    case 20:
    {
        Shader::Ray ray; ray.pos = F3(a); ray.dir = F3(a + 3); ray.invDir = 1.0f / ray.dir;
        r[0] = f2u(Shader::RayBoundingBoxDst(ray, F3(a + 6), F3(a + 9)));
        break;
    }
    case 21:
    {
        Shader::Ray ray; ray.pos = F3(a); ray.dir = F3(a + 3); ray.invDir = 1.0f / ray.dir;
        RtTriangle tri; memcpy(&tri, a + 6, sizeof(tri));
        const Shader::TriangleHitInfo h = Shader::RayTriangle(ray, tri, a[24] != 0u);
        r[0] = (h.didHit ? 1u : 0u) | (h.isBackface ? 2u : 0u);
        r[1] = f2u(h.dst);
        put3(r + 2, h.normal);
        break;
    }
    case 22:
    {
        const Shader::ModelHitInfo h = Shader::RaySphere(F3(a), F3(a + 3), F3(a + 6), u2f(a[9]));
        r[0] = (h.didHit ? 1u : 0u) | (h.isBackface ? 2u : 0u);
        r[1] = f2u(h.dst);
        break;
    }
    case 23: r[0] = f2u(Shader::CalculateReflectance(F3(a), F3(a + 3), u2f(a[6]), u2f(a[7]))); break;
    case 24: put3(r, Shader::Refract(F3(a), F3(a + 3), u2f(a[6]), u2f(a[7]))); break;
    case 25: put3(r, Shader::Reflect(F3(a), F3(a + 3))); break;
    case 26:
    {
        RtMaterial m; memset(&m, 0, sizeof(m));
        m.flag = (int)a[7];
        for (int k = 0; k < 3; k++) { m.diffuseCol[k] = u2f(a[8 + k]); m.emissionCol[k] = u2f(a[11 + k]); m.specularCol[k] = u2f(a[14 + k]); }
        put3(r, Shader::GetMaterialColour(m, F3(a), F3(a + 3), a[6] != 0u));
        break;
    }
    case 27:
    {
        Shader s; s.UseSky = 1; s.SunFocus = u2f(a[3]); s.SunIntensity = u2f(a[4]); s.dirToSun = F3(a + 5); s.SunColour = F3(a + 8);
        put3(r, s.GetEnvironmentLight(F3(a)));
        break;
    }
    default: break;
    }
}

} // namespace probe

extern "C" {

/* n cases of primitive `fn` (codes and records: tests/gpu_probe/rt_probe.cu).  in: n * nin words, or NULL for index mode (word 0 of case
 * i = base + i * stride, the others = partner); out: n * nout words or NULL; digest: nout sums or NULL.  `threads` worker threads
 * (0 = all cores).  Returns 0, or 1 for an unknown function / wrong arity. */
int orProbe(int fn, int nin, int nout, const uint* in, uint base, uint stride, uint partner, uint* out, uint floatMask, size_t n,
            unsigned long long* digest, int threads)
{
    int ein = 0, eout = 0;
    if (!probe::arity(fn, ein, eout) || ein != nin || eout != nout) return 1;
    int nt = threads > 0 ? threads : (int)std::thread::hardware_concurrency();
    if (nt < 1) nt = 1;
    if ((size_t)nt > n / 4096 + 1) nt = (int)(n / 4096 + 1);
    std::vector<unsigned long long> part((size_t)nt * 8, 0ull);
    std::vector<std::thread> pool;
    for (int t = 0; t < nt; t++)
    {
        pool.emplace_back([&, t]() {
            const size_t i0 = n * (size_t)t / (size_t)nt, i1 = n * (size_t)(t + 1) / (size_t)nt;
            unsigned long long* h = &part[(size_t)t * 8];
            uint a[32], r[8];
            for (size_t i = i0; i < i1; i++)
            {
                if (in) memcpy(a, in + i * nin, (size_t)nin * 4);
                else { a[0] = base + (uint)i * stride; for (int k = 1; k < nin; k++) a[k] = partner; }
                memset(r, 0, sizeof(r));
                probe::eval(fn, a, r);
                for (int j = 0; j < nout; j++)
                {
                    if (out) out[i * nout + j] = r[j];
                    h[j] += probe::digest_term(i, r[j], (floatMask >> j) & 1u);
                }
            }
        });
    }
    for (auto& th : pool) th.join();
    if (digest)
        for (int j = 0; j < nout; j++)
        {
            unsigned long long s = 0;
            for (int t = 0; t < nt; t++) s += part[(size_t)t * 8 + j];
            digest[j] = s;
        }
    return 0;
}

} // extern "C"

// ---- BVH builder: CPU restatement of Assets/Scripts/Types/BVH.cs:26-318 (BC below), the oracle of rtBuildBVH -------------------
// Plain single-threaded recursion in the reference's own shape: one flat node list, in-place swap partition.  Test
// infrastructure like the rest of this file.
namespace BvhCs {

struct BVHTriangle { float CentreX, CentreY, CentreZ, MinX, MinY, MinZ, MaxX, MaxY, MaxZ; int Index; };      // BC:459-496

struct Builder
{
    int quality = 1;                                              // BC:11-16: 0 Low, 1 High, 2 Disabled
    std::vector<BVHTriangle> buildTriangles;
    std::vector<RtNode> nodes;

    static RtNode Node(float minX, float minY, float minZ, float maxX, float maxY, float maxZ, int start, int count)   // BC:432-457
    {
        RtNode n; n.boundsMin[0] = minX; n.boundsMin[1] = minY; n.boundsMin[2] = minZ; n.boundsMax[0] = maxX; n.boundsMax[1] = maxY; n.boundsMax[2] = maxZ;
        n.startIndex = start; n.triangleCount = count; return n;
    }
    static float NodeCost(float sizeX, float sizeY, float sizeZ, int numTriangles)     // BC:313-318
    {
        if (numTriangles == 0) return 0;
        float area = sizeX * sizeY + sizeX * sizeZ + sizeY * sizeZ;
        return area * numTriangles;
    }
    float EvaluateSplit(int splitAxis, float splitPos, int start, int count) const    // BC:253-311
    {
        float lo[2][3], hi[2][3]; int num[2] = {0, 0};
        for (int s = 0; s < 2; s++) for (int a = 0; a < 3; a++) { lo[s][a] = 3.402823466e+38f; hi[s][a] = -3.402823466e+38f; }
        for (int i = start; i < start + count; i++)
        {
            const BVHTriangle& tri = buildTriangles[i];
            const float c = splitAxis == 0 ? tri.CentreX : splitAxis == 1 ? tri.CentreY : tri.CentreZ;
            const int s = c < splitPos ? 0 : 1;
            if (tri.MinX < lo[s][0]) lo[s][0] = tri.MinX;
            if (tri.MinY < lo[s][1]) lo[s][1] = tri.MinY;
            if (tri.MinZ < lo[s][2]) lo[s][2] = tri.MinZ;
            if (tri.MaxX > hi[s][0]) hi[s][0] = tri.MaxX;
            if (tri.MaxY > hi[s][1]) hi[s][1] = tri.MaxY;
            if (tri.MaxZ > hi[s][2]) hi[s][2] = tri.MaxZ;
            num[s]++;
        }
        const float costA = NodeCost(hi[0][0] - lo[0][0], hi[0][1] - lo[0][1], hi[0][2] - lo[0][2], num[0]);
        const float costB = NodeCost(hi[1][0] - lo[1][0], hi[1][1] - lo[1][1], hi[1][2] - lo[1][2], num[1]);
        return costA + costB;
    }
    void ChooseSplit(const RtNode& node, int start, int count, int& axisOut, float& posOut, float& costOut) const     // BC:183-250
    {
        axisOut = 0; posOut = 0; costOut = INFINITY;
        if (count <= 1) return;
        const float size[3] = {node.boundsMax[0] - node.boundsMin[0], node.boundsMax[1] - node.boundsMin[1], node.boundsMax[2] - node.boundsMin[2]};
        if (quality == 0)
        {
            const int largest = size[0] > size[1] && size[0] > size[2] ? 0 : size[1] > size[2] ? 1 : 2;
            posOut = node.boundsMin[largest] + size[largest] * 0.5f; axisOut = largest;
            costOut = EvaluateSplit(largest, posOut, start, count);
            return;
        }
        const int maxSplitTests = count < 10 ? 3 : 5;
        float maxAxis = size[0] > size[1] ? size[0] : size[1];                 // Mathf.Max of three
        if (size[2] > maxAxis) maxAxis = size[2];
        float bestCost = 3.402823466e+38f;
        for (int axis = 0; axis < 3; axis++)
        {
            const float scaled = size[axis] / maxAxis * maxSplitTests;
            int numSplitTests = scaled != scaled ? -2147483647 - 1 : (int)ceil((double)scaled);     // Mathf.CeilToInt; (int)NaN is int.MinValue in C#
            if (numSplitTests < 1) numSplitTests = 1;
            if (numSplitTests > maxSplitTests) numSplitTests = maxSplitTests;
            for (int i = 0; i < numSplitTests; i++)
            {
                const float splitT = (i + 1) / (numSplitTests + 1.0f);
                const float splitPos = node.boundsMin[axis] + size[axis] * splitT;
                const float cost = EvaluateSplit(axis, splitPos, start, count);
                if (cost < bestCost) { bestCost = cost; posOut = splitPos; axisOut = axis; }
            }
        }
        costOut = bestCost;
    }
    void Split(int parentIndex, int triGlobalStart, int triNum, int depth)     // BC:89-181
    {
        const RtNode parent = nodes[parentIndex];
        const float parentCost = NodeCost(parent.boundsMax[0] - parent.boundsMin[0], parent.boundsMax[1] - parent.boundsMin[1], parent.boundsMax[2] - parent.boundsMin[2], triNum);
        int splitAxis; float splitPos, cost;
        ChooseSplit(parent, triGlobalStart, triNum, splitAxis, splitPos, cost);
        if (cost < parentCost && depth < 32)
        {
            float lo[2][3], hi[2][3];
            for (int s = 0; s < 2; s++) for (int a = 0; a < 3; a++) { lo[s][a] = 3.402823466e+38f; hi[s][a] = -3.402823466e+38f; }
            int numOnLeft = 0;
            for (int i = triGlobalStart; i < triGlobalStart + triNum; i++)
            {
                const BVHTriangle tri = buildTriangles[i];
                const float c = splitAxis == 0 ? tri.CentreX : splitAxis == 1 ? tri.CentreY : tri.CentreZ;
                const int s = c < splitPos ? 0 : 1;
                if (tri.MinX < lo[s][0]) lo[s][0] = tri.MinX;
                if (tri.MinY < lo[s][1]) lo[s][1] = tri.MinY;
                if (tri.MinZ < lo[s][2]) lo[s][2] = tri.MinZ;
                if (tri.MaxX > hi[s][0]) hi[s][0] = tri.MaxX;
                if (tri.MaxY > hi[s][1]) hi[s][1] = tri.MaxY;
                if (tri.MaxZ > hi[s][2]) hi[s][2] = tri.MaxZ;
                if (s == 0)
                {
                    const BVHTriangle swap = buildTriangles[triGlobalStart + numOnLeft];
                    buildTriangles[triGlobalStart + numOnLeft] = tri;
                    buildTriangles[i] = swap;
                    numOnLeft++;
                }
            }
            const int numOnRight = triNum - numOnLeft;
            nodes.push_back(Node(lo[0][0], lo[0][1], lo[0][2], hi[0][0], hi[0][1], hi[0][2], triGlobalStart, 0));
            const int childIndexLeft = (int)nodes.size() - 1;
            nodes.push_back(Node(lo[1][0], lo[1][1], lo[1][2], hi[1][0], hi[1][1], hi[1][2], triGlobalStart + numOnLeft, 0));
            nodes[parentIndex].startIndex = childIndexLeft;
            Split(childIndexLeft, triGlobalStart, numOnLeft, depth + 1);
            Split(childIndexLeft + 1, triGlobalStart + numOnLeft, numOnRight, depth + 1);
        }
        else { nodes[parentIndex].startIndex = triGlobalStart; nodes[parentIndex].triangleCount = triNum; }
    }
};

} // namespace BvhCs

extern "C" int rtBuildBVH(RtContext* ctx, const float* verts, int vertCount, const int* indices, int indexCount, const float* normals, int quality,
                          RtTriangle* outTris, RtNode* outNodes, int nodeCapacity, int* outNodeCount)
{
    if (!ctx || !verts || !indices || !normals || !outTris || !outNodes || !outNodeCount || quality < 0 || quality > 2 || indexCount <= 0 || indexCount % 3 != 0 || vertCount <= 0)
        return RT_E_INVALID;
    for (int i = 0; i < indexCount; i++) if (indices[i] < 0 || indices[i] >= vertCount) return RT_E_INVALID;
    BvhCs::Builder b; b.quality = quality;
    const int triCount = indexCount / 3;
    if (nodeCapacity < 2 * triCount + 1) return RT_E_INVALID;
    b.buildTriangles.resize(triCount);
    float lo[3] = {3.402823466e+38f, 3.402823466e+38f, 3.402823466e+38f}, hi[3] = {-3.402823466e+38f, -3.402823466e+38f, -3.402823466e+38f};
    for (int i = 0; i < indexCount; i += 3)                                   // BC:44-59
    {
        const float* a = verts + 3 * (size_t)indices[i]; const float* bb = verts + 3 * (size_t)indices[i + 1]; const float* c = verts + 3 * (size_t)indices[i + 2];
        BvhCs::BVHTriangle t;
        t.CentreX = (a[0] + bb[0] + c[0]) / 3; t.CentreY = (a[1] + bb[1] + c[1]) / 3; t.CentreZ = (a[2] + bb[2] + c[2]) / 3;
        float mn[3], mx[3];
        for (int d = 0; d < 3; d++)
        {
            mn[d] = a[d] < bb[d] ? (a[d] < c[d] ? a[d] : c[d]) : (bb[d] < c[d] ? bb[d] : c[d]);
            mx[d] = a[d] > bb[d] ? (a[d] > c[d] ? a[d] : c[d]) : (bb[d] > c[d] ? bb[d] : c[d]);
            if (mn[d] < lo[d]) lo[d] = mn[d];
            if (mx[d] > hi[d]) hi[d] = mx[d];
        }
        t.MinX = mn[0]; t.MinY = mn[1]; t.MinZ = mn[2]; t.MaxX = mx[0]; t.MaxY = mx[1]; t.MaxZ = mx[2]; t.Index = i;
        b.buildTriangles[i / 3] = t;
    }
    b.nodes.push_back(BvhCs::Builder::Node(lo[0], lo[1], lo[2], hi[0], hi[1], hi[2], -1, -1));     // BC:61
    if (quality == 2) { b.nodes[0].startIndex = 0; b.nodes[0].triangleCount = triCount; }
    else b.Split(0, 0, triCount, 0);
    if ((int)b.nodes.size() > nodeCapacity) return RT_E_INVALID;               // chains of empty children can exceed 2n + 1 nodes
    for (int i = 0; i < triCount; i++)                                           // BC:69-80
    {
        const int base = b.buildTriangles[i].Index;
        RtTriangle& o = outTris[i];
        for (int d = 0; d < 3; d++)
        {
            o.posA[d] = verts[3 * (size_t)indices[base] + d]; o.posB[d] = verts[3 * (size_t)indices[base + 1] + d]; o.posC[d] = verts[3 * (size_t)indices[base + 2] + d];
            o.normA[d] = normals[3 * (size_t)indices[base] + d]; o.normB[d] = normals[3 * (size_t)indices[base + 1] + d]; o.normC[d] = normals[3 * (size_t)indices[base + 2] + d];
        }
    }
    memcpy(outNodes, b.nodes.data(), b.nodes.size() * sizeof(RtNode));
    *outNodeCount = (int)b.nodes.size();
    return RT_OK;
}
