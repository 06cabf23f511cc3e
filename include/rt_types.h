/* rt_types.h — the blittable buffer-element layouts that cross the drop-in boundary.
 *
 * These are the exact byte layouts the reference's C# host uploads with
 * ComputeBuffer.SetData (strides from Marshal.SizeOf, ComputeHelper.cs:56-59) and that its
 * HLSL kernel reads as StructuredBuffers.  Little-endian, tightly packed, FP32 / INT32.
 *
 *   RtNode      32 B   BVH.cs:432-457            == RayCommon.hlsl:87-95   (BVHNode)
 *   RtTriangle  72 B   BVH.cs:579-598            == RayCommon.hlsl:49-53   (Triangle)
 *   RtMaterial  88 B   RayTracingMaterial.cs:14-27 == RayCommon.hlsl:64-76
 *   RtModel    224 B   RayComputeManager.cs:256-263 (MeshInfo) == RayCommon.hlsl:78-85 (Model)
 *   RtSphere   104 B   extension mandated by BASELINE.json north_star ("Sphere structured buffer");
 *                      intersect semantics = RaySphere, RayCommon.hlsl:289-332 (SURVEY.md §8a row S)
 *
 * Matrices are Unity Matrix4x4 = column-major in memory (m00,m10,m20,m30,m01,...), which is also
 * HLSL's default packing; mul(M, v) is the ordinary M·v.
 */
#ifndef RT_TYPES_H
#define RT_TYPES_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#pragma pack(push, 4)

typedef struct RtNode {
    float   boundsMin[3];
    float   boundsMax[3];
    int32_t startIndex;     /* leaf: first triangle (mesh-relative); inner: first child (mesh-relative), second = +1 */
    int32_t triangleCount;  /* > 0  <=> leaf (RayCommon.hlsl:246) */
} RtNode;

typedef struct RtTriangle {
    float posA[3], posB[3], posC[3];
    float normA[3], normB[3], normC[3];
} RtTriangle;

enum { RT_MATERIAL_DEFAULT = 0, RT_MATERIAL_CHECKERED = 1, RT_MATERIAL_GLASS = 2 }; /* RayTracingMaterial.cs:7-12 */

typedef struct RtMaterial {
    float   diffuseCol[4];
    float   emissionCol[4];
    float   specularCol[4];
    float   absorption[4];
    float   absorptionStrength;   /* C# name: absorptionMultiplier */
    float   emissionStrength;
    float   smoothness;
    float   specularProbability;
    float   ior;
    int32_t flag;
} RtMaterial;

typedef struct RtModel {
    int32_t    nodeOffset;
    int32_t    triOffset;
    float      worldToLocal[16];  /* column-major */
    float      localToWorld[16];  /* column-major */
    RtMaterial material;
} RtModel;

typedef struct RtSphere {
    float      centre[3];
    float      radius;
    RtMaterial material;
} RtSphere;

/* Per-pixel traversal counters of the counting launch ("countStats" = 1; no counterpart in the reference, whose `stats`
 * (RayCommon.hlsl:254,271) are never written out).  The fields mean what the RtStats fields of the same names mean, summed
 * over all samples and bounces of that pixel since the last rtResetStats.  Unsigned 32-bit: they wrap modulo 2^32. */
typedef struct RtPixelStats {
    uint32_t rays, boxTests, triTests, sphereTests, sphereBoxTests;
} RtPixelStats;

/* A caller-supplied ray of rtTraceRays / rtTraceRaysDevice (include/rt_b200.h): world-space origin and direction.  The direction
 * need not be unit length; dst is measured in multiples of it. */
typedef struct RtRay {
    float origin[3];
    float dir[3];
} RtRay;

enum { RT_HIT_NONE = 0, RT_HIT_SPHERE = 1, RT_HIT_MODEL = 2 };

/* The closest hit of one RtRay: CalculateRayCollision's HitInfo (RayCommon.hlsl:335-374) plus which object won. */
typedef struct RtRayHit {
    float   dst;          /* ray parameter of the closest hit (HL:366); +inf = nothing hit */
    float   pos[3];       /* origin + dir * dst (HL:368); 0 on a miss */
    float   normal[3];    /* world-space normal as HL:367 (models) / HL:320 (spheres) compute it; 0 on a miss */
    int32_t isBackface;   /* 0 / 1 */
    int32_t kind;         /* RT_HIT_NONE, RT_HIT_SPHERE or RT_HIT_MODEL */
    int32_t index;        /* index of the winner in Spheres / ModelInfo; -1 on a miss */
    int32_t pad[2];       /* 0 */
} RtRayHit;

/* A caller-supplied segment of rtTraceOcclusion / rtTraceOcclusionDevice (include/rt_b200.h): the points origin + t * dir with
 * 0 <= t < tMax, t in multiples of dir as RtRayHit.dst is. */
typedef struct RtRaySegment {
    float origin[3];
    float dir[3];
    float tMax;
} RtRaySegment;

/* A caller-supplied path of rtTracePaths / rtTracePathsDevice (include/rt_b200.h): the first segment's world-space origin and
 * direction, and the RNG state the path starts from. */
typedef struct RtPathRay {
    float    origin[3];
    float    dir[3];       /* not normalised by the call: Trace uses it as given, as HL:479 does */
    uint32_t rngState;     /* the RNG state the path starts from (HL:127-138) */
} RtPathRay;

/* The radiance along one RtPathRay: the mean of its samples, and the RNG state after the last one (16 bytes: one float4 store). */
typedef struct RtPathRadiance {
    float    rgb[3];
    uint32_t rngState;     /* the state after the last sample: a caller continues the chain with it */
} RtPathRadiance;

/* One probe of rtBakeProbes / rtBakeProbesDevice (include/rt_b200.h): the radiance around a point projected onto the real L2
 * spherical harmonics, Unity's SphericalHarmonicsL2 layout before its shader-constant conversion.  112 bytes. */
typedef struct RtProbeSH {
    float    sh[3][9];     /* [r, g, b][coefficient], coefficients ordered by l, then m = -l .. l (Unity's order) */
    uint32_t rejected;     /* samples whose radiance was not finite and were left out of the sums */
} RtProbeSH;

/* One texel of rtBakeCubemaps / rtBakeCubemapsDevice (include/rt_b200.h): the mean radiance over the texel's area.  16 bytes. */
typedef struct RtCubeTexel {
    float    rgb[3];
    uint32_t rejected;     /* samples whose radiance was not finite and were left out of the sum (they count as black) */
} RtCubeTexel;

/* One texel of rtBakeLightmap / rtBakeLightmapDevice (include/rt_b200.h): a point on a surface and the normal that sets its
 * hemisphere (world space; the normal need not be unit length).  The baked value is an RtCubeTexel.  24 bytes. */
typedef struct RtSurfacePoint {
    float position[3];
    float normal[3];
} RtSurfacePoint;

/* One pixel of rtDispatchFeatures' "FeatureFrame" (include/rt_b200.h): what the pixel's feature ray hits first.  32 bytes. */
typedef struct RtPixelFeatures {
    float   albedo[3];    /* (0, 0, 0) on a miss; (1, 1, 1) for glass; GetMaterialColour (HL:450-466) otherwise */
    float   dst;          /* RtRayHit.dst of the feature ray; +inf on a miss */
    float   normal[3];    /* RtRayHit.normal; 0 on a miss */
    int32_t object;       /* ModelInfo index m -> m;  Spheres index s -> -2 - s;  miss -> -1 */
} RtPixelFeatures;

#pragma pack(pop)

#ifdef __cplusplus
}
static_assert(sizeof(RtPixelStats) == 20, "PixelStats record");
static_assert(sizeof(RtRay) == 24, "RtRay record");
static_assert(sizeof(RtRayHit) == 48, "RtRayHit record");
static_assert(sizeof(RtRaySegment) == 28, "RtRaySegment record");
static_assert(sizeof(RtPathRay) == 28, "RtPathRay record");
static_assert(sizeof(RtPathRadiance) == 16, "RtPathRadiance record");
static_assert(sizeof(RtPixelFeatures) == 32, "RtPixelFeatures record");
static_assert(sizeof(RtProbeSH) == 112, "RtProbeSH record");
static_assert(sizeof(RtCubeTexel) == 16, "RtCubeTexel record");
static_assert(sizeof(RtSurfacePoint) == 24, "RtSurfacePoint record");
static_assert(sizeof(RtNode) == 32, "BVHNode stride");
static_assert(sizeof(RtTriangle) == 72, "Triangle stride");
static_assert(sizeof(RtMaterial) == 88, "RayTracingMaterial stride");
static_assert(sizeof(RtModel) == 224, "Model/MeshInfo stride");
static_assert(sizeof(RtSphere) == 104, "Sphere stride");
#endif

#endif /* RT_TYPES_H */
