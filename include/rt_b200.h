/* rt_b200.h — C-ABI of librt_b200.so, the H100 (sm_90a) replacement for the reference's
 * RayTrace / ResetAccumulated compute kernels.
 *
 * The boundary it replaces is the Unity ComputeShader / ComputeBuffer / RenderTexture API exactly
 * as RayComputeManager drives it through ComputeHelper (SURVEY.md §8b).  Every entry point below
 * names the reference call it stands in for (paths relative to the reference repo root:
 *   RCM = Assets/Scripts/Tracer/RayComputeManager.cs, CH = Assets/Scripts/Helpers/ComputeHelper.cs,
 *   RC  = Assets/Scripts/Tracer/RayCompute.compute,   HL = Assets/Scripts/Tracer/RayCommon.hlsl).
 *
 * Conventions
 *   - plain C, no torch / CUDA types in any signature (streams and device pointers travel as void*).
 *   - every function returns 0 on success, a negative RT_E_* code on failure; rtLastError() gives text.
 *     Nothing throws or exits across the ABI.
 *   - copy-in semantics: host arrays are copied before the call returns (ComputeBuffer.SetData
 *     semantics, CH:83-153); the caller may mutate them afterwards.
 *   - single caller thread per context (Unity main thread, RCM:78); rtDispatch is asynchronous
 *     w.r.t. the CPU, rtReadback / rtSynchronize synchronise.
 *   - there is NO CPU fallback: without a CUDA device rtCreate fails with RT_E_NO_DEVICE.
 */
#ifndef RT_B200_H
#define RT_B200_H

#include <stddef.h>
#include <stdint.h>
#include "rt_types.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct RtContext RtContext;

enum {
    RT_OK              =  0,
    RT_E_INVALID       = -1,  /* bad argument (NULL, negative count, wrong stride, wrong size) */
    RT_E_UNKNOWN_NAME  = -2,  /* uniform / buffer / texture / option name not part of the kernel's interface */
    RT_E_NO_DEVICE     = -3,  /* no usable CUDA device — there is no CPU path */
    RT_E_CUDA          = -4,  /* a CUDA runtime call failed; see rtLastError */
    RT_E_STATE         = -5   /* call sequence error (e.g. dispatch before rtResize / buffers) */
};

enum { RT_KERNEL_RAYTRACE = 0, RT_KERNEL_RESET_ACCUMULATED = 1 };  /* RC:1-2, RCM:57-58 */

/* ---- lifetime ------------------------------------------------------------------------------- */

/* Replaces: the ComputeShader asset reference + lazily created GPU objects (RCM:34,126-161).
 * device = CUDA ordinal this context renders on (one context per GPU / per process). */
int rtCreate(RtContext** out, int device);

/* Replaces: OnDestroy → ComputeHelper.Release(buffers, textures) (RCM:238-247, CH:209-247). */
int rtDestroy(RtContext* ctx);

/* Text of the last error on this context (never NULL). ctx may be NULL → last rtCreate error. */
const char* rtLastError(const RtContext* ctx);

/* ---- structured buffers ------------------------------------------------------------------------ */

/* Replaces: ComputeHelper.CreateStructuredBuffer(ref buf, data) + cs.SetBuffer(kernel, name, buf)
 * (RCM:151-160,201-202; CH:83-153).  name ∈ {"Triangles"(72), "Nodes"(32), "ModelInfo"(224),
 * "Spheres"(104, extension)}; stride is validated against the element size in rt_types.h exactly as
 * Unity validates it against the HLSL struct.  The allocation is re-used when count is unchanged
 * (CH:86-92).  count == 0 (data may be NULL) empties the buffer. */
int rtSetBuffer(RtContext* ctx, const char* name, const void* data, int count, int stride);

/* ---- uniforms (same names as the HLSL globals, HL:5-26,120-121, RC:7-8) --------------------------- */

int rtSetInt   (RtContext* ctx, const char* name, int value);               /* cs.SetInt    RCM:156,165-169,178-179,203 */
int rtSetInts  (RtContext* ctx, const char* name, const int* values, int n);/* cs.SetInts   RCM:139 ("Resolution")      */
int rtSetFloat (RtContext* ctx, const char* name, float value);             /* cs.SetFloat  RCM:170-174                 */
int rtSetVector(RtContext* ctx, const char* name, const float value[4]);    /* cs.SetVector RCM:140,175-176,188         */
int rtSetMatrix(RtContext* ctx, const char* name, const float value[16]);   /* cs.SetMatrix RCM:189 (column-major)      */
int rtSetBool  (RtContext* ctx, const char* name, int value);               /* cs.SetBool   RCM:180 ("accumulate")      */

/* ---- render targets ------------------------------------------------------------------------------ */

/* Replaces: CreateRenderTexture(ref raytraceFrameTex / accumulatedResult, w, h, R32G32B32A32_SFloat)
 * + SetTexture ×3 + SetInts("Resolution") (RCM:126-139, CH:303-323).  Re-allocates only when the size
 * changes; new textures are zero-filled (a fresh RenderTexture), unchanged size keeps their content. */
int rtResize(RtContext* ctx, int width, int height);

/* Replaces: cs.Dispatch(kernelIndex, groupsX, groupsY, groupsZ) (CH:25-32, RCM:75,90).
 * Thread groups are 8×8×1 (RC:10,26): pixels with x >= min(W, 8·groupsX) or y >= min(H, 8·groupsY)
 * are left untouched, like threads that were never launched.  Asynchronous. */
int rtDispatch(RtContext* ctx, int kernelIndex, int groupsX, int groupsY, int groupsZ);

/* Extension: n = frameCount accumulated frames of RayTrace in one launch (a still rendered to many frames, RCM:84-95 called n times).
 * With F the current "Frame" uniform, the call is equal, in every byte the context exposes, to
 *     for k in 0 .. n-1:  rtSetInt("Frame", F + k); rtDispatch(RT_KERNEL_RAYTRACE, groupsX, groupsY, groupsZ)
 *     rtSetInt("Frame", F)
 * with F + k taken modulo 2^32 like the seed (HL:552):
 *   - FrameRender holds frame F + n - 1; AccumulatedRender receives the n frames' (col, 1) per pixel in frame order, with the same
 *     float additions (one thread or pool slot owns a pixel for all n frames);
 *   - RtStats rays / boxTests / triTests / sphereTests / sphereBoxTests and PixelStats equal the n dispatches' totals; dispatches
 *     grows by n; kernelMs is the one launch's time;
 *   - "Frame" is unchanged afterwards.
 * Partial dispatch, rtSetTile row bands, peers and the sphere accelerator behave as in rtDispatch.  On a group context (rtCreateMulti,
 * rtCommInit) the call reaches every GPU and, with "exchange" = 1, ends with ONE exchange of the tiles for the whole batch.
 * n = 1 is rtDispatch(RT_KERNEL_RAYTRACE, ...).  Asynchronous.
 * Refused: frameCount < 1 or frameCount * max(1, NumRaysPerPixel) > RT_MAX_BATCH_SAMPLES (the pooled kernel counts a slot's samples
 * across the batch in a 20-bit field) -> RT_E_INVALID; "accumulate" = 0 (only the last frame would be observable) -> RT_E_STATE;
 * n > 1 with "sampleChunks" forced to 2 or more (a batch runs whole pixels; the automatic setting does) -> RT_E_STATE. */
#define RT_MAX_BATCH_SAMPLES ((1 << 20) - 1)
int rtDispatchFrames(RtContext* ctx, int groupsX, int groupsY, int groupsZ, int frameCount);

/* Extension: closest-hit queries for caller-supplied rays (picking, autofocus, line of sight, visibility / occlusion baking).
 * hits[i] = CalculateRayCollision(rays[i], forceDontCullBack = flags & RT_TRACE_NO_CULL) (HL:335-374, HL:356), with the sphere
 * extension tested first as in rtDispatch: the same bits as the camera rays' intersection.  Ties keep the reference's order: spheres
 * before models, the lower buffer index first, strict <.  RtRayHit (rt_types.h): dst = +inf, pos = normal = 0, isBackface = 0,
 * kind = RT_HIT_NONE and index = -1 on a miss; kind / index name the winning Spheres or ModelInfo entry otherwise.
 *   - Reads the current Spheres, ModelInfo, Nodes, Triangles and "modelCount" and no other uniform; needs no rtResize and no
 *     earlier dispatch.  Leaves FrameRender, AccumulatedRender, "Frame", PixelStats, RtStats.dispatches and kernelMs alone and
 *     does not change what later dispatches render.
 *   - RtStats.rays grows by n.  With "countStats" = 1 the box / triangle / sphere / sphere-accelerator counters grow as a counting
 *     dispatch's do (every model is walked, like the reference).
 *   - Model skipping, the TLAS and the sphere accelerator are used only for rays whose origin lies inside the box their records were
 *     padded for (the camera and all geometry, with room) and whose direction has 2^-20 <= dot(dir, dir) <= 2^20 (the range in which
 *     the padding's error argument holds); any other ray (origin far away or NaN, direction very short, very long, zero or NaN) walks
 *     every model and tests every sphere in buffer order.  Rays that may skip share the open grazing-ray defect of model skipping
 *     (DESIGN.md section 5) with the camera rays; "modelSkip" = 0 avoids it.
 *   - On a group context (rtCreateMulti) the rays are traced on devices[0], which holds the whole scene; call it on the context
 *     rtCreateMulti returned.
 * Refused: ctx NULL, n < 0, rays / hits NULL with n > 0, flags outside {0, RT_TRACE_NO_CULL}, a device dRays not 4-byte or dHits not
 * 16-byte aligned -> RT_E_INVALID; a member context of a group other than the one rtCreateMulti returned (as rtDispatch) and the scene
 * checks of rtDispatch (modelCount beyond ModelInfo, models without Nodes / Triangles, an offset out of range, a tree deeper than 63
 * inner levels) -> RT_E_STATE.  n = 0 is RT_OK and launches nothing.
 * rtTraceRays: host arrays, traced in batches of at most RT_TRACE_CHUNK_RAYS through two device buffers the context keeps for later
 * calls (72 bytes per ray of the largest batch so far, at most 72 MiB; freed by rtDestroy); synchronises.  rtTraceRaysDevice: n RtRay /
 * RtRayHit in device memory of the context's device, no allocation; asynchronous on the context's stream (rtSetStream). */
#define RT_TRACE_NO_CULL 1
#define RT_TRACE_CHUNK_RAYS (1 << 20)
int rtTraceRays(RtContext* ctx, const RtRay* rays, int n, RtRayHit* hits, int flags);
int rtTraceRaysDevice(RtContext* ctx, const void* dRays, void* dHits, int n, int flags);

/* Extension: occlusion queries for caller-supplied segments (shadow and ambient-occlusion rays, line of sight, visibility baking).
 * occluded[i] = 1 if and only if CalculateRayCollision(ray, forceDontCullBack = flags & RT_TRACE_NO_CULL) (HL:335-374, sphere
 * extension first) finds a hit when its result.dst starts at segs[i].tMax instead of +inf; 0 otherwise.  Every < stays strict, as in
 * the reference: TMax as DXR / OptiX define it, in the reference's own arithmetic.  The walk stops at its first hit.  That is exact
 * whatever order the primitives are visited in: before the first hit the running bound is the constant tMax, so a box is entered when
 * its entry is < tMax and a primitive counts when its dst < tMax, whatever was visited before.
 *   - This is NOT always rtTraceRays(ray).dst < tMax: a box whose float entry is >= tMax can hold a triangle whose float hit is < tMax;
 *     the reference from +inf enters that box, a walk bounded by tMax does not.  occluded = 1 implies rtTraceRays(ray).dst < tMax, and
 *     with tMax = +inf the two are equal (occluded == (kind != RT_HIT_NONE)).
 *   - tMax needs no validation: NaN, 0, -0 and negative values are never occluded (every comparison with them fails); +inf is any hit.
 *   - With "countStats" = 1 the box / triangle / sphere counters count the walk in the reference's order (spheres in buffer order,
 *     then every model in buffer order, each BVH near child first) up to and including the test that produced the first hit; with
 *     the sphere accelerator the sphere counters are the accelerator's, as in rtTraceRays.
 *   - Everything else is rtTraceRays': what it reads and leaves alone, RtStats.rays growing by n, the conditions under which model
 *     skipping, the TLAS and the sphere accelerator are used, the grazing-ray defect, devices[0] on a group context, the refusals (with
 *     dSegs 4-byte aligned, dOccluded unaligned) and n = 0.
 * rtTraceOcclusion: host arrays, in batches of at most RT_TRACE_CHUNK_RAYS through the two device buffers rtTraceRays keeps (29 of their
 * 72 bytes per segment); synchronises.  rtTraceOcclusionDevice: n RtRaySegment / bytes in device memory of the context's device, no
 * allocation; asynchronous on the context's stream (rtSetStream). */
int rtTraceOcclusion(RtContext* ctx, const RtRaySegment* segs, int n, uint8_t* occluded, int flags);
int rtTraceOcclusionDevice(RtContext* ctx, const void* dSegs, void* dOccluded, int n, int flags);

/* Extension: the path tracer's radiance along caller-supplied rays (custom cameras: equirectangular, cube map, fisheye, stereo,
 * orthographic; light-probe and irradiance-volume baking; reflection probes; what one path or direction contributes).  The reference's
 * per-pixel sample loop (HL:560-581) with the caller's ray in place of the jittered camera ray, and no camera draws:
 *     state = rays[i].rngState; total = (0, 0, 0)
 *     for k in 0 .. samples - 1: total += Trace(CreateRay(origin, dir, transmittance 1, bounce 0), state)      (HL:578, in order)
 *     out[i].rgb = total / (float)samples; out[i].rngState = state                                            (HL:581)
 * Trace is HL:479-542 with its glass / diffuse / specular / emissive shading, the sky and Russian roulette; dir is used as given.
 *   - Exactness: the oracle's bits.  A NaN appears exactly where the oracle has one (its payload is free).  forceDontCullBack is false,
 *     as at HL:487, so the call takes no flags; material culling is the reference's.  With a camera ray and the state after its four
 *     jitter draws (HL:565-572), samples = 1 returns that camera sample's Trace bit for bit: a pixel of rtDispatch is the float sum of
 *     its R samples' results, in order, over (float)R.
 *   - Reads the scene buffers, "modelCount", "MaxBounceCount", "UseSky", "SunFocus", "SunIntensity", "SunColour" and "dirToSun".  Reads
 *     no camera, "Frame", "renderSeed", "NumRaysPerPixel" or "Resolution", and needs no rtResize.
 *   - Leaves FrameRender, AccumulatedRender, PixelStats, "Frame", RtStats.dispatches and kernelMs alone and does not change what later
 *     dispatches render.
 *   - RtStats.rays grows by the number of CalculateRayCollision calls: one per path segment, as for the camera kernels (not by n).  With
 *     "countStats" = 1 the box / triangle / sphere counters grow as a counting dispatch's do, walking every model.
 *   - Model skipping, the TLAS and the sphere accelerator are used per SEGMENT under rtTraceRays' conditions: the segment's origin inside
 *     the padded box and 2^-20 <= dot(dir, dir) <= 2^20.  The test applies to every bounce, not only the first: a bounce starts at a hit
 *     point, and a first segment from a far origin or with an extreme direction length puts that point where the padding argument was
 *     not made.  Any other segment walks every model and tests every sphere in buffer order.  Segments that may skip share the open
 *     grazing-ray defect (DESIGN.md section 5) with the camera rays.
 *   - On a group context (rtCreateMulti) the paths are traced on devices[0]; call it on the context rtCreateMulti returned.
 *   - Throughput: one lane traces one ray's samples (one RNG chain), so a batch fills the GPU from about as many rays as the persistent
 *     grid has lanes (132 SMs x 6 CTAs x 128 threads, about 101k on an H100 SXM); smaller batches leave it partly idle.
 * Refused: ctx NULL, n < 0, rays / out NULL with n > 0, samples < 1 or > RT_MAX_BATCH_SAMPLES (the per-launch sample budget of a batch
 * of frames), a device dRays not 4-byte or dOut not 16-byte aligned -> RT_E_INVALID; a member context of a group other than the one
 * rtCreateMulti returned, the scene checks of rtDispatch, and "MaxBounceCount" outside 0 .. 200 (as rtDispatch) -> RT_E_STATE.  n = 0 is
 * RT_OK and launches nothing.
 * rtTracePaths: host arrays, in batches of at most RT_TRACE_CHUNK_RAYS through the two device buffers rtTraceRays keeps (rays in the
 * hit buffer, 28 of its 48 bytes; results in the ray buffer, 16 of its 24); synchronises.  rtTracePathsDevice: n RtPathRay /
 * RtPathRadiance in device memory of the context's device, no allocation; asynchronous on the context's stream (rtSetStream). */
int rtTracePaths(RtContext* ctx, const RtPathRay* rays, int n, int samples, RtPathRadiance* out);
int rtTracePathsDevice(RtContext* ctx, const void* dRays, void* dOut, int n, int samples);

/* Extension: light-probe baking.  For each of n probe positions, the path tracer's radiance arriving from S = samples directions,
 * projected onto the real L2 spherical harmonics (Unity's SphericalHarmonicsL2 before its shader-constant conversion; DESIGN.md
 * section 7d''''''''' gives the constants of that conversion and of the cosine-lobe convolution, which belong to the host).  Every
 * bit is stated; each operation is one IEEE binary32 operation in the order written (no contraction).
 *   - Directions: a spherical Fibonacci set, the same for every probe, with no RNG draw.  For sample k = 0 .. S-1:
 *         t = (float)(uint32_t)(k * 2654435769u) * 2^-32          (RandomValue's conversion, HL:137)
 *         phi = t * 6.28318548f;  (s, c) = (sin phi, cos phi) as RandomPointInCircle computes them (rt_devmath.cuh sincos_rt)
 *         z = 1 - (float)(2k + 1) / (float)S;  r = sqrt(max(1 - z * z, 0));  d_k = (r * c, r * s, z), used as given
 *   - Paths: with H(x) the value NextRandom (HL:127-133) returns from state x and p the probe's index in the call,
 *         L_pk = Trace(CreateRay(positions[p], d_k, 1, 0), state = H(H(seed + p) + k))        (HL:439-448, HL:479-542)
 *     so L_pk is rtTracePaths({positions[p], d_k, H(H(seed + p) + k)}, samples = 1).rgb bit for bit.
 *   - Basis at d = (x, y, z):  Y0 = 0.282094792;  Y1 = 0.488602512 * y;  Y2 = 0.488602512 * z;  Y3 = 0.488602512 * x;
 *         Y4 = 1.09254843 * (x * y);  Y5 = 1.09254843 * (y * z);  Y6 = 0.315391565 * ((3 * (z * z)) - 1);
 *         Y7 = 1.09254843 * (x * z);  Y8 = 0.546274215 * ((x * x) - (y * y))
 *   - Sums: the samples fall into chunks of RT_PROBE_CHUNK consecutive k.  A chunk's 27 sums start at +0 and add L_pk.ch * Y_i(d_k)
 *     in k order.  A sample with any non-finite component of L_pk adds nothing and counts in `rejected` (a NaN path does not
 *     poison its probe).  The chunk sums are combined by the full binary tree that pairs adjacent chunks, the chunk count padded with
 *     +0 chunks to the next power of two (within an aligned group of 32 chunks: a warp's xor 1 / 2 / 4 / 8 / 16 shuffle sum), and
 *         out[p].sh[ch][i] = tree * (12.566371f / (float)S)
 *   - Everything else is rtTracePaths': what it reads (the scene, "modelCount", "MaxBounceCount" and the sky / sun uniforms; no camera,
 *     "Frame", "renderSeed", "NumRaysPerPixel" or "Resolution"; no rtResize needed), what it leaves alone (the images, PixelStats,
 *     "Frame", RtStats.dispatches and kernelMs), RtStats.rays growing by segments and the countStats counters as there, the per-segment
 *     gate of model skipping, the TLAS and the sphere accelerator, devices[0] on a group context.  Positions are not validated: a far or
 *     NaN origin fails the gate and walks every model.
 *   - Launches: a call runs its probes in launches of floor(RT_PROBE_SCRATCH_CHUNKS / ceil(S / RT_PROBE_CHUNK)) probes (the last one
 *     partial), each through a device scratch of 112 bytes per chunk (at most RT_PROBE_SCRATCH_CHUNKS chunks: 112 MiB) that the context
 *     keeps, grown on first use, freed by rtDestroy.  The launches change no bits: p is the index in the call.
 * Refused: ctx NULL, n < 0, positions / out NULL with n > 0, samples < 1 or > RT_MAX_BATCH_SAMPLES, a device dPositions not 4-byte or
 * dOut not 16-byte aligned -> RT_E_INVALID; a member context of a group other than the one rtCreateMulti returned, the scene checks of
 * rtDispatch and "MaxBounceCount" outside 0 .. 200 -> RT_E_STATE.  n = 0 is RT_OK and launches nothing.
 * rtBakeProbes: host arrays (positions n x 3 floats), through a launch's worth of device buffers the context keeps (12 + 112 bytes per
 * probe; freed by rtDestroy); synchronises.  rtBakeProbesDevice: n x 3 floats and n RtProbeSH in device memory of the context's
 * device; allocates only the scratch; asynchronous on the context's stream (rtSetStream). */
#define RT_PROBE_CHUNK 32
#define RT_PROBE_SCRATCH_CHUNKS (1 << 20)
int rtBakeProbes(RtContext* ctx, const float* positions, int n, int samples, uint32_t seed, RtProbeSH* out);
int rtBakeProbesDevice(RtContext* ctx, const void* dPositions, void* dOut, int n, int samples, uint32_t seed);

/* Extension: reflection-probe baking.  For each of n positions, an HDR cube map of the path tracer's radiance: 6 faces of N x N texels
 * (N = faceSize), out[((p * 6 + f) * N + y) * N + x], faces in Unity's CubemapFace order +X, -X, +Y, -Y, +Z, -Z, row y = 0 first in
 * memory and the top of the face.  Each texel is the mean of S = samples paths spread over its area.  Every bit is stated; each
 * operation is one IEEE binary32 operation in the order written (no contraction); H(x) is the value NextRandom (HL:127-133) returns
 * from state x.
 *   - Sub-texel offset of sample k: an R2 low-discrepancy point, the same for every texel, with no RNG draw, k = 0 at the centre:
 *         u = (float)(uint32_t)(k * 3242174889u + 2147483648u) * 2^-32;  v = (float)(uint32_t)(k * 2447445414u + 2147483648u) * 2^-32
 *     (RandomValue's conversion, HL:137; the constants are 2^32 / g and 2^32 / g^2 rounded, g = 1.3247... the plastic number)
 *   - Face coordinates:  a = (((float)x + u) / (float)N) * 2 - 1;  b = (((float)y + v) / (float)N) * 2 - 1
 *   - Face vectors (the Direct3D / OpenGL cube-map table of DDS and KTX):  +X (1, -b, -a);  -X (-1, -b, a);  +Y (a, 1, b);
 *     -Y (a, -1, -b);  +Z (a, -b, 1);  -Z (-a, -b, -1).  d = normalize(vector) = vector * (1 / sqrt(dot(vector, vector))), the dot
 *     summed left to right.  Seen from inside the cube in Unity's left-handed, y-up world every face is upright and unmirrored:
 *     texel (0, 0) of +X points towards (1, 1, 1).
 *   - Paths: with tau = ((p * 6 + f) * N + y) * N + x the texel's index in the call (uint32),
 *         L = Trace(CreateRay(positions[p], d, 1, 0), state = H(H(seed + tau) + k))        (HL:439-448, HL:479-542)
 *     so a sample is rtTracePaths({positions[p], d, H(H(seed + tau) + k)}, samples = 1).rgb bit for bit.
 *   - Sums: as rtBakeProbes' with 3 words: chunks of RT_PROBE_CHUNK consecutive k, each summing L from +0 in k order; a sample with any
 *     non-finite component adds nothing and counts in `rejected`; the chunks combined by the full binary tree over the chunk count
 *     padded with +0 chunks to a power of two, and
 *         out.rgb = tree / (float)S
 *     one IEEE division, as rtTracePaths divides its total: a rejected sample counts as black, and a texel is never 0 / 0.
 *   - Everything else is rtBakeProbes': what it reads and leaves alone, RtStats.rays growing by segments and the countStats counters, the
 *     per-segment gate of model skipping, the TLAS and the sphere accelerator, devices[0] on a group context, positions not validated.
 *   - Launches: a call runs its texels in launches of floor(RT_CUBE_SCRATCH_CHUNKS / ceil(S / RT_PROBE_CHUNK)) texels (the last one
 *     partial; a launch may end inside a probe or a face), each through rtBakeProbes' device scratch at 16 bytes per chunk (at most
 *     RT_CUBE_SCRATCH_CHUNKS chunks: 112 MiB).  The launches change no bits: tau is the index in the call.
 * Refused: rtBakeProbes' RT_E_INVALID cases, faceSize < 1 or > RT_CUBE_MAX_FACE, n * 6 * faceSize^2 > 2^31 - 1 texels, a device
 * dPositions not 4-byte or dOut not 16-byte aligned -> RT_E_INVALID; rtBakeProbes' RT_E_STATE cases -> RT_E_STATE.  n = 0 is RT_OK and
 * launches nothing.
 * rtBakeCubemaps: host arrays (positions n x 3 floats, out n * 6 * N^2 RtCubeTexel); the positions are copied to the device once and
 * the texels come back a launch at a time, through device buffers the context keeps (12 bytes per probe, 16 per texel of a launch;
 * freed by rtDestroy); synchronises.  rtBakeCubemapsDevice: the same arrays in device memory of the context's device; allocates only
 * the scratch; asynchronous on the context's stream (rtSetStream). */
#define RT_CUBE_MAX_FACE 4096
#define RT_CUBE_SCRATCH_CHUNKS (7 << 20)
int rtBakeCubemaps(RtContext* ctx, const float* positions, int n, int faceSize, int samples, uint32_t seed, RtCubeTexel* out);
int rtBakeCubemapsDevice(RtContext* ctx, const void* dPositions, void* dOut, int n, int faceSize, int samples, uint32_t seed);

/* Extension: lightmap baking.  For each of n surface texels, the diffuse lighting arriving at points[p].position over the hemisphere of
 * points[p].normal: out[p].rgb is the mean of S = samples paths along a cosine-weighted set of directions, an estimate of E / pi, the
 * radiance a white Lambertian surface at the texel reflects (multiply by a diffuse colour for that surface's baked lighting; the
 * irradiance is pi * rgb).  It is the expected value of what the reference's own diffuse bounce (HL:524-525, normalize(normal +
 * RandomDirection), cosine-distributed) gathers there.  Every bit is stated; each operation is one IEEE binary32 operation in the order
 * written (no contraction); H(x) is the value NextRandom (HL:127-133) returns from state x; p is the texel's index in the call.
 *   - Normal: m = points[p].normal;  n = m * (1 / sqrt(dot(m, m))), the dot summed left to right.  Normals are not validated: a zero,
 *     denormal-underflowing or non-finite normal gives the NaN directions Trace makes of it.
 *   - Tangent frame (Duff et al. 2017, "Building an Orthonormal Basis, Revisited"):
 *         sg = copysign(1, n.z);  a = -1 / (sg + n.z);  b = (n.x * n.y) * a
 *         T = (1 + ((sg * n.x) * n.x) * a,  sg * b,  -(sg * n.x));  B = (b,  sg + (n.y * n.y) * a,  -n.y)
 *   - Direction of sample k: (u, v) the R2 point of rtBakeCubemaps (the same constants; k = 0 at (0.5, 0.5)), with no RNG draw;
 *         r = sqrt(u);  (s, c) = (sin, cos)(v * 6.28318548f) as RandomPointInCircle computes them (rt_devmath.cuh sincos_rt);
 *         x = r * c;  y = r * s;  z = sqrt(max(1 - u, 0));  d = normalize(w), w.i = (T.i * x + B.i * y) + n.i * z
 *     with normalize as rtBakeCubemaps': a cosine-weighted hemisphere around n.
 *   - Origin: o = points[p].position + (n * 0.001f), the offset of the reference's diffuse bounce (HL:524, epsilon of HL:468).
 *   - Paths:  L = Trace(CreateRay(o, d, 1, 0), state = H(H(seed + p) + k))        (HL:439-448, HL:479-542)
 *     so a sample is rtTracePaths({o, d, H(H(seed + p) + k)}, samples = 1).rgb bit for bit.
 *   - Sums: rtBakeCubemaps': chunks of RT_PROBE_CHUNK consecutive k, each summing L from +0 in k order; a sample with any non-finite
 *     component adds nothing and counts in `rejected`; the chunks combined by the full binary tree over the chunk count padded with +0
 *     chunks to a power of two, and out.rgb = tree / (float)S.
 *   - Everything else is rtBakeCubemaps': what it reads and leaves alone (no camera, "Frame", "renderSeed", "NumRaysPerPixel" or
 *     "Resolution"; no rtResize needed), RtStats.rays growing by segments and the countStats counters, the per-segment gate of model
 *     skipping, the TLAS and the sphere accelerator, devices[0] on a group context, the "MaxBounceCount" and scene-check refusals.
 *     Positions are not validated: a far or NaN origin fails the gate and walks every model.
 *   - Launches: a call runs its texels in launches of floor(RT_CUBE_SCRATCH_CHUNKS / ceil(S / RT_PROBE_CHUNK)) texels, rtBakeCubemaps'
 *     rule, through rtBakeProbes' device scratch at 16 bytes per chunk.  The launches change no bits: p is the index in the call.
 * Refused: ctx NULL, n < 0, points / out NULL with n > 0, samples < 1 or > RT_MAX_BATCH_SAMPLES, a device dPoints not 4-byte or dOut
 * not 16-byte aligned -> RT_E_INVALID; rtBakeCubemaps' RT_E_STATE cases -> RT_E_STATE.  n = 0 is RT_OK and launches nothing.
 * rtBakeLightmap: host arrays, in batches of at most RT_TRACE_CHUNK_RAYS texels through the two device buffers rtTraceRays keeps (points
 * in the ray buffer, 24 of its 24 bytes; texels in the hit buffer, 16 of its 48), so a 4096^2 atlas needs no more device memory than
 * one batch; synchronises.  rtBakeLightmapDevice: n RtSurfacePoint and n RtCubeTexel in device memory of the context's device;
 * allocates only the scratch; asynchronous on the context's stream (rtSetStream). */
int rtBakeLightmap(RtContext* ctx, const RtSurfacePoint* points, int n, int samples, uint32_t seed, RtCubeTexel* out);
int rtBakeLightmapDevice(RtContext* ctx, const void* dPoints, void* dOut, int n, int samples, uint32_t seed);

/* Extension: first-hit feature images for denoisers (albedo, shading normal, depth, object id: the guides OIDN, a-trous / SVGF filters
 * and mattes take next to the colour), and the camera's own rays.
 *
 * The FEATURE RAY of pixel (x, y) is the ray RayTrace starts that pixel's first path of the current frame with: the per-pixel setup
 * for thread id (x, y) under the current "Resolution", "CamLocalToWorldMatrix", "ViewParams", "Frame" and "renderSeed" (RC:15,
 * HL:547-558: uv = id / (Resolution - 1), the pixel index recomputed from uv as there, rngState = pixelIndex + Frame * 719393 +
 * renderSeed modulo 2^32), then ONE camera sample (HL:567-576: four draws, the defocus disc by "DefocusStrength", the jitter by
 * "DivergeStrength", the normalised direction).  With "NumRaysPerPixel" = 1 it is exactly the ray the frame's path started with, so the
 * guides are anti-aliased and defocused like the colour.  With more samples per pixel it is the FIRST sample's ray only: a later sample
 * starts from the RNG state the whole path before it left behind (one chain per pixel, HL:563-579), which only tracing those paths
 * can produce.
 *
 * rtCameraRays / rtCameraRaysDevice write, for every pixel of the image, W*H RtPathRay in [y][x] order (row 0 = bottom): the feature
 * ray's origin and direction and the RNG state after its four draws: what rtTracePaths takes (rtTracePaths(rays, samples = 1).rgb is
 * FrameRender.rgb of a 1-sample rtDispatch of this frame, bit for bit) and what rtTraceRays takes in its first 24 bytes.
 *   - A query about the camera, not a render: partial dispatch and rtSetTile do not apply; no scene is needed; nothing the context
 *     exposes changes (no image, no RtStats field).
 *   - Refused: ctx NULL, rays NULL, bytes != W*H*28, a device pointer not 4-byte aligned -> RT_E_INVALID; before rtResize, "Resolution"
 *     different from the render textures or above 65535, a member context of a group other than the one rtCreateMulti returned ->
 *     RT_E_STATE.
 *   - rtCameraRays: host memory, through a device buffer of W*H*28 bytes the context keeps for later calls (freed by rtDestroy and by
 *     rtResize to a new size); synchronises.  rtCameraRaysDevice: device memory of the context's device, no allocation; asynchronous
 *     on the context's stream (rtSetStream).
 *
 * rtDispatchFeatures covers the pixels rtDispatch(RT_KERNEL_RAYTRACE, groupsX, groupsY, groupsZ) would cover (8x8 groups, partial
 * dispatch, this context's rtSetTile row bands) and touches no other.  For each, hit = CalculateRayCollision(feature ray,
 * forceDontCullBack = false) (HL:335-374, HL:487; the sphere extension first: rtTraceRays' hit of that ray with flags 0) and the
 * pixel's RtPixelFeatures record (rt_types.h) in the device image "FeatureFrame" (W*H records, [y][x], row 0 = bottom) becomes
 *     miss:                   albedo (0, 0, 0), dst +inf, normal (0, 0, 0), object -1
 *     hit:                    dst = hit.dst, normal = hit.normal, object = m for ModelInfo[m], -2 - s for Spheres[s]
 *       material.flag == 2:   albedo (1, 1, 1)       (glass: the usual convention for a transmissive surface)
 *       any other material:   albedo = GetMaterialColour(material, hit.pos, hit.normal, isSpecularBounce = false) as written at
 *                             HL:450-466: diffuseCol, or for flag == 1 the checker pattern choosing between diffuseCol and emissionCol,
 *                             then lerp(col, specularCol, 0) = col + (specularCol - col) * 0 evaluated in binary32 (a non-finite
 *                             specularCol - col gives NaN, as it does in Trace)
 * With "accumulate" != 0 a HIT is also added into two float4 images, one binary32 addition per component:
 *     AccumulatedAlbedo[pixel] += (albedo.r, albedo.g, albedo.b, 1)        AccumulatedNormal[pixel] += (normal.x, normal.y, normal.z, dst)
 * and a miss changes neither.  So AccumulatedAlbedo.w counts the feature rays that hit, AccumulatedNormal.w / AccumulatedAlbedo.w is
 * the mean depth over hits, AccumulatedNormal.xyz / AccumulatedAlbedo.w the mean normal, and AccumulatedAlbedo.rgb /
 * numAccumulatedFrames the anti-aliased albedo (a miss counts as black).  With "accumulate" = 0 only FeatureFrame is written.
 *   - The three images are allocated, zero-filled, by the first rtDispatchFeatures (even one that covers no pixel).  rtResize to a new
 *     size zeroes all three.  rtDispatch(RT_KERNEL_RESET_ACCUMULATED, gx, gy, gz) also zeroes the region it covers in both accumulators,
 *     if they exist, and leaves FeatureFrame: a host that resets its colour accumulation resets its guides with the same call.  A context
 *     that never calls rtDispatchFeatures allocates nothing and behaves as before.
 *   - Reads the scene buffers, "modelCount", the camera uniforms, "Frame", "renderSeed", "accumulate" and "Resolution".  Does not read
 *     "NumRaysPerPixel", "MaxBounceCount" or the sky.  Leaves FrameRender, AccumulatedRender, PixelStats, "Frame", RtStats.dispatches and
 *     kernelMs alone and does not change what later dispatches render.  Call it before or after the frame's rtDispatch, with the same
 *     "Frame"; it does not advance anything.
 *   - RtStats.rays grows by the pixels traced.  With "countStats" = 1 the box / triangle / sphere counters grow as a counting
 *     dispatch's first segments do (every model walked).
 *   - Model skipping, the TLAS and the sphere accelerator are used as for the camera rays of rtDispatch (which these are), with the
 *     same preparation and the open grazing-ray defect of model skipping (DESIGN.md section 5); "modelSkip" = 0 avoids it.
 *   - Reading: rtReadback and rtGetDevicePointer accept "FeatureFrame" (bytes = W*H*32), "AccumulatedAlbedo" and "AccumulatedNormal"
 *     (W*H*16); RT_E_STATE before the first rtDispatchFeatures.  rtReadbackAsync serves the two colour images only.
 *   - Refused: ctx NULL, a negative group count -> RT_E_INVALID; before rtResize, "Resolution" different from the render textures or
 *     above 65535, the scene checks of rtDispatch (modelCount beyond ModelInfo, models without Nodes / Triangles, an offset out of range,
 *     a tree deeper than 63 inner levels), and any context of a group (rtCreateMulti: the tile exchange carries the two colour images
 *     only) -> RT_E_STATE.  A single context with rtSetTile works and writes only its bands.
 * Asynchronous on the context's stream. */
int rtDispatchFeatures(RtContext* ctx, int groupsX, int groupsY, int groupsZ);
int rtCameraRays(RtContext* ctx, RtPathRay* rays, size_t bytes);
int rtCameraRaysDevice(RtContext* ctx, void* dRays, size_t bytes);

/* Extension: an edge-avoiding a-trous wavelet denoiser (Dammertz et al., HPG 2010) guided by the feature images, with the colour
 * demodulated by the albedo as in SVGF.  rtDenoise filters the whole image into the device image "DenoisedRender": W*H float4, [y][x],
 * row 0 = bottom, rgb = the denoised MEAN colour (already divided by the frame count), w = 1.  Every bit is stated below; each
 * operation is one IEEE binary32 operation in the order written (no contraction), max is NaN-ignoring.
 *
 * Constants, computed by the host in binary32 from the arguments (K = iterations):
 *     invC = 1 / (sigmaColour * sigmaColour)      cK[k] = invC * 4^k (k = 0 .. K-1)      invN = 1 / (sigmaNormal * sigmaNormal)
 *     invZ = 1 / sigmaDepth                       rd[k][d] = 2^-(k + d - 1) = 1 / (2^k * d) for d = 1, 2 (exact)
 *     h = (1/16, 1/4, 3/8, 1/4, 1/16) for offsets -2 .. 2; hh(i, j) = h[i] * h[j] (exact)
 * Per pixel p, its inputs (c colour, a albedo, n normal, z depth):
 *     useAccumulated = 1: A = AccumulatedRender, L = AccumulatedAlbedo, N = AccumulatedNormal;
 *                         c = A.rgb / A.w, a = L.rgb / L.w, n = N.xyz / L.w, z = N.w / L.w (the means over frames and over hits)
 *     useAccumulated = 0: c = FrameRender.rgb; a, n, z = albedo, normal, dst of FeatureFrame
 *     m = max(a, 2^-8) per channel, e = c / m per channel (the demodulated colour: the filter smooths lighting, not texture)
 * p is BACKGROUND when A.w == 0 or L.w == 0 (accumulated), object == -1 (frame), or any of the ten values of c, a, n, z or the three of
 * e is not finite.  A background pixel is written as (c, 1), with c = (0, 0, 0) when A.w == 0, and is never read as a neighbour.
 * Iteration k = 0 .. K-1, step s = 2^k, reads only the previous iteration's e (the first reads the e above) and writes e' for every
 * non-background p = (x, y):
 *     rz = invZ / z_p;  Sw = Sr = Sg = Sb = +0
 *     for j = -2 .. 2 (outer), i = -2 .. 2 (inner): q = (x + s*i, y + s*j); a q outside the image or on background is skipped;
 *         i = j = 0:   w = 9/64
 *         otherwise:   de = e_p - e_q, dn = n_p - n_q, t = ((z_p - z_q) * rz) * rd[k][max(|i|, |j|)]
 *                      D = (((de.r*de.r + de.g*de.g) + de.b*de.b) * cK[k] + ((dn.x*dn.x + dn.y*dn.y) + dn.z*dn.z) * invN) + t*t
 *                      w = hh(i, j) * exp_rt(-D) if D <= 103.972076416015625, else 0 (also for a NaN D: 0*inf, 0/0)
 *         a tap with w == 0 is skipped (w * e_q is not added); otherwise Sw += w, Sr += w * e_q.r, Sg += w * e_q.g, Sb += w * e_q.b
 *     e'_p = (Sr / Sw, Sg / Sw, Sb / Sw)       (Sw >= 9/64: the centre is always a tap)
 * exp_rt is the contract's exponential (DESIGN.md section 2); it returns exactly 0 for arguments below -103.972076416015625, so skipping it
 * there is bit-exact.  The normal is the mean normal, unnormalised: its shortening at silhouettes is part of the guide.  After the last
 * iteration DenoisedRender[p] = (e'.r * m.r, e'.g * m.g, e'.b * m.b, 1).
 *   - Reads the two colour images and the three feature images; leaves FrameRender, AccumulatedRender, FeatureFrame,
 *     AccumulatedAlbedo, AccumulatedNormal, PixelStats, "Frame" and every RtStats field alone and changes nothing a later dispatch
 *     renders.  Asynchronous on the context's stream.
 *   - "DenoisedRender" and the filter's scratch images are allocated by the first rtDenoise: 64 bytes of device memory per pixel in all
 *     (DenoisedRender 16, scratch 48).  rtResize to a new size zeroes DenoisedRender and frees the scratch; ResetAccumulated leaves both.
 *     rtReadback and rtGetDevicePointer accept "DenoisedRender" (W*H*16 bytes); RT_E_STATE before the first rtDenoise.
 *   - Refused: ctx NULL, useAccumulated not 0 or 1, iterations outside 1 .. RT_DENOISE_MAX_ITERATIONS, a sigma that is not finite and
 *     > 0, or a constant invC * 4^(K-1), invN or invZ that is not finite -> RT_E_INVALID; before rtResize, "Resolution" different from
 *     the render textures or above 65535, before the first rtDispatchFeatures, any context of a group (rtCreateMulti) and a context
 *     with rtSetTile world > 1 (its images hold its own bands only) -> RT_E_STATE.
 * rtDisplayDenoised is rtDisplay's encode of DenoisedRender with Frame = 1: dst receives W*H RGBA8, bytes must equal W*H*4
 * (RT_E_INVALID otherwise, and for ctx or dst NULL); RT_E_STATE before the first rtDenoise.  Synchronises. */
#define RT_DENOISE_MAX_ITERATIONS 5
int rtDenoise(RtContext* ctx, int useAccumulated, int iterations, float sigmaColour, float sigmaNormal, float sigmaDepth);
int rtDisplayDenoised(RtContext* ctx, uint8_t* dst, size_t bytes);

/* Extension: a temporal denoiser for a moving camera, SVGF (Schied et al., HPG 2017): each pixel's first hit is reprojected into the
 * previous call's camera, its demodulated colour and luminance moments are blended with the history found there, and the variance of
 * those moments steers an a-trous filter of the integrated colour.  One call per frame, after the frame's rtDispatch(RAYTRACE) and
 * rtDispatchFeatures with the same "Frame"; it reads FrameRender (the frame's own colour: any "accumulate" works), FeatureFrame,
 * "CamLocalToWorldMatrix", "ViewParams" and "Resolution", and writes "DenoisedRender" (as rtDenoise does: W*H float4, w = 1, so
 * rtDisplayDenoised, rtReadback and rtGetDevicePointer serve it) and "TemporalFrame": W*H float4, [y][x], row 0 = bottom,
 * (prevX, prevY, len, variance).  The operations are binary32 in the order written, as for rtDenoise; min / max are NaN-ignoring.
 *
 * Constants: RT_TEMPORAL_TAU_Z, RT_TEMPORAL_TAU_N, RT_TEMPORAL_MAX_HISTORY, RT_TEMPORAL_EPSILON below; from the arguments, in binary32:
 *     invN = 1 / (sigmaNormal * sigmaNormal)     invZ = 1 / sigmaDepth     invL = 1 / sigmaLuminance
 *     lum(v) = (0.2126 * v.r + 0.7152 * v.g) + 0.0722 * v.b       (the binary32 literals)
 * Per pixel p = (x, y): c = FrameRender.rgb; a, z, n, object from FeatureFrame; m = max(a, 2^-8), e = c / m; p is BACKGROUND under
 * rtDenoise's frame rule (object == -1 or one of c, a, n, z, e not finite).  A background pixel gets DenoisedRender (c, 1),
 * TemporalFrame (NaN, NaN, 0, 0), no history record, and is never read.  Otherwise l = lum(e), and:
 * 1. Reprojection.  The previous camera is that of the last successful call, unless resetHistory = 1, rtResize to a new size came
 *    between, or there is none: then (prevX, prevY) = (NaN, NaN).  If the previous call's "CamLocalToWorldMatrix" and "ViewParams" equal
 *    the current ones bit for bit (the image size is equal: a new size discards the history), prevX = x, prevY = y and zexp = z.
 *    Otherwise, with camOrigin and focusPoint of the pixel's SetupPixel (HL:547-558) and the previous camera M', VP':
 *        d = normalize(focusPoint - camOrigin)   X = camOrigin + d * z (per component: o + d * z)
 *        A = M' rows 0..2, columns 0..2; t = M' column 3 rows 0..2.  In float64: cofactors c_rc of A, det = (a00*c00 + a01*c01) + a02*c02,
 *        R[r][k] = c_kr / det; b[r] = -((R[r][0]*t0 + R[r][1]*t1) + R[r][2]*t2); each R and b entry then rounded once to binary32.
 *        L[r] = ((R[r][0]*X.x + R[r][1]*X.y) + R[r][2]*X.z) + b[r]
 *        u = (L.x / L.z) * kx + 0.5, v = (L.y / L.z) * ky + 0.5 with kx = VP'.z / VP'.x, ky = VP'.z / VP'.y (binary32)
 *        prevX = u * (W - 1), prevY = v * (H - 1);  zexp = sqrt((dx*dx + dy*dy) + dz*dz), (dx, dy, dz) = X - t (binary32 t)
 *    and the projection fails ((prevX, prevY) = (NaN, NaN)) unless L.z > 0 and X, L, u, v, prevX, prevY and zexp are all finite.
 * 2. History.  With (prevX, prevY) not NaN and -1 < prevX < W, -1 < prevY < H: x0 = floor(prevX), fx = prevX - x0 (y likewise), and
 *    the taps (x0, y0), (x0 + 1, y0), (x0, y0 + 1), (x0 + 1, y0 + 1) in that order with weight w = wx * wy, wx = 1 - fx or fx,
 *    wy = 1 - fy or fy.  A tap q counts when w != 0, q is inside the image, q has a history record (not background in the previous
 *    call), object_q == object, |z_q - zexp| <= RT_TEMPORAL_TAU_Z * zexp and (n.x*n_q.x + n.y*n_q.y) + n.z*n_q.z >= RT_TEMPORAL_TAU_N.
 *    Over the counted taps: Sw += w, Sc += w * colour_q (per channel), S1 += w * m1_q, S2 += w * m2_q, lenH = max(lenH, len_q).
 * 3. Integration.  No counted tap: len = 1, colour = e, (m1, m2) = (l, l*l).  Otherwise h = Sc / Sw, h1 = S1 / Sw, h2 = S2 / Sw,
 *    len = min(lenH + 1, RT_TEMPORAL_MAX_HISTORY), a = max(alpha, 1 / len), colour = h + a * (e - h), m1 = h1 + a * (l - h1),
 *    m2 = h2 + a * (l*l - h2).  p's history record becomes (n, z, object, m1, m2, len).  TemporalFrame.xyz = (prevX, prevY, len).
 * 4. Variance.  len >= 4: var = max(m2 - m1*m1, 0).  Otherwise, over the 7x7 neighbours q = (x + i, y + j), j = -3 .. 3 (outer),
 *    i = -3 .. 3, inside the image and not background: w = 1 for q = p, else with dn = n - n_q, t = (z - z_q) * (invZ / z):
 *        D = (|m1 - m1_q| * invL + ((dn.x*dn.x + dn.y*dn.y) + dn.z*dn.z) * invN) + t*t, w = exp_rt(-D) (0 when D > 103.972076416015625
 *        or NaN); a tap with w == 0 is skipped; Sw += w, S1 += w * m1_q, S2 += w * m2_q
 *    and var = max(S2 / Sw - (S1 / Sw) * (S1 / Sw), 0) * (4 / len).  TemporalFrame.w = var.
 * 5. Filter.  Iterations k = 0 .. K-1 run rtDenoise's pass (step s = 2^k, the same taps, order, hh(i, j), t with rd[k][d], skip rules
 *    and sums, over the current guides n, z) on the pair (colour, var), starting from step 3's colour and step 4's var, with two changes:
 *        gv_p = Sg / Sk over the 3x3 immediate neighbours q = (x + i, y + j), j = -1 .. 1 (outer), i = -1 .. 1, inside the image
 *               and not background, of this iteration's input var (SVGF's prefilter, at every step):
 *               k = k1[i] * k1[j], k1 = (1/4, 1/2, 1/4); Sk += k, Sg += k * var_q
 *        kL = 1 / (sigmaLuminance * sqrt(gv_p) + RT_TEMPORAL_EPSILON)
 *        D = (|lum(colour_p) - lum(colour_q)| * kL + ((dn.x*dn.x + dn.y*dn.y) + dn.z*dn.z) * invN) + t*t     (no colour distance)
 *        for each added tap also Sv += (w * w) * var_q (the centre: w = 9/64), and var'_p = Sv / (Sw * Sw).
 *    The output colour of iteration 0 is p's colour history for the next call.  After the last iteration DenoisedRender[p] =
 *    (colour'.r * m.r, colour'.g * m.g, colour'.b * m.b, 1).
 *   - Geometry is assumed static between calls: a moved model gets no motion vectors; the object, depth and normal tests are what
 *     limit its ghosting.
 *   - Leaves FrameRender, AccumulatedRender, the feature images, PixelStats, "Frame", every RtStats field and what later dispatches
 *     render alone.  rtDenoise and rtDenoiseTemporal do not affect each other's results (they share only DenoisedRender and the
 *     filter's scratch images).  ResetAccumulated leaves the history alone.  Asynchronous on the context's stream.
 *   - Memory: "TemporalFrame" and the history are allocated by the first call, 112 bytes of device memory per pixel (TemporalFrame 16,
 *     two alternating sets of guide, moments and colour history 96), plus rtDenoise's 64 if rtDenoise has not allocated them.
 *     rtResize to a new size zeroes TemporalFrame and discards the history.  rtReadback and rtGetDevicePointer accept "TemporalFrame"
 *     (W*H*16 bytes); RT_E_STATE before the first rtDenoiseTemporal.
 *   - Refused: ctx NULL, iterations outside 1 .. RT_DENOISE_MAX_ITERATIONS, a sigma that is not finite and > 0, invN, invZ or invL not
 *     finite, alpha outside (0, 1], resetHistory not 0 or 1 -> RT_E_INVALID; before rtResize, "Resolution" different from the render
 *     textures or above 65535, before the first rtDispatchFeatures, any context of a group and a context with rtSetTile world > 1 ->
 *     RT_E_STATE.  A refused call leaves the history and the previous camera as they were. */
#ifndef RT_TEMPORAL_TAU_Z                  /* overridable only by the A/B build variants of tools/build_variants.py */
#define RT_TEMPORAL_TAU_Z 0.05f
#endif
#ifndef RT_TEMPORAL_TAU_N
#define RT_TEMPORAL_TAU_N 0.9f
#endif
#define RT_TEMPORAL_MAX_HISTORY 32
#define RT_TEMPORAL_EPSILON 0.0000152587890625f     /* 2^-16 */
int rtDenoiseTemporal(RtContext* ctx, int iterations, float sigmaLuminance, float sigmaNormal, float sigmaDepth, float alpha, int resetHistory);

/* Extension: adaptive sampling.  One call renders the next frame of a progressive accumulation only in the pixels whose estimated error
 * is still above `threshold`.  Covered pixels are those rtDispatch(RT_KERNEL_RAYTRACE, groupsX, groupsY, groupsZ) covers (8x8 groups,
 * partial dispatch, this context's rtSetTile row bands).
 *   - "AdaptiveMoments": W*H float4, [y][x], row 0 = bottom; per pixel (s1, s2, n, 0) = the sums of l and l*l and the number of frames
 *     over the frames rtDispatchAdaptive traced there.  It counts adaptive frames only: rtDispatch, rtDispatchFrames and rtResetStats
 *     leave it alone.
 *   - Selection, per covered pixel, on the moments as they were before the call (binary32, one operation each in the order written,
 *     no contraction; max ignores NaN):
 *         mu = s1 / n;   v = max(s2 / n - mu * mu, 0)
 *         active = n < (float)minFrames || (n < (float)maxFrames && v > ((threshold * threshold) * n) * (mu * mu + RT_ADAPTIVE_EPSILON))
 *     i.e. the standard error of the mean luminance is above threshold times the mean, with an absolute floor for dark pixels.  A pixel
 *     whose moments are not finite becomes inactive after minFrames (the comparison with NaN is false); maxFrames bounds every pixel.
 *   - Tracing: each active pixel is traced exactly as rtDispatch(RAYTRACE) traces it at the current "Frame" (FrameRender,
 *     AccumulatedRender, PixelStats with "countStats" = 1 and the traversal counters, bit for bit); then, with (r, g, b) the frame
 *     colour it wrote, l = (0.2126f * r + 0.7152f * g) + 0.0722f * b (rtDenoiseTemporal's lum) and AdaptiveMoments = (s1 + l,
 *     s2 + l * l, n + 1, 0).  Inactive and uncovered pixels are not touched in any image.  Which lane traces which pixel, and in which
 *     order, changes no bit.
 *   - *activePixels (may be NULL) receives the number of pixels traced.  The call synchronises once, between the device-side selection
 *     and the render launch, and returns with the render queued.  With at least one active pixel RtStats.dispatches grows by 1, kernelMs
 *     by the render launch's time, rays and the test counters by what was traced; with none, nothing is rendered and no RtStats field
 *     changes.  "Frame" is read and not advanced, as in rtDispatch.
 *   - Memory: AdaptiveMoments is allocated, zero-filled, by the first call, with a pixel list: 20 bytes of device memory per pixel plus
 *     4 bytes per 32 pixels of selection scratch.  rtResize to a new size zeroes it; rtDispatch(RT_KERNEL_RESET_ACCUMULATED, ...) zeroes
 *     the region it covers.  A context that never calls rtDispatchAdaptive allocates none of it.  rtReadback and rtGetDevicePointer
 *     accept "AdaptiveMoments" (W*H*16 bytes); RT_E_STATE before the first call.
 *   - Refused: ctx NULL, a negative group count, threshold not finite or < 0 or threshold * threshold not finite, minFrames < 2,
 *     maxFrames < minFrames or > RT_ADAPTIVE_MAX_FRAMES -> RT_E_INVALID; every state refusal of rtDispatch, "accumulate" = 0,
 *     "sampleChunks" forced to 2 or more, a group context (rtCreateMulti), a context with a communicator (rtCommInit) or with peers
 *     (rtSetPeers) -> RT_E_STATE.  A refused call changes nothing.
 * rtDisplayMean: W*H RGBA8, [y][x]: (0, 0, 0, 255) where AccumulatedRender.w == 0, else rtDisplay's encode of all four components of
 * A / A.w (the per-pixel mean of an adaptively sampled image).  Where every A.w equals "Frame" it is byte-equal to rtDisplay(1, Frame).
 * bytes != W*H*4 -> RT_E_INVALID.  Its scratch is the W*H float4 image rtReadbackAsync snapshots into (allocated by the first use of
 * either).  Synchronises. */
#ifndef RT_ADAPTIVE_EPSILON                /* overridable only by the A/B build variants of tools/build_variants.py */
#define RT_ADAPTIVE_EPSILON 0.00390625f    /* 2^-8 */
#endif
#define RT_ADAPTIVE_MAX_FRAMES (1 << 24)    /* the frame count is a binary32 in the moments image: exact up to 2^24 */
int rtDispatchAdaptive(RtContext* ctx, int groupsX, int groupsY, int groupsZ, float threshold, int minFrames, int maxFrames, int64_t* activePixels);
int rtDisplayMean(RtContext* ctx, uint8_t* dst, size_t bytes);

/* Replaces: reading the RenderTexture back (ComputeHelper.ReadbackData / AsyncGPUReadback; the
 * reference itself only samples it on-GPU in Display.shader).  tex ∈ {"FrameRender",
 * "AccumulatedRender"}; dst receives W·H float4 in [y][x] order (row 0 = bottom of the view plane),
 * bytes must equal W·H·16.  After the first rtDispatchFeatures also "AccumulatedAlbedo",
 * "AccumulatedNormal" (float4 as well) and "FeatureFrame" (W·H RtPixelFeatures: bytes must equal W·H·32), and after the first
 * rtDenoise "DenoisedRender" (float4), and after the first rtDenoiseTemporal "TemporalFrame" (float4).  Synchronises. */
int rtReadback(RtContext* ctx, const char* tex, float* dst, size_t bytes);

/* Replaces: RayTraceDisplay.OnRenderImage -> Graphics.Blit(rt, destination, displayMat) with Display.shader
 * (Assets/Scripts/Tracer/RayTraceDisplay.cs:9-23, Display.shader:42-47): col = tex / Frame, where tex is the accumulated
 * image and Frame = numAccumulatedFrames when accumulating, else the frame image and Frame = 1.  The quotient is then
 * encoded like Unity's linear-colour-space back buffer: clamp to [0,1], sRGB transfer function, 8 bits per channel.
 * dst receives W*H RGBA8 pixels in [y][x] order (row 0 = bottom), bytes must equal W*H*4.  Synchronises. */
int rtDisplay(RtContext* ctx, int useAccumulated, int Frame, uint8_t* dst, size_t bytes);

/* Pipelined forms of rtReadback / rtDisplay for hosts that read every frame: the call snapshots the texture (or encodes the
 * display image) on the dispatch stream as it is after the work queued so far, starts the device -> host copy on a stream of
 * its own and returns; the next rtDispatch runs while the copy is in flight.  dst (pinned memory for a real overlap) is valid
 * after rtReadbackWait (or rtSynchronize).  One copy in flight per context: a second call waits — on the device — for the first
 * copy to have read the snapshot. */
int rtReadbackAsync(RtContext* ctx, const char* tex, float* dst, size_t bytes);
int rtDisplayAsync(RtContext* ctx, int useAccumulated, int Frame, uint8_t* dst, size_t bytes);
int rtReadbackWait(RtContext* ctx);

/* Block until all work queued on this context has finished. */
int rtSynchronize(RtContext* ctx);

/* ---- extensions (no counterpart in the reference) ------------------------------------------------------- */

/* Run the context's work on a caller-owned CUDA stream (cudaStream_t passed as void*; NULL = the
 * context's own stream).  Lets a host that owns streams (e.g. torch) time and order the dispatches. */
int rtSetStream(RtContext* ctx, void* cudaStream);

/* Row-band tiling for multi-GPU rendering (SURVEY.md §8e): the image is cut into bands of bandRows
 * rows; band b belongs to rank (b mod worldSize).  After this call rtDispatch(RAYTRACE) traces only
 * this rank's bands (pixels keep their GLOBAL index, so seeds and results equal the 1-GPU run) and
 * writes them into the textures at their global position.  rank 0 / worldSize 1 = whole image. */
int rtSetTile(RtContext* ctx, int rank, int worldSize, int bandRows);

/* Gather / scatter staging for the per-frame all-gather of finished tiles.
 * rtPackTile   : copies this rank's bands of FrameRender and AccumulatedRender into the contiguous
 *                "TileSend" buffer ([frame bands | accumulated bands]).
 * rtUnpackTiles: scatters "TileRecv" (worldSize × TileSend, rank-major — what ncclAllGather produces)
 *                back into the two full-size textures.  Both are asynchronous on the context stream. */
int rtPackTile(RtContext* ctx);
int rtUnpackTiles(RtContext* ctx);

/* Fused tile exchange (alternative to rtPackTile / all-gather / rtUnpackTiles): every rank exports CUDA-IPC handles of
 * its two images (rtGetIpcHandles: 2 x 72 bytes = {cudaIpcMemHandle_t of the allocation, byte offset inside it} for
 * FrameRender and AccumulatedRender), the host
 * exchanges them, and each rank maps the images of the other ranks (rtSetPeers: nPeers x 2 x 72 bytes, at most 7 peers).
 * From then on the RayTrace kernel stores every finished pixel into its own images AND into every peer's, over NVLink,
 * as part of the kernel that produced it; the host only needs a stream-ordered barrier across ranks after the dispatch
 * before any rank reads its images.  rtResize with a new size and rtSetPeers(0) drop the mappings. */
int rtGetIpcHandles(RtContext* ctx, void* handles, size_t bytes);
int rtSetPeers(RtContext* ctx, int nPeers, const void* handles, size_t bytes);

/* ---- multi-GPU inside the boundary (SURVEY.md 8b / 8e) -----------------------------------------------------------------------
 * The reference host is ONE object issuing ONE dispatch per frame (RayComputeManager.RenderFrame, RCM:84-95); it must reach all
 * GPUs of the box without hand-rolling a collective.  Two ways, same exchange (pack this GPU's row bands -> one ncclAllGather
 * over NVLink -> scatter into both full-size textures, issued by rtDispatch(RT_KERNEL_RAYTRACE) itself on the context's stream):
 *
 *  (a) one process, several GPUs — what a Unity / C# host is:
 *        rtCreateMulti(&ctx, devices, n)   devices = n CUDA ordinals (NULL = 0 .. n-1).  The returned context LEADS a group: every
 *        rtSet* / rtSetBuffer / rtResize / rtSetOption call on it reaches all n GPUs (each keeps the whole scene, SURVEY 8e),
 *        rtDispatch traces tile r of n on GPU r and exchanges, rtReadback / rtDisplay read GPU devices[0], whose textures are
 *        complete after the exchange; rtGetStats sums the counters of the group (times: the slowest GPU).  rtDestroy frees all.
 *        n = 1 is rtCreate.  The call sequence of RayComputeManager does not change at all.
 *  (b) one process per GPU (torchrun, mpirun, N copies of a C++ host):
 *        rank 0: rtGetUniqueId(id, 128); the host hands the 128 bytes to the other ranks by any means (file, socket, MPI,
 *        torch.distributed store); every rank: rtCreate(&ctx, localDevice) + rtCommInit(ctx, id, 128, rank, world)  — collective,
 *        returns when all ranks have joined; it also makes the context render tile `rank` of `world` (rtSetTile, bands of 8 rows;
 *        call rtSetTile afterwards with the same rank / world to change bandRows).  rtCommDestroy returns to one GPU.
 *
 * NCCL is loaded at run time (the libnccl.so.2 already in the process, else the loader's; RT_B200_NCCL_LIB overrides): the
 * library has no link-time NCCL dependency and single-GPU hosts never load it.  Option "exchange" = 0 leaves the exchange to the
 * caller (rtExchangeTiles, or rtPackTile / own collective / rtUnpackTiles as in round 1). */
#define RT_UNIQUE_ID_BYTES 128
int rtCreateMulti(RtContext** out, const int* devices, int nDevices);
int rtGetUniqueId(void* id, size_t bytes);
int rtCommInit(RtContext* ctx, const void* id, size_t bytes, int rank, int worldSize);
int rtCommDestroy(RtContext* ctx);
/* The exchange alone (pack -> all-gather -> unpack), asynchronous on the context's stream(s).  rtDispatch calls it. */
int rtExchangeTiles(RtContext* ctx);

/* Device address + size of a named device object, for zero-copy plumbing (NCCL, torch views).
 * name ∈ {"FrameRender","AccumulatedRender","TileSend","TileRecv","PixelStats","FeatureFrame","AccumulatedAlbedo","AccumulatedNormal",
 * "DenoisedRender","TemporalFrame"}. */
int rtGetDevicePointer(RtContext* ctx, const char* name, void** devPtr, size_t* bytes);

/* Replaces `new BVH(mesh.vertices, mesh.triangles, mesh.normals, quality)` (BVH.cs:26; called once per shared mesh from
 * RayComputeManager.CreateAllMeshData, RayComputeManager.cs:209-232) by a build on the GPU that takes the reference's decisions
 * node for node — the same candidate planes, costs, split test and partition order — and therefore returns the Nodes and
 * Triangles buffers the reference's builder returns (mesh-relative indices, children adjacent, left subtree first, triangles
 * in leaf order).  verts / normals: vertCount x 3 floats; indices: 3 per triangle; quality: 0 Low, 1 High, 2 Disabled
 * (BVH.cs:11-16).  outTris: indexCount / 3 entries; outNodes: nodeCapacity >= 2 * triangles + 1 entries; *outNodeCount
 * receives the number of nodes written. */
int rtBuildBVH(RtContext* ctx, const float* verts, int vertCount, const int* indices, int indexCount, const float* normals, int quality,
               RtTriangle* outTris, RtNode* outNodes, int nodeCapacity, int* outNodeCount);

/* Tuning / instrumentation switches.  name ∈
 *   "kernel"      0 = reference-shaped per-pixel megakernel, 1 = persistent threads (one path per lane),
 *                 2 = persistent-thread wavefront with per-warp path pools, sorting and ray compaction,
 *                 -1 = automatic (default): 2 when the scene has meshes, 1 for sphere-only scenes and for tiles so small that
 *                 a pool slot gets about one pixel (below 1.5 pixels per slot; 2.5 with NumRaysPerPixel = 1: multi-GPU tiles),
 *                 and 1 whenever NumRaysPerPixel > RT_MAX_BATCH_SAMPLES.  Kernel 2 counts a pixel's samples in a 20-bit field, so
 *                 rtDispatch / rtDispatchAdaptive with "kernel" = 2 and NumRaysPerPixel > RT_MAX_BATCH_SAMPLES are refused
 *                 (RT_E_STATE, nothing changed); kernels 0 and 1 take any NumRaysPerPixel up to 2^31 - 1, like the reference
 *   "countStats"  1 = also count box / triangle tests (HL:254,271) — slower, off by default
 *   "sampleChunks"  kernel 1: a pixel's NumRaysPerPixel samples as this many consecutive jobs, the RNG state and the running sum
 *                 handed from the lane that finishes a chunk to the lane that takes the next (same samples in the same order:
 *                 same bits).  -1 (default) = automatic: mesh scenes on small tiles only (more than one and fewer than four
 *                 pixels per resident lane: multi-GPU tiles), about eight chunk-rounds per launch; 0 / 1 = whole pixels; 2..64 forced.
 *                 A forced value is an upper bound: kernel 1 counts at most 2^31 chunk jobs ((8x4-pixel tiles x 32) x chunks), so large
 *                 images get fewer chunks (whole pixels when fewer than two fit: 8192 x 8192 takes at most 32).  Same bits either way
 *   "exchange"    1 (default) = rtDispatch(RAYTRACE) on a context with a communicator (rtCommInit / rtCreateMulti) ends with the
 *                 all-gather of the frame's tiles; 0 = the caller exchanges (rtExchangeTiles or its own collective)
 *   "smemNodes"   number of top-of-tree node pairs staged in shared memory by TMA bulk copy (0 = off; -1 = automatic, which
 *                 is currently 0: the staging never beat leaving that shared memory to L1)
 *   "poolSlots"   paths per warp pool of kernel 2: 32, 64 or 96; 0 (default) = automatic, which is 64
 *   "modelSkip"   1 (default) = kernels 1 and 2 skip a model when the ray misses its padded world-space box or enters it beyond
 *                 the closest hit so far (exact: such a model cannot change the result); 0 = walk every model like the
 *                 reference.  Always 0 when "countStats" = 1, so that the test counts equal the reference's
 *   "tlas"        kernels 1 and 2, with "modelSkip" = 1: a tree over the models' padded world boxes (the per-frame model loop of
 *                 RayCommon.hlsl:347 for many-Model scenes).  One walk per ray segment marks the models the ray can reach; they
 *                 are then processed in buffer order against the running result, exactly like the linear loop, so the output
 *                 is unchanged.  Rebuilt on the host whenever ModelInfo is re-sent.  -1 (default) = automatic: used above 128
 *                 models; 0 = off; 1 = on for any model count (up to 4096 models; above that the linear test is used)
 *   "extInstantiation"  1 = launch the kernel instantiation that carries the extensions (peer stores, sphere accelerator)
 *                 even when none is active — for testing that instantiation on one GPU
 *   "sortRays"    kernel 2: 1 = group each warp's ray queue by direction octant before tracing, 0 = slot order (default;
 *                 off by default)
 *   "tailLanes"   kernel 2 leaves its trace phase when the ray queue is empty and at most this many lanes still trace
 *   "gridFit"     kernels 1 and 2: 1 = shrink the persistent grid so that every lane (pool slot) gets a whole number of pixels
 *                 — fewer, fully occupied rounds instead of a last round of mostly empty warps when the image is small for the
 *                 machine (multi-GPU tiles); 0 = one CTA set filling the machine (default; the fit is slower on whole images, kept as an option)
 *   "l2Persist"   1 = persisting L2 access-policy window over the node-pair records on the dispatch stream (0 = default; not yet
 *                 measured)
 *   "treeletPrefetch"  1 = two-level treelet layout with flagged treelet roots and an L1 prefetch of both possible next records
 *                 (only in a library built with -DRT_TREELET_PREFETCH; the default build returns RT_E_INVALID)
 *   "pairOrder"   order of the repacked node-pair records inside a mesh: 0 = breadth-first (default), d = 1..32 = treelets of d
 *                 levels laid out depth-first (1 = plain pre-order: child A's record follows its parent's).  Layout only: the
 *                 traversal visits the same nodes in the same order
 * Unknown names return RT_E_UNKNOWN_NAME. */
int rtSetOption(RtContext* ctx, const char* name, int value);

typedef struct RtStats {
    uint64_t rays;          /* CalculateRayCollision calls (HL:487) since the last rtResetStats          */
    uint64_t boxTests;      /* stats[1] (HL:271), only when "countStats" = 1                               */
    uint64_t triTests;      /* stats[0] (HL:254), only when "countStats" = 1                               */
    uint64_t sphereTests;   /* RaySphere calls (extension), only when "countStats" = 1                     */
    uint64_t dispatches;    /* RAYTRACE dispatches since the last reset                                    */
    double   kernelMs;      /* CUDA-event time of the RAYTRACE kernels since the last reset (sum)          */
    uint64_t sphereBoxTests;/* box tests of the sphere accelerator (Spheres buffers above 64 entries), "countStats" = 1;
                               with the accelerator, sphereTests counts the sphere tests actually made               */
    double   exchangeMs;    /* CUDA-event time of the per-frame tile exchanges (pack + ncclAllGather + unpack) issued by
                               rtDispatch / rtExchangeTiles since the last reset (sum)                              */
} RtStats;

/* Synchronises, then reports the counters accumulated since the last rtResetStats (which also zeroes "PixelStats"). */
int rtGetStats(RtContext* ctx, RtStats* out);
int rtResetStats(RtContext* ctx);

/* ---- per-pixel cost (the reference's debug view, HL:24-26,119: visMode / debugVisScale / stats, never written out there) ----
 * Every RT_KERNEL_RAYTRACE dispatch with "countStats" = 1 also adds each traced pixel's counts into the device image
 * "PixelStats": W*H RtPixelStats (rt_types.h), [y][x], row 0 = bottom, covering all samples and bounces of the pixel.  The image
 * is allocated (zero-filled) by the first counting dispatch, zeroed by rtResetStats and by rtResize to a new size, and accumulates
 * across dispatches in between, like RtStats.  Counts wrap modulo 2^32.  Pixels outside a partial dispatch or outside this
 * context's row bands (rtSetTile / rtCommInit) are not touched.  Not available on a group context (rtCreateMulti): RT_E_STATE.
 * rtGetDevicePointer also accepts "PixelStats" (after the first counting dispatch). */

/* W*H RtPixelStats, [y][x], row 0 = bottom; bytes must equal W*H*20.  RT_E_STATE before any counting dispatch.  Synchronises. */
int rtReadbackPixelStats(RtContext* ctx, RtPixelStats* dst, size_t bytes);

/* Heat map of PixelStats as W*H RGBA8 ([y][x], row 0 = bottom); bytes must equal W*H*4.  Synchronises.
 *   visMode 1: boxTests / rays   2: triTests / rays   3: (sphereTests + sphereBoxTests) / rays   4: rays (segments per pixel)
 *   debugVisScale: the value shown as full white; above it the pixel is red.  Must be finite and > 0.
 * Encode, binary32 with round-to-nearest-even, one operation at a time (so that any implementation restates it bit for bit):
 *   rays == 0                        -> (0, 0, 0, 255)
 *   v = (float)count / (float)rays   (mode 3: count = sphereTests + sphereBoxTests in uint32, wrapping; mode 4: v = (float)rays)
 *   t = v / debugVisScale
 *   t > 1                            -> (255, 0, 0, 255)
 *   else g = (uint8)trunc(t * 255 + 0.5)  -> (g, g, g, 255)
 * RT_E_INVALID for visMode outside 1..4, a bad debugVisScale or a wrong bytes; RT_E_STATE before any counting dispatch. */
int rtDisplayPixelStats(RtContext* ctx, int visMode, float debugVisScale, uint8_t* dst, size_t bytes);

/* ABI version of this header: (major << 16) | minor. */
int rtGetVersion(void);
#define RT_B200_VERSION ((1 << 16) | 1)

#ifdef __cplusplus
}
#endif

#endif /* RT_B200_H */
