// Shipped as source, NEVER COMPILED (no C# toolchain in the build image: dotnet, mono, mcs, csc are absent): the P/Invoke host for librt_b200.so.
// Compiled twin: ray_tracing_b200/host/RayComputeManager.cpp.  See INTEGRATION.md.
// Assets/Scripts/Tracer/RtB200.cs
using System;
using System.Runtime.InteropServices;
using Seb.AccelerationStructures;     // BVH (Assets/Scripts/Types/BVH.cs declares it in this namespace)

public static class RtB200
{
    const string Lib = "rt_b200";            // librt_b200.so next to the player / in Assets/Plugins/x86_64

    [DllImport(Lib)] public static extern int rtCreate(out IntPtr ctx, int device);
    [DllImport(Lib)] public static extern int rtDestroy(IntPtr ctx);
    [DllImport(Lib)] public static extern IntPtr rtLastError(IntPtr ctx);
    [DllImport(Lib)] public static extern int rtSetBuffer(IntPtr ctx, string name, BVH.Triangle[] data, int count, int stride);
    [DllImport(Lib)] public static extern int rtSetBuffer(IntPtr ctx, string name, BVH.Node[] data, int count, int stride);
    [DllImport(Lib)] public static extern int rtSetBuffer(IntPtr ctx, string name, RayTracingManager.MeshInfo[] data, int count, int stride);
    [DllImport(Lib)] public static extern int rtSetBuffer(IntPtr ctx, string name, RayTracingManager.Sphere[] data, int count, int stride);
    [DllImport(Lib)] public static extern int rtSetInt(IntPtr ctx, string name, int value);
    [DllImport(Lib)] public static extern int rtSetInts(IntPtr ctx, string name, int[] values, int n);
    [DllImport(Lib)] public static extern int rtSetFloat(IntPtr ctx, string name, float value);
    [DllImport(Lib)] public static extern int rtSetVector(IntPtr ctx, string name, ref UnityEngine.Vector4 value);
    [DllImport(Lib)] public static extern int rtSetMatrix(IntPtr ctx, string name, ref UnityEngine.Matrix4x4 value);   // column-major, as Unity stores it
    [DllImport(Lib)] public static extern int rtSetBool(IntPtr ctx, string name, int value);
    [DllImport(Lib)] public static extern int rtResize(IntPtr ctx, int width, int height);
    [DllImport(Lib)] public static extern int rtDispatch(IntPtr ctx, int kernelIndex, int gx, int gy, int gz);
    [DllImport(Lib)] public static extern int rtDispatchFrames(IntPtr ctx, int gx, int gy, int gz, int frameCount);
    [DllImport(Lib)] public static extern int rtReadback(IntPtr ctx, string tex, float[] dst, UIntPtr bytes);
    [DllImport(Lib)] public static extern int rtSynchronize(IntPtr ctx);
    // optional: new BVH(verts, indices, normals, quality) built on the GPU — the same Triangles / Nodes arrays (BVH.cs:26)
    [DllImport(Lib)] public static extern int rtBuildBVH(IntPtr ctx, UnityEngine.Vector3[] verts, int vertCount, int[] indices, int indexCount, UnityEngine.Vector3[] normals,
                                                         int quality, [Out] BVH.Triangle[] tris, [Out] BVH.Node[] nodes, int nodeCapacity, out int nodeCount);

    // Display.shader:42-47 (tex / Frame, sRGB 8-bit): RayTraceDisplay.OnRenderImage and the screenshot of RayComputeManager.cs:106-111
    [DllImport(Lib)] public static extern int rtDisplay(IntPtr ctx, int useAccumulated, int frame, byte[] rgba, UIntPtr bytes);

    // pipelined forms: the copy of frame k travels while frame k+1 renders (dst pinned: GCHandle.Alloc(..., GCHandleType.Pinned))
    [DllImport(Lib)] public static extern int rtReadbackAsync(IntPtr ctx, string tex, IntPtr dst, UIntPtr bytes);
    [DllImport(Lib)] public static extern int rtDisplayAsync(IntPtr ctx, int useAccumulated, int frame, IntPtr rgba, UIntPtr bytes);
    [DllImport(Lib)] public static extern int rtReadbackWait(IntPtr ctx);

    // ---- extensions (no counterpart in the reference) ----
    [DllImport(Lib)] public static extern int rtGetVersion();
    [DllImport(Lib)] public static extern int rtSetOption(IntPtr ctx, string name, int value);           // "kernel", "tlas", "modelSkip", ... (rt_b200.h)
    [DllImport(Lib)] public static extern int rtSetStream(IntPtr ctx, IntPtr cudaStream);
    [StructLayout(LayoutKind.Sequential)]
    public struct Stats { public ulong rays, boxTests, triTests, sphereTests, dispatches; public double kernelMs; public ulong sphereBoxTests; public double exchangeMs; }
    [DllImport(Lib)] public static extern int rtGetStats(IntPtr ctx, out Stats stats);
    [DllImport(Lib)] public static extern int rtResetStats(IntPtr ctx);
    // the reference's debug view (visMode / debugVisScale, RayCommon.hlsl:24-26): per-pixel counters of the "countStats" = 1 launches and their heat map
    [StructLayout(LayoutKind.Sequential)]
    public struct PixelStats { public uint rays, boxTests, triTests, sphereTests, sphereBoxTests; }
    [DllImport(Lib)] public static extern int rtReadbackPixelStats(IntPtr ctx, [Out] PixelStats[] dst, UIntPtr bytes);
    [DllImport(Lib)] public static extern int rtDisplayPixelStats(IntPtr ctx, int visMode, float debugVisScale, byte[] rgba, UIntPtr bytes);
    // closest-hit queries (CalculateRayCollision, RayCommon.hlsl:335-374): click to pick a Model, autofocus (focusDistance = hit.dst of the
    // centre pixel's ray), line of sight.  kind: 0 nothing hit, 1 Spheres[index], 2 ModelInfo[index]; flags 1 = forceDontCullBack
    [StructLayout(LayoutKind.Sequential)]
    public struct Ray { public UnityEngine.Vector3 origin, dir; }
    [StructLayout(LayoutKind.Sequential)]
    public struct RayHit { public float dst; public UnityEngine.Vector3 pos, normal; public int isBackface, kind, index, pad0, pad1; }
    [DllImport(Lib)] public static extern int rtTraceRays(IntPtr ctx, Ray[] rays, int n, [Out] RayHit[] hits, int flags);
    [DllImport(Lib)] public static extern int rtTraceRaysDevice(IntPtr ctx, IntPtr dRays, IntPtr dHits, int n, int flags);
    // occlusion queries: is anything on origin + t * dir, 0 <= t < tMax?  Shadow rays (tMax just below 1 with dir = light point - origin),
    // ambient occlusion, line of sight.  occluded[i] = 1 or 0; stops at the first hit, so cheaper than rtTraceRays for yes / no questions
    [StructLayout(LayoutKind.Sequential)]
    public struct RaySegment { public UnityEngine.Vector3 origin, dir; public float tMax; }
    [DllImport(Lib)] public static extern int rtTraceOcclusion(IntPtr ctx, RaySegment[] segs, int n, [Out] byte[] occluded, int flags);
    [DllImport(Lib)] public static extern int rtTraceOcclusionDevice(IntPtr ctx, IntPtr dSegs, IntPtr dOccluded, int n, int flags);
    // radiance along caller rays: the path tracer's Trace (glass / diffuse / specular / emissive, sky, Russian roulette) from origin along
    // dir (used as given), `samples` paths on the RNG chain that starts at rngState; out[i].rgb = their mean, out[i].rngState = the state
    // after the last one.  Custom cameras (360 panoramas, cube maps, fisheye, stereo), light / reflection probe baking
    [StructLayout(LayoutKind.Sequential)]
    public struct PathRay { public UnityEngine.Vector3 origin, dir; public uint rngState; }
    [StructLayout(LayoutKind.Sequential)]
    public struct PathRadiance { public UnityEngine.Vector3 rgb; public uint rngState; }
    [DllImport(Lib)] public static extern int rtTracePaths(IntPtr ctx, PathRay[] rays, int n, int samples, [Out] PathRadiance[] output);
    [DllImport(Lib)] public static extern int rtTracePathsDevice(IntPtr ctx, IntPtr dRays, IntPtr dOut, int n, int samples);
    // light probes: the radiance arriving at each position from `samples` spherical Fibonacci directions (the same for every probe), path
    // traced with state H(H(seed + p) + k) and projected onto the real L2 spherical harmonics.  sh[ch * 9 + i]: channel r, g, b, coefficient
    // i in Unity's SphericalHarmonicsL2 order, before its shader-constant conversion; rejected = samples left out for a non-finite radiance.
    // positions: 3 floats per probe (UnityEngine.Vector3[] marshals as such)
    [StructLayout(LayoutKind.Sequential)]
    public struct ProbeSH { [MarshalAs(UnmanagedType.ByValArray, SizeConst = 27)] public float[] sh; public uint rejected; }
    [DllImport(Lib)] public static extern int rtBakeProbes(IntPtr ctx, UnityEngine.Vector3[] positions, int n, int samples, uint seed, [Out] ProbeSH[] output);
    [DllImport(Lib)] public static extern int rtBakeProbesDevice(IntPtr ctx, IntPtr dPositions, IntPtr dOut, int n, int samples, uint seed);
    // reflection probes: an HDR cube map per position, output[((p * 6 + f) * N + y) * N + x] with faces in CubemapFace order (+X, -X, +Y,
    // -Y, +Z, -Z) and row 0 the top of the face; each texel the mean of `samples` paths over its area (R2 sub-texel offsets), rejected =
    // samples left out for a non-finite radiance (they count as black).  Cubemap.SetPixels takes one face's rows bottom-up: flip y.
    [StructLayout(LayoutKind.Sequential)]
    public struct CubeTexel { public UnityEngine.Vector3 rgb; public uint rejected; }
    [DllImport(Lib)] public static extern int rtBakeCubemaps(IntPtr ctx, UnityEngine.Vector3[] positions, int n, int faceSize, int samples, uint seed, [Out] CubeTexel[] output);
    [DllImport(Lib)] public static extern int rtBakeCubemapsDevice(IntPtr ctx, IntPtr dPositions, IntPtr dOut, int n, int faceSize, int samples, uint seed);
    // lightmaps: per surface texel (world position and normal; the normal need not be unit length) the mean of `samples` paths over the
    // normal's cosine-weighted hemisphere, output[p].rgb an estimate of E / pi (multiply by the surface's diffuse colour); rejected as
    // for cube maps.  INTEGRATION.md shows how Mesh.uv2 atlas texels become SurfacePoints.
    [StructLayout(LayoutKind.Sequential)]
    public struct SurfacePoint { public UnityEngine.Vector3 position; public UnityEngine.Vector3 normal; }
    [DllImport(Lib)] public static extern int rtBakeLightmap(IntPtr ctx, SurfacePoint[] points, int n, int samples, uint seed, [Out] CubeTexel[] output);
    [DllImport(Lib)] public static extern int rtBakeLightmapDevice(IntPtr ctx, IntPtr dPoints, IntPtr dOut, int n, int samples, uint seed);
    // one pixel of "FeatureFrame": object = ModelInfo index m -> m, Spheres index s -> -2 - s, miss -> -1 (dst = +inf, the rest 0)
    [StructLayout(LayoutKind.Sequential)]
    public struct PixelFeatures { public UnityEngine.Vector3 albedo; public float dst; public UnityEngine.Vector3 normal; public int objectId; }
    // first-hit feature images (denoiser guides) of every pixel's own camera ray, and those rays (W*H PathRay, [y][x], bytes = W*H*28)
    [DllImport(Lib)] public static extern int rtDispatchFeatures(IntPtr ctx, int groupsX, int groupsY, int groupsZ);
    [DllImport(Lib)] public static extern int rtCameraRays(IntPtr ctx, [Out] PathRay[] rays, UIntPtr bytes);
    [DllImport(Lib)] public static extern int rtCameraRaysDevice(IntPtr ctx, IntPtr dRays, UIntPtr bytes);
    [DllImport(Lib, EntryPoint = "rtReadback")] public static extern int rtReadbackFeatures(IntPtr ctx, string tex, [Out] PixelFeatures[] dst, UIntPtr bytes);   // tex = "FeatureFrame", bytes = W*H*32
    // the a-trous denoiser guided by the feature images: "DenoisedRender" (W*H float4 through rtReadback, the denoised mean colour) and its
    // display encode (W*H RGBA8, bytes = W*H*4).  iterations 1 .. 5; the managers default to 5, sigmas 64, 1, 0.1
    [DllImport(Lib)] public static extern int rtDenoise(IntPtr ctx, int useAccumulated, int iterations, float sigmaColour, float sigmaNormal, float sigmaDepth);
    [DllImport(Lib)] public static extern int rtDisplayDenoised(IntPtr ctx, [Out] byte[] dst, UIntPtr bytes);
    // the temporal (SVGF) denoiser for a moving camera, once per frame after rtDispatch and rtDispatchFeatures: "DenoisedRender" as above and
    // "TemporalFrame" (W*H float4 through rtReadback: prevX, prevY, history length, variance); the managers default to 5 iterations,
    // sigmas 8, 1, 0.1, alpha 0.1; resetHistory = 1 on a jump cut
    [DllImport(Lib)] public static extern int rtDenoiseTemporal(IntPtr ctx, int iterations, float sigmaLuminance, float sigmaNormal, float sigmaDepth, float alpha, int resetHistory);
    // adaptive sampling: the next accumulated frame only in the pixels whose error estimate is still above threshold; activePixels gets
    // the number traced (0 = converged).  "AdaptiveMoments" (W*H float4 through rtReadback); rtDisplayMean shows A / A.w per pixel.
    [DllImport(Lib)] public static extern int rtDispatchAdaptive(IntPtr ctx, int gx, int gy, int gz, float threshold, int minFrames, int maxFrames, out long activePixels);
    [DllImport(Lib)] public static extern int rtDisplayMean(IntPtr ctx, [Out] byte[] dst, UIntPtr bytes);
    // multi-GPU inside the boundary.  A Unity host is ONE process: rtCreateMulti(out ctx, null, 8) instead of rtCreate, and nothing else changes —
    // every rtSet* / rtSetBuffer reaches all GPUs, rtDispatch(kernelRayTrace) traces tile r of 8 on GPU r and ends with the NCCL all-gather of the frame's
    // tiles, rtReadback / rtDisplay read GPU 0.  One process per GPU instead: rtGetUniqueId on rank 0, rtCommInit on every rank.
    [DllImport(Lib)] public static extern int rtCreateMulti(out IntPtr ctx, int[] devices, int nDevices);
    [DllImport(Lib)] public static extern int rtGetUniqueId(byte[] id128, UIntPtr bytes);
    [DllImport(Lib)] public static extern int rtCommInit(IntPtr ctx, byte[] id128, UIntPtr bytes, int rank, int worldSize);
    [DllImport(Lib)] public static extern int rtCommDestroy(IntPtr ctx);
    [DllImport(Lib)] public static extern int rtExchangeTiles(IntPtr ctx);
    // row bands by hand (option "exchange" = 0): the caller owns the collective between rtPackTile and rtUnpackTiles
    [DllImport(Lib)] public static extern int rtSetTile(IntPtr ctx, int rank, int worldSize, int bandRows);
    [DllImport(Lib)] public static extern int rtPackTile(IntPtr ctx);
    [DllImport(Lib)] public static extern int rtUnpackTiles(IntPtr ctx);
    [DllImport(Lib)] public static extern int rtGetDevicePointer(IntPtr ctx, string name, out IntPtr devPtr, out UIntPtr bytes);
    [DllImport(Lib)] public static extern int rtGetIpcHandles(IntPtr ctx, byte[] handles, UIntPtr bytes);
    [DllImport(Lib)] public static extern int rtSetPeers(IntPtr ctx, int nPeers, byte[] handles, UIntPtr bytes);

    public static void Check(IntPtr ctx, int rc)
    {
        if (rc != 0) throw new InvalidOperationException("rt_b200: " + Marshal.PtrToStringAnsi(rtLastError(ctx)));
    }
}
